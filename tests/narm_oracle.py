"""float64 NumPy restatement of NARM as the device trains and ranks it (DESIGN §3s): the piece builder and the epoch plan, the
dropout masks, the forward pass and a hand-written backward pass of one mini-batch, Adam, the eval-mode encoder and the ranking
(bpr_oracle's sequential float64 scores of given q vectors against double(E)).  Written independently of the package's
vectorised helpers, which the tests compare against it.  Test infrastructure: the device (g4r_narm.cuh) is compared against it."""
import numpy as np

from gru4rec_oracle import dropout_mask
import bpr_oracle

STREAM_EMB, STREAM_CT = 200, 201
B1, B2, EPS = 0.9, 0.999, 1e-8
NAMES = ('E', 'Wx', 'Wrz', 'Wh', 'Bh', 'A1', 'A2', 'v', 'B')


def shapes(n_items, d, H):
    return [('E', (n_items, d)), ('Wx', (d, 3 * H)), ('Wrz', (H, 2 * H)), ('Wh', (H, H)), ('Bh', (3 * H,)), ('A1', (H, H)),
            ('A2', (H, H)), ('v', (H,)), ('B', (d, 2 * H))]


def unpack(flat, n_items, d, H):
    out, o = {}, 0
    for name, shp in shapes(n_items, d, H):
        n = int(np.prod(shp))
        out[name] = np.asarray(flat[o:o + n], dtype=np.float64).reshape(shp)
        o += n
    return out


def pack(p):
    return np.concatenate([p[n].ravel() for n in NAMES])


def init(n_items, d, H, rs):
    """Glorot-uniform draws in the vector's order, v as [H x 1]; Bh zero without a draw; float32"""
    parts = []
    for name, shp in shapes(n_items, d, H):
        if name == 'Bh':
            parts.append(np.zeros(3 * H))
            continue
        r, c = (shp[0], 1) if len(shp) == 1 else shp
        lim = np.sqrt(6.0 / (r + c))
        parts.append(rs.uniform(-lim, lim, size=shp).ravel())
    return np.concatenate(parts).astype(np.float32)


def pieces(sessions, max_len):
    """list of pieces (lists of item indices) from sessions (lists in time order), one loop"""
    out = []
    for s in sessions:
        a = 0
        while len(s) >= 2:
            b = min(a + max_len, len(s))
            out.append(list(s[a:b]))
            if b == len(s):
                break
            a = b - 1
    return out


def plan(n_items, d, H, n_pieces, seed, n_epochs):
    """(initial parameters, per epoch the permutation of the pieces) from one RandomState(seed)"""
    rs = np.random.RandomState(seed)
    th = init(n_items, d, H, rs)
    return th, [rs.permutation(n_pieces) for _ in range(n_epochs)]


def masks(seed, step, nb, max_len, d, H, p_emb, p_ct):
    """(embedding masks [nb, max_len, d], c masks [nb, max_len, 2H]) of one step: element (slot, t, unit) of each stream"""
    me = dropout_mask(seed, step, STREAM_EMB, (nb, max_len, d), p_emb).astype(np.float64)
    mc = dropout_mask(seed, step, STREAM_CT, (nb, max_len, 2 * H), p_ct).astype(np.float64)
    return me, mc


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def piece_forward(p, x, me=None, mc=None):
    """the causal encoder of one piece's inputs x: the cache and q [n, d] (masks [n, d] / [n, 2H] or None)"""
    H = p['Wh'].shape[0]
    n = len(x)
    emb = p['E'][x] * (me if me is not None else 1.0)
    h = np.zeros(H)
    hp, R, Z, HT, HS = [], [], [], [], []
    for t in range(n):
        vec = emb[t] @ p['Wx'] + p['Bh']
        rz = _sig(vec[H:] + h @ p['Wrz'])
        r, z = rz[:H], rz[H:]
        ht = np.tanh((h * r) @ p['Wh'] + vec[:H])
        hp.append(h); R.append(r); Z.append(z); HT.append(ht)
        h = (1.0 - z) * h + z * ht
        HS.append(h)
    hp, R, Z, HT, HS = map(np.array, (hp, R, Z, HT, HS))
    a1, a2 = HS @ p['A1'].T, HS @ p['A2'].T
    U = _sig(a1[:, None, :] + a2[None, :, :])                    # [t, j, H]
    AL = np.tril(U @ p['v'])                                     # alpha[t, j], j <= t
    C = np.concatenate([HS, AL @ HS], axis=1)
    mcv = mc if mc is not None else np.ones_like(C)
    Cm = C * mcv
    Q = Cm @ p['B'].T
    return dict(x=np.asarray(x), emb=emb, me=me, mc=mcv, hp=hp, R=R, Z=Z, HT=HT, HS=HS, U=U, AL=AL, Cm=Cm), Q


def batch_forward(p, batch, seed=0, step=0, p_emb=0.0, p_ct=0.0, max_len=None):
    """every piece of the batch (slot order): caches, Q [P, d], targets [P]"""
    H, d = p['Wh'].shape[0], p['E'].shape[1]
    L = max_len if max_len is not None else max(len(b) for b in batch)
    drop = p_emb > 0 or p_ct > 0
    me, mc = masks(seed, step, len(batch), L, d, H, p_emb, p_ct) if drop else (None, None)
    caches, qs, ys = [], [], []
    for b, pc in enumerate(batch):
        n = len(pc) - 1
        c, q = piece_forward(p, pc[:-1], None if me is None else me[b, :n], None if mc is None else mc[b, :n])
        caches.append(c); qs.append(q); ys.extend(pc[1:])
    return caches, np.concatenate(qs), np.array(ys)


def loss_and_grads(p, batch, seed=0, step=0, p_emb=0.0, p_ct=0.0, max_len=None, mag=False):
    """(mean loss, name -> gradient) of one mini-batch.  mag: the same backward over |every factor| with every difference
    made a sum -- per element the sum of the magnitudes of the terms the gradient adds up (the scale of its rounding error)"""
    caches, Q, Y = batch_forward(p, batch, seed, step, p_emb, p_ct, max_len)
    E = p['E']
    S = Q @ E.T
    m = S.max(axis=1, keepdims=True)
    ex = np.exp(S - m)
    pr = ex / ex.sum(axis=1, keepdims=True)
    P = len(Y)
    loss = float(np.mean(np.log(ex.sum(axis=1)) + m[:, 0] - S[np.arange(P), Y]))
    A = np.abs if mag else (lambda a: a)
    sub = (lambda a, b: a + b) if mag else (lambda a, b: a - b)
    pa = {k: A(v) for k, v in p.items()}
    if mag:
        dS = (pr + (np.arange(E.shape[0])[None, :] == Y[:, None])) / P
        Qa = np.concatenate([np.abs(c['Cm']) for c in caches]) @ np.abs(p['B']).T   # q's summands, not |q|: q may cancel
    else:
        dS = pr.copy()
        dS[np.arange(P), Y] -= 1.0
        dS /= P
        Qa = Q
    g = {k: np.zeros_like(v) for k, v in p.items()}
    dQ = dS @ pa['E']
    g['E'] += dS.T @ Qa
    H = p['Wh'].shape[0]
    o = 0
    for c in caches:
        n = len(c['x'])
        dq = dQ[o:o + n]
        o += n
        Cm, HS, U, AL = A(c['Cm']), A(c['HS']), c['U'], A(c['AL'])
        g['B'] += dq.T @ Cm
        dc = (dq @ pa['B']) * c['mc']
        ds, dh = dc[:, H:], dc[:, :H].copy()
        dA = np.tril(ds @ HS.T)                                  # d alpha[t, j]
        dh += AL.T @ ds
        gtj = dA[:, :, None] * pa['v'][None, None, :] * (U * (1.0 - U))   # [t, j, H]
        gtj = gtj * np.tril(np.ones((n, n)))[:, :, None]
        G1, G2 = gtj.sum(axis=1), gtj.sum(axis=0)
        g['v'] += np.einsum('tj,tjk->k', dA, U * np.tril(np.ones((n, n)))[:, :, None])
        g['A1'] += G1.T @ HS
        g['A2'] += G2.T @ HS
        dh += G1 @ pa['A1'] + G2 @ pa['A2']
        dn = np.zeros(H)
        for t in range(n - 1, -1, -1):
            hp, r, z, ht = A(c['hp'][t]), c['R'][t], c['Z'][t], A(c['HT'][t])
            dht = dh[t] + dn
            dz = dht * sub(ht, hp)
            dah = dht * z * (1.0 - ht * ht if not mag else 1.0 + ht * ht)
            dhr = pa['Wh'] @ dah
            g['Wh'] += np.outer(hp * r, dah)
            drz = np.concatenate([dhr * hp * r * (1.0 - r), dz * z * (1.0 - z)])
            g['Wrz'] += np.outer(hp, drz)
            dvec = np.concatenate([dah, drz])
            g['Wx'] += np.outer(A(c['emb'][t]), dvec)
            g['Bh'] += dvec
            dem = pa['Wx'] @ dvec
            g['E'][c['x'][t]] += dem * (c['me'][t] if c['me'] is not None else 1.0)
            dn = dht * (1.0 - z) + dhr * r + pa['Wrz'] @ drz
    return loss, g


def adam(theta, grad, m, v, t, lr):
    """one bias-corrected Adam step (Kingma & Ba): (theta, m, v) after step t (1-based), float64"""
    m = B1 * m + (1.0 - B1) * grad
    v = B2 * v + (1.0 - B2) * grad * grad
    mh, vh = m / (1.0 - B1 ** t), v / (1.0 - B2 ** t)
    return theta - lr * mh / (np.sqrt(vh) + EPS), m, v


def train(th0, shape, piece_list, orders, batch_size, lr, seed, p_emb, p_ct, max_len):
    """the fit of parameters of shape (n_items, d, H): per epoch, mini-batches of batch_size pieces in the order, one Adam step
    each.  Returns (theta, per-step losses)"""
    th = np.asarray(th0, dtype=np.float64)
    m, v = np.zeros_like(th), np.zeros_like(th)
    losses, step = [], 0
    for order in orders:
        for b0 in range(0, len(order), batch_size):
            batch = [piece_list[k] for k in order[b0:b0 + batch_size]]
            p = unpack(th, *shape)
            loss, g = loss_and_grads(p, batch, seed, step, p_emb, p_ct, max_len)
            step += 1
            th, m, v = adam(th, pack(g), m, v, step, lr)
            losses.append(loss)
    return th, losses


def encode(p, prefix, max_len):
    """eval-mode q of a prefix: the GRU over its last max_len inputs, then the attention and q of the last position only (the
    others' are not needed, and at max_len 512 the whole triangle would cost [n, n, H] doubles per event)"""
    H = p['Wh'].shape[0]
    h, HS = np.zeros(H), []
    for x in list(prefix)[-max_len:]:
        vec = p['E'][x] @ p['Wx'] + p['Bh']
        rz = _sig(vec[H:] + h @ p['Wrz'])
        r, z = rz[:H], rz[H:]
        h = (1.0 - z) * h + z * np.tanh((h * r) @ p['Wh'] + vec[:H])
        HS.append(h)
    HS = np.array(HS)
    alpha = _sig(HS[-1] @ p['A1'].T + HS @ p['A2'].T) @ p['v']
    return p['B'] @ np.concatenate([HS[-1], alpha @ HS])


def encode_events(p, items, offsets, n_history, max_len):
    """every counted event's q in evaluate's order"""
    out = []
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for pos in range(st + max(h, 1) - 1, en - 1):
            out.append(encode(p, items[st:pos + 1], max_len))
    return np.array(out).reshape(-1, p['E'].shape[1])


def rank_events(E, qs, items, offsets, n_history=None, mode='standard', cand=None, exclude_seen=False, k=0):
    """bpr_oracle.rank_events with each counted event's session vector replaced by qs[e]: scores against I = double(E), bI = 0"""
    I = np.asarray(E, dtype=np.float64)
    bI = np.zeros(I.shape[0])
    n_items = I.shape[0]
    items = np.asarray(items, dtype=np.int64)
    w0 = np.ones(n_items, np.int64) if cand is None else np.bincount(np.asarray(cand, dtype=np.int64), minlength=n_items)
    counts, li, ls = [], [], []
    e = 0
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for p in range(st + max(h, 1) - 1, en - 1):
            y = items[p + 1]
            prefix = items[st:p + 1]
            sc = bpr_oracle.scores(I, bI, np.asarray(qs[e], dtype=np.float64))
            w = w0.copy()
            if exclude_seen:
                w[prefix] = 0
            cmp = sc + bpr_oracle.tie_noise(e, np.arange(n_items)) if mode == 'tiebreaking' else sc
            t = cmp[y]
            if exclude_seen and y in set(prefix.tolist()):
                counts.append((-1, -1))
            else:
                counts.append((int(w[cmp > t].sum()), int(w[cmp == t].sum())))
            if k:
                elig = np.flatnonzero(w > 0)
                o = elig[np.lexsort((elig, -sc[elig]))][:k]
                row_i = np.full(k, -1, np.int64); row_s = np.full(k, np.nan)
                row_i[:len(o)] = o; row_s[:len(o)] = sc[o]
                li.append(row_i); ls.append(row_s)
            e += 1
    counts = np.array(counts, dtype=np.int64).reshape(-1, 2)
    if not k:
        return counts, None, None
    return counts, np.array(li).reshape(-1, k), np.array(ls).reshape(-1, k)
