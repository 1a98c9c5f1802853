"""float64 NumPy restatement of NextItNet as the device trains and ranks it (DESIGN §3w): the parameter layout and init, the
causal dilated convolutions, the forward pass of each piece and a hand-written backward pass of one mini-batch, with a magnitude
pass for the rounding bound, the encoder, the ranking of given q against W with the bias bW and, from narm_oracle, Adam and the
piece builder.  Written independently of the package's helpers, which the tests compare against it.  Test infrastructure: the
device (g4r_nextitnet.cuh) is compared against it."""
import numpy as np

import bpr_oracle
import narm_oracle

EPS_LN = 1e-8
BLOCK = ('C1', 'c1', 'g1', 'n1', 'C2', 'c2', 'g2', 'n2')
adam, B1, B2, EPS = narm_oracle.adam, narm_oracle.B1, narm_oracle.B2, narm_oracle.EPS


def pieces(sessions, max_len):
    """pieces of at most max_len inputs (max_len + 1 events), consecutive pieces overlapping by one event"""
    return narm_oracle.pieces(sessions, max_len + 1)


def shapes(n_items, d, dilations, K):
    out = [('E', (n_items, d))]
    for b in range(len(dilations)):
        out += [('%s_%d' % (k, b), (K * d, d) if k[0] == 'C' else (d,)) for k in BLOCK]
    return out + [('W', (n_items, d)), ('bW', (n_items,))]


def n_params(n_items, d, dilations, K):
    return 2 * n_items * d + n_items + len(dilations) * (2 * K * d * d + 6 * d)


def unpack(flat, n_items, d, dilations, K):
    out, o = {}, 0
    for name, shp in shapes(n_items, d, dilations, K):
        n = int(np.prod(shp))
        out[name] = np.asarray(flat[o:o + n], dtype=np.float64).reshape(shp)
        o += n
    assert o == len(flat)
    return out


def pack(p, dilations, K):
    NI, d = p['E'].shape
    return np.concatenate([p[n].ravel() for n, _ in shapes(NI, d, dilations, K)])


def init(n_items, d, dilations, K, rs):
    """Glorot-uniform draws for every matrix in the vector's order; biases 0, gains 1, no draws; float32"""
    parts = []
    for name, shp in shapes(n_items, d, dilations, K):
        if len(shp) == 2:
            lim = np.sqrt(6.0 / (shp[0] + shp[1]))
            parts.append(rs.uniform(-lim, lim, size=shp).ravel())
        else:
            parts.append(np.ones(shp) if name[0] == 'g' else np.zeros(shp))
    return np.concatenate(parts).astype(np.float32)


def plan(n_items, d, dilations, K, n_pieces, seed, n_epochs):
    rs = np.random.RandomState(seed)
    th = init(n_items, d, dilations, K, rs)
    return th, [rs.permutation(n_pieces) for _ in range(n_epochs)]


def taps(x, K, l):
    """the causal gather [n, K d]: block k of row t is x[t - (K - 1 - k) l], zero before the start"""
    n, d = x.shape
    col = np.zeros((n, K * d))
    for k in range(K):
        back = (K - 1 - k) * l
        if back < n:
            col[back:, k * d:(k + 1) * d] = x[:n - back]
    return col


def taps_adjoint(dcol, K, l):
    """the transpose of taps: dx[s] = sum_k dcol[s + (K - 1 - k) l, block k], zero past the end"""
    n = dcol.shape[0]
    d = dcol.shape[1] // K
    dx = np.zeros((n, d))
    for k in range(K):
        fwd = (K - 1 - k) * l
        if fwd < n:
            dx[:n - fwd] += dcol[fwd:, k * d:(k + 1) * d]
    return dx


def _ln(x, g, c):
    """(y, xh, rs, xa): xa = (|x| + |mean|) rs, the scale of xh's rounding (x - mean cancels)"""
    mu = x.mean(axis=1, keepdims=True)
    rs = 1.0 / np.sqrt(((x - mu) ** 2).mean(axis=1, keepdims=True) + EPS_LN)
    xh = (x - mu) * rs
    return g * xh + c, xh, rs, (np.abs(x) + np.abs(mu)) * rs


def _ln_bwd(dy, xh, rs, g, mag):
    """(dx, dg, dc); mag: each difference a sum over magnitudes"""
    e = dy * g
    if mag:
        dx = rs * (e + e.mean(axis=1, keepdims=True) + xh * (e * xh).mean(axis=1, keepdims=True))
    else:
        dx = rs * (e - e.mean(axis=1, keepdims=True) - xh * (e * xh).mean(axis=1, keepdims=True))
    return dx, (dy * xh).sum(axis=0), dy.sum(axis=0)


def piece_forward(p, x, dilations, K):
    """the causal encoder of one piece's inputs x: (cache, q [n, d]); q_t sees x_0 .. x_t only"""
    h = p['E'][list(x)]
    hm = np.abs(h)
    blocks = []
    for b, l in enumerate(dilations):
        w = {k: p['%s_%d' % (k, b)] for k in BLOCK}
        c = dict(hin=h, hm=hm, l=l)
        u = taps(h, K, l) @ w['C1'] + w['c1']
        y1, c['xh1'], c['rs1'], c['xa1'] = _ln(u, w['g1'], w['n1'])
        c['a'] = np.maximum(y1, 0.0)
        v = taps(c['a'], K, 2 * l) @ w['C2'] + w['c2']
        c['y2'], c['xh2'], c['rs2'], c['xa2'] = _ln(v, w['g2'], w['n2'])
        c['am'] = (c['xa1'] * np.abs(w['g1']) + np.abs(w['n1'])) * (c['a'] > 0)
        h = h + np.maximum(c['y2'], 0.0)
        hm = hm + (c['xa2'] * np.abs(w['g2']) + np.abs(w['n2'])) * (c['y2'] > 0)
        blocks.append(c)
    return dict(x=np.asarray(x), blocks=blocks, hm=hm), h


def batch_forward(p, batch, dilations, K):
    """every piece of the batch (slot order, pieces of inputs and targets): caches, Q [P, d], targets [P]"""
    caches, qs, ys = [], [], []
    for pc in batch:
        c, q = piece_forward(p, list(pc[:-1]), dilations, K)
        caches.append(c); qs.append(q); ys.extend(pc[1:])
    return caches, np.concatenate(qs), np.array(ys)


def loss_and_grads(p, batch, dilations, K, mag=False):
    """(mean loss, name -> gradient) of one mini-batch.  mag: the same backward over the magnitudes of every factor (forward values
    as the sums of their terms' magnitudes, every difference a sum): per element the scale of its rounding error"""
    caches, Qo, Y = batch_forward(p, batch, dilations, K)
    W, bW = p['W'], p['bW']
    S = Qo @ W.T + bW
    m = S.max(axis=1, keepdims=True)
    ex = np.exp(S - m)
    pr = ex / ex.sum(axis=1, keepdims=True)
    P = len(Y)
    loss = float(np.mean(np.log(ex.sum(axis=1)) + m[:, 0] - S[np.arange(P), Y]))
    A_ = np.abs if mag else (lambda a: a)
    pa = {k: A_(v) for k, v in p.items()}
    if mag:
        # a probability's relative rounding scales with its logit's and the row maximum's magnitudes (the sums of |q_u W_iu| + |bW_i|)
        Qa = np.concatenate([c['hm'] for c in caches])
        Sm = Qa @ pa['W'].T + pa['bW']
        dS = (pr * (1.0 + Sm + Sm.max(axis=1, keepdims=True)) + (np.arange(W.shape[0])[None, :] == Y[:, None])) / P
    else:
        dS = pr.copy()
        dS[np.arange(P), Y] -= 1.0
        dS /= P
        Qa = Qo
    g = {k: np.zeros_like(v) for k, v in p.items()}
    g['W'] += dS.T @ Qa
    g['bW'] += dS.sum(axis=0)
    dQo = dS @ pa['W']
    o = 0
    for c in caches:
        n = len(c['x'])
        dh = dQo[o:o + n]
        o += n
        for b in range(len(dilations) - 1, -1, -1):
            bc, l = c['blocks'][b], dilations[b]
            w = {k: pa['%s_%d' % (k, b)] for k in BLOCK}
            G = {k: g['%s_%d' % (k, b)] for k in BLOCK}
            a = bc['am'] if mag else bc['a']
            hin = bc['hm'] if mag else bc['hin']
            # h' = h + relu(LN2(v)), v = c2 + taps(a, 2l) C2
            dv, dg, dc = _ln_bwd(dh * (bc['y2'] > 0), bc['xa2'] if mag else bc['xh2'], bc['rs2'], w['g2'], mag)
            G['g2'] += dg; G['n2'] += dc
            G['C2'] += taps(a, K, 2 * l).T @ dv; G['c2'] += dv.sum(axis=0)
            da = taps_adjoint(dv @ w['C2'].T, K, 2 * l) * (bc['a'] > 0)
            # a = relu(LN1(u)), u = c1 + taps(h, l) C1
            du, dg, dc = _ln_bwd(da, bc['xa1'] if mag else bc['xh1'], bc['rs1'], w['g1'], mag)
            G['g1'] += dg; G['n1'] += dc
            G['C1'] += taps(hin, K, l).T @ du; G['c1'] += du.sum(axis=0)
            dh = dh + taps_adjoint(du @ w['C1'].T, K, l)
        np.add.at(g['E'], c['x'], dh)
    return loss, g


def train(th0, shape, piece_list, orders, batch_size, lr):
    """the fit of parameters of shape (n_items, d, dilations, K): per epoch, mini-batches of batch_size pieces in the order, one
    Adam step each.  Returns (theta, per-step losses)"""
    th = np.asarray(th0, dtype=np.float64)
    m, v = np.zeros_like(th), np.zeros_like(th)
    losses, step = [], 0
    for order in orders:
        for b0 in range(0, len(order), batch_size):
            batch = [piece_list[k] for k in order[b0:b0 + batch_size]]
            loss, g = loss_and_grads(unpack(th, *shape), batch, shape[2], shape[3])
            step += 1
            th, m, v = adam(th, pack(g, shape[2], shape[3]), m, v, step, lr)
            losses.append(loss)
    return th, losses


def encode(p, prefix, dilations, K, max_len):
    """q of a prefix: the encoder over its last max_len inputs, q of the last position"""
    return piece_forward(p, list(prefix)[-max_len:], dilations, K)[1][-1]


def encode_events(p, items, offsets, n_history, dilations, K, max_len):
    """every counted event's q in evaluate's order"""
    out = []
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for pos in range(st + max(h, 1) - 1, en - 1):
            out.append(encode(p, items[st:pos + 1], dilations, K, max_len))
    return np.array(out).reshape(-1, p['E'].shape[1])


def rank_events(W, bW, qs, items, offsets, n_history=None, mode='standard', cand=None, exclude_seen=False, k=0):
    """narm_oracle.rank_events against I = double(W) and bI = double(bW): per counted event (target counts), top-k items and scores"""
    I = np.asarray(W, dtype=np.float64)
    bI = np.asarray(bW, dtype=np.float64)
    n_items = I.shape[0]
    items = np.asarray(items, dtype=np.int64)
    w0 = np.ones(n_items, np.int64) if cand is None else np.bincount(np.asarray(cand, dtype=np.int64), minlength=n_items)
    counts, li, ls = [], [], []
    e = 0
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for pos in range(st + max(h, 1) - 1, en - 1):
            y = items[pos + 1]
            prefix = items[st:pos + 1]
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
