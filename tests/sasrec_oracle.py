"""float64 NumPy restatement of SASRec as the device trains and ranks it (DESIGN §3t): the parameter layout and init, the dropout
masks, the forward pass of each piece and a hand-written backward pass of one mini-batch, with a magnitude pass for the rounding
bound, the eval-mode encoder and, from narm_oracle, Adam, the piece builder and the ranking of given q vectors.  Written
independently of the package's helpers, which the tests compare against it.  Test infrastructure: the device (g4r_sasrec.cuh) is
compared against it."""
import numpy as np

from gru4rec_oracle import _mix32
import narm_oracle

STREAM_H0, STREAM_ATT, STREAM_FFN = 210, 211, 212
EPS_LN = 1e-8
BLOCK = ('g1', 'c1', 'Wq', 'bq', 'Wk', 'bk', 'Wv', 'bv', 'Wo', 'bo', 'g2', 'c2', 'W1', 'b1', 'W2', 'b2')
adam, rank_events, B1, B2, EPS = narm_oracle.adam, narm_oracle.rank_events, narm_oracle.B1, narm_oracle.B2, narm_oracle.EPS


def pieces(sessions, max_len):
    """pieces of at most max_len inputs (max_len + 1 events), consecutive pieces overlapping by one event"""
    return narm_oracle.pieces(sessions, max_len + 1)


def shapes(n_items, d, n_blocks, max_len):
    out = [('E', (n_items, d)), ('Pe', (max_len, d))]
    for b in range(n_blocks):
        out += [('%s_%d' % (k, b), (d, d) if k.startswith('W') else (d,)) for k in BLOCK]
    return out + [('gf', (d,)), ('cf', (d,))]


def n_params(n_items, d, n_blocks, max_len):
    return n_items * d + max_len * d + n_blocks * (6 * d * d + 10 * d) + 2 * d


def unpack(flat, n_items, d, n_blocks, max_len):
    out, o = {}, 0
    for name, shp in shapes(n_items, d, n_blocks, max_len):
        n = int(np.prod(shp))
        out[name] = np.asarray(flat[o:o + n], dtype=np.float64).reshape(shp)
        o += n
    assert o == len(flat)
    return out


def pack(p):
    d = p['E'].shape[1]
    nb = sum(1 for k in p if k.startswith('g1_'))
    return np.concatenate([p[n].ravel() for n, _ in shapes(p['E'].shape[0], d, nb, p['Pe'].shape[0])])


def init(n_items, d, n_blocks, max_len, rs):
    """Glorot-uniform draws for every matrix in the vector's order; biases 0, gains 1, no draws; float32"""
    parts = []
    for name, shp in shapes(n_items, d, n_blocks, max_len):
        if len(shp) == 2:
            lim = np.sqrt(6.0 / (shp[0] + shp[1]))
            parts.append(rs.uniform(-lim, lim, size=shp).ravel())
        else:
            parts.append(np.ones(shp) if name[0] == 'g' else np.zeros(shp))
    return np.concatenate(parts).astype(np.float32)


def plan(n_items, d, n_blocks, max_len, n_pieces, seed, n_epochs):
    rs = np.random.RandomState(seed)
    th = init(n_items, d, n_blocks, max_len, rs)
    return th, [rs.permutation(n_pieces) for _ in range(n_epochs)]


def scales(d, n_heads):
    return float(np.float32(np.sqrt(float(d)))), float(np.float32(1.0 / np.sqrt(float(d // n_heads))))


def mask(seed, step, stream, idx, p):
    """the dropout factors (0 or 1 / retain in float32) of mask indices idx"""
    if p <= 0.0:
        return np.ones(np.shape(idx))
    retain = np.float32(1.0 - p)
    with np.errstate(over='ignore'):
        k = _mix32(np.array([np.uint32(seed) ^ (np.uint32(0x9E3779B9) * np.uint32(stream + 1))], dtype=np.uint32))
        k = _mix32(k + np.uint32(step))
        r = _mix32(k + np.asarray(idx, dtype=np.uint64).astype(np.uint32))
    u = (r >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return ((u < retain).astype(np.float32) / retain).astype(np.float64)


def piece_masks(seed, step, p, slot, n, d, n_blocks, bs, L):
    """per mask block (0: h0, b + 1: block b) the [n, d] factors of a piece in slot `slot`: index ((blk bs + slot) L + t) d + u"""
    t, u = np.meshgrid(np.arange(n), np.arange(d), indexing='ij')
    out = []
    for blk in range(n_blocks + 1):
        idx = ((blk * bs + slot) * L + t) * d + u
        if blk == 0:
            out.append(mask(seed, step, STREAM_H0, idx, p))
        else:
            out.append((mask(seed, step, STREAM_ATT, idx, p), mask(seed, step, STREAM_FFN, idx, p)))
    return out


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


def piece_forward(p, x, n_heads, masks=None):
    """the causal encoder of one piece's inputs x: (cache, q [n, d]).  masks: piece_masks, or None (eval mode)"""
    d = p['E'].shape[1]
    dh = d // n_heads
    sd, sh = scales(d, n_heads)
    n = len(x)
    nb = sum(1 for k in p if k.startswith('g1_'))
    m0 = masks[0] if masks is not None else np.ones((n, d))
    h = (p['E'][x] * sd + p['Pe'][:n]) * m0
    causal = np.tril(np.ones((n, n), bool))
    blocks = []
    for b in range(nb):
        w = {k: p['%s_%d' % (k, b)] for k in BLOCK}
        ma, mf = masks[b + 1] if masks is not None else (np.ones((n, d)), np.ones((n, d)))
        c = dict(hin=h, ma=ma, mf=mf)
        c['u1'], c['xh1'], c['rs1'], c['xa1'] = _ln(h, w['g1'], w['c1'])
        c['Q'], c['K'], c['V'] = (c['u1'] @ w[k] + w['b' + k[1]] for k in ('Wq', 'Wk', 'Wv'))
        c['P'] = []
        A = np.zeros((n, d))
        for k in range(n_heads):
            cs = slice(k * dh, (k + 1) * dh)
            S = np.where(causal, (c['Q'][:, cs] @ c['K'][:, cs].T) * sh, -np.inf)
            P = np.exp(S - S.max(axis=1, keepdims=True))
            P /= P.sum(axis=1, keepdims=True)
            c['P'].append(P)
            A[:, cs] = P @ c['V'][:, cs]
        c['A'] = A
        a = h + ma * (A @ w['Wo'] + w['bo'])
        c['ar'] = a
        c['u2'], c['xh2'], c['rs2'], c['xa2'] = _ln(a, w['g2'], w['c2'])
        c['F1'] = np.maximum(c['u2'] @ w['W1'] + w['b1'], 0.0)
        h = a + mf * (c['F1'] @ w['W2'] + w['b2'])
        blocks.append(c)
    q, xhf, rsf, xaf = _ln(h, p['gf'], p['cf'])
    return dict(x=np.asarray(x), m0=m0, blocks=blocks, xhf=xhf, rsf=rsf, xaf=xaf, q=q), q


def batch_forward(p, batch, n_heads, seed=0, step=0, dropout=0.0, max_len=None, bs=None):
    """every piece of the batch (slot order, pieces of inputs and targets): caches, Q [P, d], targets [P]"""
    d = p['E'].shape[1]
    nb = sum(1 for k in p if k.startswith('g1_'))
    L = max_len if max_len is not None else p['Pe'].shape[0]
    bs = bs if bs is not None else len(batch)
    caches, qs, ys = [], [], []
    for slot, pc in enumerate(batch):
        n = len(pc) - 1
        masks = piece_masks(seed, step, dropout, slot, n, d, nb, bs, L) if dropout > 0 else None
        c, q = piece_forward(p, list(pc[:-1]), n_heads, masks)
        caches.append(c); qs.append(q); ys.extend(pc[1:])
    return caches, np.concatenate(qs), np.array(ys)


def loss_and_grads(p, batch, n_heads, seed=0, step=0, dropout=0.0, max_len=None, bs=None, mag=False):
    """(mean loss, name -> gradient) of one mini-batch.  mag: the same backward over the magnitudes of every factor (forward values
    as the sums of their terms' magnitudes, every difference a sum): per element the scale of its rounding error"""
    caches, Qo, Y = batch_forward(p, batch, n_heads, seed, step, dropout, max_len, bs)
    E = p['E']
    d = E.shape[1]
    dh = d // n_heads
    sd, sh = scales(d, n_heads)
    nb = sum(1 for k in p if k.startswith('g1_'))
    S = Qo @ E.T
    m = S.max(axis=1, keepdims=True)
    ex = np.exp(S - m)
    pr = ex / ex.sum(axis=1, keepdims=True)
    P = len(Y)
    loss = float(np.mean(np.log(ex.sum(axis=1)) + m[:, 0] - S[np.arange(P), Y]))
    A_ = np.abs if mag else (lambda a: a)
    pa = {k: A_(v) for k, v in p.items()}
    if mag:
        # q's rounding scales with the normalisation's operands; a probability's relative rounding with its logit's and the row
        # maximum's magnitudes (the sums of |q_u E_iu|)
        Qa = np.concatenate([c['xaf'] * pa['gf'] + pa['cf'] for c in caches])
        Sm = Qa @ np.abs(E).T
        dS = (pr * (1.0 + Sm + Sm.max(axis=1, keepdims=True)) + (np.arange(E.shape[0])[None, :] == Y[:, None])) / P
    else:
        dS = pr.copy()
        dS[np.arange(P), Y] -= 1.0
        dS /= P
        Qa = Qo
    g = {k: np.zeros_like(v) for k, v in p.items()}
    dQo = dS @ pa['E']
    g['E'] += dS.T @ Qa
    o = 0
    for c in caches:
        n = len(c['x'])
        dq = dQo[o:o + n]
        o += n
        dh_, dg, dc = _ln_bwd(dq, c['xaf'] if mag else c['xhf'], c['rsf'], pa['gf'], mag)
        g['gf'] += dg; g['cf'] += dc
        for b in range(nb - 1, -1, -1):
            bc = c['blocks'][b]
            w = {k: pa['%s_%d' % (k, b)] for k in BLOCK}
            G = {k: g['%s_%d' % (k, b)] for k in BLOCK}
            u1 = bc['xa1'] * w['g1'] + w['c1'] if mag else bc['u1']
            u2 = bc['xa2'] * w['g2'] + w['c2'] if mag else bc['u2']
            F1 = (bc['F1'] > 0) * (u2 @ w['W1'] + w['b1']) if mag else bc['F1']
            Qm, Km, Vm = ((u1 @ w[k] + w['b' + k[1]]) for k in ('Wq', 'Wk', 'Wv')) if mag else (bc['Q'], bc['K'], bc['V'])
            # the FFN
            dF2 = dh_ * bc['mf']
            G['W2'] += F1.T @ dF2; G['b2'] += dF2.sum(axis=0)
            dZ = (dF2 @ w['W2'].T) * (bc['F1'] > 0)
            G['W1'] += u2.T @ dZ; G['b1'] += dZ.sum(axis=0)
            du2 = dZ @ w['W1'].T
            dx, dg, dc = _ln_bwd(du2, bc['xa2'] if mag else bc['xh2'], bc['rs2'], w['g2'], mag)
            G['g2'] += dg; G['c2'] += dc
            da = dh_ + dx
            # the attention
            dO = da * bc['ma']
            Am = np.zeros((n, d)) if mag else bc['A']
            if mag:
                for k in range(n_heads):
                    cs = slice(k * dh, (k + 1) * dh)
                    Am[:, cs] = bc['P'][k] @ Vm[:, cs]
            G['Wo'] += Am.T @ dO; G['bo'] += dO.sum(axis=0)
            dA = dO @ w['Wo'].T
            dQ, dK, dV = np.zeros((n, d)), np.zeros((n, d)), np.zeros((n, d))
            for k in range(n_heads):
                cs = slice(k * dh, (k + 1) * dh)
                Pk = bc['P'][k]
                dV[:, cs] = Pk.T @ dA[:, cs]
                dP = np.tril(dA[:, cs] @ Vm[:, cs].T)
                D = (dA[:, cs] * Am[:, cs]).sum(axis=1, keepdims=True)
                dSk = Pk * (dP + D) if mag else Pk * (dP - D)
                dQ[:, cs] = sh * dSk @ Km[:, cs]
                dK[:, cs] = sh * dSk.T @ Qm[:, cs]
            du1 = np.zeros((n, d))
            for dX, Wn, bn in ((dQ, 'Wq', 'bq'), (dK, 'Wk', 'bk'), (dV, 'Wv', 'bv')):
                G[Wn] += u1.T @ dX; G[bn] += dX.sum(axis=0)
                du1 += dX @ w[Wn].T
            dx, dg, dc = _ln_bwd(du1, bc['xa1'] if mag else bc['xh1'], bc['rs1'], w['g1'], mag)
            G['g1'] += dg; G['c1'] += dc
            dh_ = da + dx
        dpre = dh_ * c['m0']
        g['Pe'][:n] += dpre
        np.add.at(g['E'], c['x'], dpre * sd)
    return loss, g


def train(th0, shape, n_heads, piece_list, orders, batch_size, lr, seed, dropout):
    """the fit of parameters of shape (n_items, d, n_blocks, max_len): per epoch, mini-batches of batch_size pieces in the order,
    one Adam step each.  Returns (theta, per-step losses)"""
    th = np.asarray(th0, dtype=np.float64)
    m, v = np.zeros_like(th), np.zeros_like(th)
    losses, step = [], 0
    for order in orders:
        for b0 in range(0, len(order), batch_size):
            batch = [piece_list[k] for k in order[b0:b0 + batch_size]]
            loss, g = loss_and_grads(unpack(th, *shape), batch, n_heads, seed, step, dropout, shape[3], batch_size)
            step += 1
            th, m, v = adam(th, pack(g), m, v, step, lr)
            losses.append(loss)
    return th, losses


def encode(p, prefix, n_heads, max_len):
    """eval-mode q of a prefix: the encoder over its last max_len inputs, q of the last position"""
    return piece_forward(p, list(prefix)[-max_len:], n_heads)[1][-1]


def encode_events(p, items, offsets, n_history, n_heads, max_len):
    """every counted event's q in evaluate's order"""
    out = []
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for pos in range(st + max(h, 1) - 1, en - 1):
            out.append(encode(p, items[st:pos + 1], n_heads, max_len))
    return np.array(out).reshape(-1, p['E'].shape[1])
