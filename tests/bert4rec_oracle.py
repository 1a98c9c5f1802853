"""float64 NumPy restatement of BERT4Rec as the device trains and ranks it (DESIGN §3x): the parameter layout and init, the cloze
masks, the dropout masks, the forward pass of each piece and a hand-written backward pass of one mini-batch, with a magnitude pass
for the rounding bound, the eval-mode encoder and, from narm_oracle / sasrec_oracle / nextitnet_oracle, Adam, the piece builder,
the dropout hash and the ranking of given q vectors with an output bias.  Written independently of the package's helpers, which
the tests compare against it.  Test infrastructure: the device (g4r_bert4rec.cuh) is compared against it."""
import math

import numpy as np

import narm_oracle
import nextitnet_oracle
import sasrec_oracle

STREAM_H0, STREAM_ATT, STREAM_FFN = 220, 221, 222
EPS_LN = 1e-8
BLOCK = ('Wq', 'bq', 'Wk', 'bk', 'Wv', 'bv', 'Wo', 'bo', 'g1', 'c1', 'W1', 'b1', 'W2', 'b2', 'g2', 'c2')
adam, B1, B2, EPS = narm_oracle.adam, narm_oracle.B1, narm_oracle.B2, narm_oracle.EPS
rank_events = nextitnet_oracle.rank_events
_erf = np.frompyfunc(math.erf, 1, 1)


def pieces(sessions, max_len):
    """pieces of at most max_len events, all of them inputs, consecutive pieces overlapping by one event"""
    return narm_oracle.pieces(sessions, max_len)


def shapes(n_items, d, n_blocks, max_len):
    out = [('E', (n_items + 1, d)), ('Pe', (max_len, d)), ('g0', (d,)), ('c0', (d,))]
    wide = {'W1': (d, 4 * d), 'b1': (4 * d,), 'W2': (4 * d, d)}
    for b in range(n_blocks):
        out += [('%s_%d' % (k, b), wide.get(k, (d, d) if k.startswith('W') else (d,))) for k in BLOCK]
    return out + [('Wp', (d, d)), ('bp', (d,)), ('gp', (d,)), ('cp', (d,)), ('bO', (n_items,))]


def n_params(n_items, d, n_blocks, max_len):
    return (n_items + 1) * d + max_len * d + 2 * d + n_blocks * (12 * d * d + 13 * d) + d * d + 3 * d + n_items


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
    return np.concatenate([p[n].ravel() for n, _ in shapes(p['E'].shape[0] - 1, d, nb, p['Pe'].shape[0])])


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


def cloze(piece_lens, mask_prob, rs):
    """one epoch's masks, a list per piece (storage order): an entry is masked when its draw of one rs.random_sample over every
    entry is below mask_prob; a piece with none masked gets its last entry masked"""
    u = rs.random_sample(int(sum(piece_lens)))
    out, o = [], 0
    for n in piece_lens:
        m = [bool(v < mask_prob) for v in u[o:o + n]]
        if not any(m):
            m[-1] = True
        out.append(m)
        o += n
    return out


def plan(n_items, d, n_blocks, max_len, piece_lens, seed, n_epochs, mask_prob):
    """the init, then per epoch (order, masks) drawn from one RandomState(seed)"""
    rs = np.random.RandomState(seed)
    th = init(n_items, d, n_blocks, max_len, rs)
    out = []
    for _ in range(n_epochs):
        order = rs.permutation(len(piece_lens))
        out.append((order, cloze(piece_lens, mask_prob, rs)))
    return th, out


def piece_masks(seed, step, p, slot, n, d, n_blocks, bs, L):
    """per mask block (0: h0, b + 1: block b) the [n, d] factors of a piece in slot `slot`: index ((blk bs + slot) L + t) d + u"""
    t, u = np.meshgrid(np.arange(n), np.arange(d), indexing='ij')
    out = []
    for blk in range(n_blocks + 1):
        idx = ((blk * bs + slot) * L + t) * d + u
        if blk == 0:
            out.append(sasrec_oracle.mask(seed, step, STREAM_H0, idx, p))
        else:
            out.append((sasrec_oracle.mask(seed, step, STREAM_ATT, idx, p), sasrec_oracle.mask(seed, step, STREAM_FFN, idx, p)))
    return out


def _ln(x, g, c):
    """(y, xh, rs, xa): xa = (|x| + |mean|) rs, the scale of xh's rounding (x - mean cancels)"""
    mu = x.mean(axis=1, keepdims=True)
    rs = 1.0 / np.sqrt(((x - mu) ** 2).mean(axis=1, keepdims=True) + EPS_LN)
    xh = (x - mu) * rs
    return g * xh + c, xh, rs, (np.abs(x) + np.abs(mu)) * rs


def _ln_bwd(dy, xh, rs, g, mag):
    e = dy * g
    if mag:
        dx = rs * (e + e.mean(axis=1, keepdims=True) + xh * (e * xh).mean(axis=1, keepdims=True))
    else:
        dx = rs * (e - e.mean(axis=1, keepdims=True) - xh * (e * xh).mean(axis=1, keepdims=True))
    return dx, (dy * xh).sum(axis=0), dy.sum(axis=0)


def _cdf(z):
    return 0.5 * (1.0 + _erf(z / np.sqrt(2.0)).astype(np.float64))


def _pdf(z):
    return np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi)


def gelu(z):
    return z * _cdf(z)


def gelu_grad(z, mag=False):
    """gelu'(z) = Phi(z) + z phi(z); mag: Phi(z) + |z| phi(z)"""
    return _cdf(z) + (np.abs(z) if mag else z) * _pdf(z)


def _nb(p):
    return sum(1 for k in p if k.startswith('g1_'))


def piece_forward(p, x, masked, n_heads, masks=None):
    """the bidirectional encoder of one piece's inputs x, the entries where masked is true replaced by the mask token: (cache,
    q [n, d]).  masks: piece_masks, or None (eval mode)"""
    NI = p['E'].shape[0] - 1
    d = p['E'].shape[1]
    dh = d // n_heads
    sh = sasrec_oracle.scales(d, n_heads)[1]
    n = len(x)
    xs = np.where(np.asarray(masked, bool), NI, np.asarray(x))
    m0 = masks[0] if masks is not None else np.ones((n, d))
    c0 = dict(xs=xs, m0=m0)
    y0, c0['xh'], c0['rs'], c0['xa'] = _ln(p['E'][xs] + p['Pe'][:n], p['g0'], p['c0'])
    h = y0 * m0
    blocks = []
    for b in range(_nb(p)):
        w = {k: p['%s_%d' % (k, b)] for k in BLOCK}
        ma, mf = masks[b + 1] if masks is not None else (np.ones((n, d)), np.ones((n, d)))
        c = dict(hin=h, ma=ma, mf=mf)
        c['Q'], c['K'], c['V'] = (h @ w[k] + w['b' + k[1]] for k in ('Wq', 'Wk', 'Wv'))
        c['P'] = []
        A = np.zeros((n, d))
        for k in range(n_heads):
            cs = slice(k * dh, (k + 1) * dh)
            S = (c['Q'][:, cs] @ c['K'][:, cs].T) * sh
            P = np.exp(S - S.max(axis=1, keepdims=True))
            P /= P.sum(axis=1, keepdims=True)
            c['P'].append(P)
            A[:, cs] = P @ c['V'][:, cs]
        c['A'] = A
        c['a1'], c['xh1'], c['rs1'], c['xa1'] = _ln(h + ma * (A @ w['Wo'] + w['bo']), w['g1'], w['c1'])
        c['Z1'] = c['a1'] @ w['W1'] + w['b1']
        c['G1'] = gelu(c['Z1'])
        h, c['xh2'], c['rs2'], c['xa2'] = _ln(c['a1'] + mf * (c['G1'] @ w['W2'] + w['b2']), w['g2'], w['c2'])
        blocks.append(c)
    ZH = h @ p['Wp'] + p['bp']
    q, xhp, rsp, xap = _ln(gelu(ZH), p['gp'], p['cp'])
    return dict(c0=c0, blocks=blocks, hout=h, ZH=ZH, xhp=xhp, rsp=rsp, xap=xap, q=q), q


def batch_forward(p, batch, masked, n_heads, seed=0, step=0, dropout=0.0, max_len=None, bs=None):
    """every piece of the batch (slot order) with its cloze masks: caches, q of the masked positions [Pm, d], their targets [Pm]"""
    d = p['E'].shape[1]
    L = max_len if max_len is not None else p['Pe'].shape[0]
    bs = bs if bs is not None else len(batch)
    caches, qs, ys = [], [], []
    for slot, (pc, mk) in enumerate(zip(batch, masked)):
        n = len(pc)
        masks = piece_masks(seed, step, dropout, slot, n, d, _nb(p), bs, L) if dropout > 0 else None
        c, q = piece_forward(p, list(pc), mk, n_heads, masks)
        at = np.flatnonzero(mk)
        c['at'] = at
        caches.append(c); qs.append(q[at]); ys.extend(np.asarray(pc)[at])
    return caches, np.concatenate(qs), np.array(ys)


def loss_and_grads(p, batch, masked, n_heads, seed=0, step=0, dropout=0.0, max_len=None, bs=None, mag=False):
    """(mean loss over the masked positions, name -> gradient) of one mini-batch.  mag: the same backward over the magnitudes of
    every factor (forward values as the sums of their terms' magnitudes, every difference a sum): per element the scale of its
    rounding error"""
    caches, Qo, Y = batch_forward(p, batch, masked, n_heads, seed, step, dropout, max_len, bs)
    NI = p['E'].shape[0] - 1
    E = p['E'][:NI]
    d = E.shape[1]
    dh = d // n_heads
    sh = sasrec_oracle.scales(d, n_heads)[1]
    nb = _nb(p)
    S = Qo @ E.T + p['bO']
    m = S.max(axis=1, keepdims=True)
    ex = np.exp(S - m)
    pr = ex / ex.sum(axis=1, keepdims=True)
    Pm = len(Y)
    loss = float(np.mean(np.log(ex.sum(axis=1)) + m[:, 0] - S[np.arange(Pm), Y]))
    A_ = np.abs if mag else (lambda a: a)
    pa = {k: A_(v) for k, v in p.items()}
    if mag:
        Qa = np.concatenate([(c['xap'] * pa['gp'] + pa['cp'])[c['at']] for c in caches])
        Sm = Qa @ np.abs(E).T + pa['bO']
        dS = (pr * (1.0 + Sm + Sm.max(axis=1, keepdims=True)) + (np.arange(NI)[None, :] == Y[:, None])) / Pm
    else:
        dS = pr.copy()
        dS[np.arange(Pm), Y] -= 1.0
        dS /= Pm
        Qa = Qo
    g = {k: np.zeros_like(v) for k, v in p.items()}
    dQo = dS @ pa['E'][:NI]
    g['E'][:NI] += dS.T @ Qa
    g['bO'] += dS.sum(axis=0)
    o = 0
    for c in caches:
        n = len(c['c0']['xs'])
        dq = np.zeros((n, d))
        dq[c['at']] = dQo[o:o + len(c['at'])]
        o += len(c['at'])
        # the head
        dGH, dg, dc = _ln_bwd(dq, c['xap'] if mag else c['xhp'], c['rsp'], pa['gp'], mag)
        g['gp'] += dg; g['cp'] += dc
        dZH = dGH * gelu_grad(c['ZH'], mag)
        blk = c['blocks']
        hL = (blk[-1]['xa2'] * pa['g2_%d' % (nb - 1)] + pa['c2_%d' % (nb - 1)]) if mag else c['hout']
        g['Wp'] += hL.T @ dZH; g['bp'] += dZH.sum(axis=0)
        dh_ = dZH @ pa['Wp'].T
        for b in range(nb - 1, -1, -1):
            bc = blk[b]
            w = {k: pa['%s_%d' % (k, b)] for k in BLOCK}
            G = {k: g['%s_%d' % (k, b)] for k in BLOCK}
            if mag:
                hin = (c['c0']['xa'] * pa['g0'] + pa['c0']) * c['c0']['m0'] if b == 0 else blk[b - 1]['xa2'] * pa['g2_%d' % (b - 1)] + pa['c2_%d' % (b - 1)]
                a1 = bc['xa1'] * w['g1'] + w['c1']
                Zm = a1 @ w['W1'] + w['b1']
                G1 = gelu_grad(bc['Z1'], True) * Zm
                Qm, Km, Vm = (hin @ w[k] + w['b' + k[1]] for k in ('Wq', 'Wk', 'Wv'))
            else:
                hin, a1, G1, Qm, Km, Vm = bc['hin'], bc['a1'], bc['G1'], bc['Q'], bc['K'], bc['V']
            # h' = LN2(a1 + mf (gelu(a1 W1 + b1) W2 + b2))
            dX2, dg, dc = _ln_bwd(dh_, bc['xa2'] if mag else bc['xh2'], bc['rs2'], w['g2'], mag)
            G['g2'] += dg; G['c2'] += dc
            dF = dX2 * bc['mf']
            G['W2'] += G1.T @ dF; G['b2'] += dF.sum(axis=0)
            dZ = (dF @ w['W2'].T) * gelu_grad(bc['Z1'], mag)
            G['W1'] += a1.T @ dZ; G['b1'] += dZ.sum(axis=0)
            da1 = dZ @ w['W1'].T + dX2
            # a1 = LN1(hin + ma (A Wo + bo))
            dX1, dg, dc = _ln_bwd(da1, bc['xa1'] if mag else bc['xh1'], bc['rs1'], w['g1'], mag)
            G['g1'] += dg; G['c1'] += dc
            dO = dX1 * bc['ma']
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
                dP = dA[:, cs] @ Vm[:, cs].T
                D = (dA[:, cs] * Am[:, cs]).sum(axis=1, keepdims=True)
                dSk = Pk * (dP + D) if mag else Pk * (dP - D)
                dQ[:, cs] = sh * dSk @ Km[:, cs]
                dK[:, cs] = sh * dSk.T @ Qm[:, cs]
            dh_ = dX1.copy()
            for dX, Wn, bn in ((dQ, 'Wq', 'bq'), (dK, 'Wk', 'bk'), (dV, 'Wv', 'bv')):
                G[Wn] += hin.T @ dX; G[bn] += dX.sum(axis=0)
                dh_ += dX @ w[Wn].T
        # h0 = m0 LN0(E[x'] + Pe[t])
        c0 = c['c0']
        dX0, dg, dc = _ln_bwd(dh_ * c0['m0'], c0['xa'] if mag else c0['xh'], c0['rs'], pa['g0'], mag)
        g['g0'] += dg; g['c0'] += dc
        g['Pe'][:n] += dX0
        np.add.at(g['E'], c0['xs'], dX0)
    return loss, g


def train(th0, shape, n_heads, piece_list, epochs, batch_size, lr, seed, dropout):
    """the fit of parameters of shape (n_items, d, n_blocks, max_len): per epoch (order, masks), mini-batches of batch_size pieces in
    the order, one Adam step each.  Returns (theta, per-step losses)"""
    th = np.asarray(th0, dtype=np.float64)
    m, v = np.zeros_like(th), np.zeros_like(th)
    losses, step = [], 0
    for order, masked in epochs:
        for b0 in range(0, len(order), batch_size):
            ks = order[b0:b0 + batch_size]
            loss, g = loss_and_grads(unpack(th, *shape), [piece_list[k] for k in ks], [masked[k] for k in ks], n_heads, seed, step, dropout,
                                     shape[3], batch_size)
            step += 1
            th, m, v = adam(th, pack(g), m, v, step, lr)
            losses.append(loss)
    return th, losses


def encode(p, prefix, n_heads, max_len):
    """eval-mode q of a prefix: the encoder over its last max_len - 1 inputs followed by the mask token, q at the mask"""
    x = list(prefix)[-(max_len - 1):]
    return piece_forward(p, x + [0], [False] * len(x) + [True], n_heads)[1][-1]


def encode_events(p, items, offsets, n_history, n_heads, max_len):
    """every counted event's q in evaluate's order"""
    out = []
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for pos in range(st + max(h, 1) - 1, en - 1):
            out.append(encode(p, items[st:pos + 1], n_heads, max_len))
    return np.array(out).reshape(-1, p['E'].shape[1])
