"""float64 NumPy restatement of STAMP as the device trains and ranks it (DESIGN §3v): the parameter layout and init, the samples
(SR-GNN's), the forward pass of one prefix and a hand-written backward pass of one mini-batch, with a magnitude pass for the
rounding bound, the eval-mode encoder and, from narm_oracle, Adam and the ranking of given q vectors.  Written independently of the
package's helpers, which the tests compare against it.  Test infrastructure: the device (g4r_stamp.cuh) is compared against it."""
import numpy as np

import narm_oracle

adam, rank_events, B1, B2, EPS = narm_oracle.adam, narm_oracle.rank_events, narm_oracle.B1, narm_oracle.B2, narm_oracle.EPS
BIASES = ('b_a', 'bs', 'bt')


def shapes(n_items, d):
    return [('E', (n_items, d)), ('W1', (d, d)), ('W2', (d, d)), ('W3', (d, d)), ('b_a', (d,)), ('w0', (d,)), ('Ws', (d, d)), ('bs', (d,)),
            ('Wt', (d, d)), ('bt', (d,))]


def n_params(n_items, d):
    return n_items * d + 5 * d * d + 4 * d


def unpack(flat, n_items, d):
    out, o = {}, 0
    for name, shp in shapes(n_items, d):
        n = int(np.prod(shp))
        out[name] = np.asarray(flat[o:o + n], dtype=np.float64).reshape(shp)
        o += n
    assert o == len(flat)
    return out


def pack(p):
    return np.concatenate([p[n].ravel() for n, _ in shapes(*p['E'].shape)])


def init(n_items, d, init_std, rs):
    """per block in the vector's order: a bias 0 without a draw, any other block from normal(0, init_std); float32"""
    return np.concatenate([np.zeros(int(np.prod(shp))) if name in BIASES else rs.normal(0.0, init_std, size=shp).ravel()
                           for name, shp in shapes(n_items, d)]).astype(np.float32)


def plan(n_items, d, init_std, n_samples, seed, n_epochs):
    rs = np.random.RandomState(seed)
    th = init(n_items, d, init_std, rs)
    return th, [rs.permutation(n_samples) for _ in range(n_epochs)]


def samples(sessions, max_len):
    """every (prefix of at most max_len inputs, next item) pair, sessions in order, then positions"""
    return [(list(s[max(0, j - max_len):j]), s[j]) for s in sessions for j in range(1, len(s))]


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def forward(p, x):
    """the encoder of one prefix x: (cache, q [d])"""
    X = p['E'][list(x)]
    n = len(x)
    ms = X.sum(axis=0) / n
    mt = X[-1]
    sg = _sig(X @ p['W1'] + (mt @ p['W2'] + ms @ p['W3']) + p['b_a'])
    a = sg @ p['w0']
    ma = a @ X
    hs = np.tanh(ma @ p['Ws'] + p['bs'])
    ht = np.tanh(mt @ p['Wt'] + p['bt'])
    return dict(x=list(x), X=X, ms=ms, mt=mt, sg=sg, a=a, ma=ma, hs=hs, ht=ht), hs * ht


def _magnitudes(p, c):
    """per forward value the scale of its rounding error: every product of magnitudes, every sum of them, a tanh or sigmoid's
    error carried from its argument"""
    A = {k: np.abs(v) for k, v in p.items()}
    X = np.abs(c['X'])
    ms, mt = X.mean(axis=0), X[-1]
    pre = X @ A['W1'] + mt @ A['W2'] + ms @ A['W3'] + A['b_a']
    sg = c['sg'] + c['sg'] * (1.0 - c['sg']) * pre
    a = sg @ A['w0']
    ma = a @ X
    hs = np.abs(c['hs']) + ma @ A['Ws'] + A['bs']
    ht = np.abs(c['ht']) + mt @ A['Wt'] + A['bt']
    return dict(X=X, ms=ms, mt=mt, sg=sg, a=a, ma=ma, hs=hs, ht=ht, q=hs * ht)


def loss_and_grads(p, batch, mag=False):
    """(mean loss, name -> gradient of the loss) of one mini-batch of (prefix, target) samples.  mag: the same backward over the
    magnitudes of every factor (every difference a sum): per element the scale of its rounding error"""
    E = p['E']
    d = E.shape[1]
    caches, Q = zip(*[forward(p, x) for x, _ in batch])
    Q = np.array(Q)
    Y = np.array([y for _, y in batch])
    B = len(batch)
    S = Q @ E.T
    m = S.max(axis=1, keepdims=True)
    ex = np.exp(S - m)
    pr = ex / ex.sum(axis=1, keepdims=True)
    loss = float(np.mean(np.log(ex.sum(axis=1)) + m[:, 0] - S[np.arange(B), Y]))
    pa = {k: np.abs(v) for k, v in p.items()} if mag else p
    if mag:
        cs = [_magnitudes(p, c) for c in caches]
        Qa = np.array([c['q'] for c in cs])
        Sm = Qa @ np.abs(E).T
        dS = (pr * (1.0 + Sm + Sm.max(axis=1, keepdims=True)) + (np.arange(E.shape[0])[None, :] == Y[:, None])) / B
    else:
        cs = caches
        dS = pr.copy()
        dS[np.arange(B), Y] -= 1.0
        dS /= B
        Qa = Q
    g = {k: np.zeros_like(v) for k, v in p.items()}
    dQ = dS @ pa['E']
    g['E'] += dS.T @ Qa
    for c0, c, dq in zip(caches, cs, dQ):
        X, ms, mt, sg, a, ma, hs, ht = (c[k] for k in ('X', 'ms', 'mt', 'sg', 'a', 'ma', 'hs', 'ht'))
        n = len(c0['x'])
        if mag:
            das = dq * ht * (1.0 + 2.0 * np.abs(c0['hs']) * hs)
            dat = dq * hs * (1.0 + 2.0 * np.abs(c0['ht']) * ht)
            sgd = c0['sg'] * (1.0 - c0['sg']) + sg
        else:
            das = dq * ht * (1.0 - hs * hs)
            dat = dq * hs * (1.0 - ht * ht)
            sgd = sg * (1.0 - sg)
        g['Ws'] += np.outer(ma, das)
        g['bs'] += das
        g['Wt'] += np.outer(mt, dat)
        g['bt'] += dat
        dma = pa['Ws'] @ das
        dmt = pa['Wt'] @ dat
        da = X @ dma
        dX = np.outer(a, dma)
        dsig = da[:, None] * pa['w0'][None, :] * sgd
        g['w0'] += sg.T @ da
        g['W1'] += X.T @ dsig
        dX += dsig @ pa['W1'].T
        dv = dsig.sum(axis=0)
        g['b_a'] += dv
        g['W2'] += np.outer(mt, dv)
        g['W3'] += np.outer(ms, dv)
        dmt = dmt + pa['W2'] @ dv
        dX += (pa['W3'] @ dv) / n
        dX[-1] += dmt
        np.add.at(g['E'], c0['x'], dX)
    return loss, g


def train(th0, n_items, d, sample_list, orders, batch_size, lr):
    """the fit: per epoch mini-batches of batch_size samples in the order, one Adam step each.  Returns (theta, per-step losses)"""
    th = np.asarray(th0, dtype=np.float64)
    m, v = np.zeros_like(th), np.zeros_like(th)
    losses, t = [], 0
    for order in orders:
        for b0 in range(0, len(order), batch_size):
            loss, g = loss_and_grads(unpack(th, n_items, d), [sample_list[k] for k in order[b0:b0 + batch_size]])
            t += 1
            th, m, v = adam(th, pack(g), m, v, t, lr)
            losses.append(loss)
    return th, losses


def encode(p, prefix, max_len):
    """eval-mode q of a prefix: its last max_len inputs"""
    return forward(p, list(prefix)[-max_len:])[1]


def encode_events(p, items, offsets, n_history, max_len):
    """every counted event's q in evaluate's order"""
    out = []
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for pos in range(st + max(h, 1) - 1, en - 1):
            out.append(encode(p, items[st:pos + 1], max_len))
    return np.array(out).reshape(-1, p['E'].shape[1])
