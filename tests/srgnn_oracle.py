"""float64 NumPy restatement of SR-GNN as the device trains and ranks it (DESIGN §3u): the parameter layout and init, the samples,
each prefix's graph (dense adjacency), the forward pass of one sample and a hand-written backward pass of one mini-batch, with a
magnitude pass for the rounding bound, coupled L2 before Adam, the eval-mode encoder and, from narm_oracle, Adam and the ranking
of given s_h vectors.  Written independently of the package's helpers, which the tests compare against it.  Test
infrastructure: the device (g4r_srgnn.cuh) is compared against it."""
import numpy as np

import narm_oracle

adam, rank_events, B1, B2, EPS = narm_oracle.adam, narm_oracle.rank_events, narm_oracle.B1, narm_oracle.B2, narm_oracle.EPS


def shapes(n_items, d):
    return [('E', (n_items, d)), ('W_in', (d, d)), ('W_out', (d, d)), ('b_in', (d,)), ('b_out', (d,)), ('b_iah', (d,)), ('b_oah', (d,)),
            ('W_ih', (2 * d, 3 * d)), ('b_ih', (3 * d,)), ('W_hh', (d, 3 * d)), ('b_hh', (3 * d,)), ('W1', (d, d)), ('W2', (d, d)),
            ('b1', (d,)), ('b2', (d,)), ('q', (d,)), ('W3', (2 * d, d)), ('b3', (d,))]


def n_params(n_items, d):
    return n_items * d + 15 * d * d + 14 * d


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


def init(n_items, d, rs):
    """every entry, in the vector's order, from uniform(-1 / sqrt(d), 1 / sqrt(d)); float32"""
    s = 1.0 / np.sqrt(d)
    return rs.uniform(-s, s, size=n_params(n_items, d)).astype(np.float32)


def plan(n_items, d, n_samples, seed, n_epochs):
    rs = np.random.RandomState(seed)
    th = init(n_items, d, rs)
    return th, [rs.permutation(n_samples) for _ in range(n_epochs)]


def samples(sessions, max_len):
    """every (prefix of at most max_len inputs, next item) pair, sessions in order, then positions"""
    return [(list(s[max(0, j - max_len):j]), s[j]) for s in sessions for j in range(1, len(s))]


def graph(x):
    """(nodes ascending, alias per position, A_in [K, K], A_out [K, K]): edges u -> v per consecutive pair, each once"""
    nodes = sorted(set(x))
    alias = [nodes.index(i) for i in x]
    K = len(nodes)
    adj = np.zeros((K, K))
    for t in range(len(x) - 1):
        adj[alias[t], alias[t + 1]] = 1.0
    indeg, outdeg = adj.sum(axis=0), adj.sum(axis=1)
    a_in = np.where(indeg[:, None] > 0, adj.T / np.maximum(indeg, 1)[:, None], 0.0)
    a_out = np.where(outdeg[:, None] > 0, adj / np.maximum(outdeg, 1)[:, None], 0.0)
    return nodes, alias, a_in, a_out


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def forward(p, x, step):
    """the encoder of one prefix x: (cache, s_h [d])"""
    d = p['E'].shape[1]
    nodes, alias, a_in, a_out = graph(x)
    H = p['E'][nodes]
    steps = []
    for _ in range(step):
        A = np.concatenate([a_in @ (H @ p['W_in'] + p['b_in']) + p['b_iah'], a_out @ (H @ p['W_out'] + p['b_out']) + p['b_oah']], axis=1)
        gi = A @ p['W_ih'] + p['b_ih']
        gh = H @ p['W_hh'] + p['b_hh']
        r = _sig(gi[:, :d] + gh[:, :d])
        z = _sig(gi[:, d:2 * d] + gh[:, d:2 * d])
        n = np.tanh(gi[:, 2 * d:] + r * gh[:, 2 * d:])
        steps.append(dict(H=H, A=A, r=r, z=z, n=n, ghn=gh[:, 2 * d:]))
        H = n + z * (H - n)
    hs = H[alias]
    sl = hs[-1]
    u = _sig(sl @ p['W1'] + p['b1'] + hs @ p['W2'] + p['b2'])
    alpha = u @ p['q']
    cat = np.concatenate([alpha @ hs, sl])
    sh = cat @ p['W3'] + p['b3']
    return dict(nodes=nodes, alias=alias, a_in=a_in, a_out=a_out, steps=steps, hs=hs, u=u, alpha=alpha, cat=cat), sh


def loss_and_grads(p, batch, step, mag=False):
    """(mean loss, name -> gradient of the loss) of one mini-batch of (prefix, target) samples.  mag: the same backward over the
    magnitudes of every factor (every difference a sum): per element the scale of its rounding error"""
    E = p['E']
    d = E.shape[1]
    caches, SH = zip(*[forward(p, x, step) for x, _ in batch])
    SH = np.array(SH)
    Y = np.array([y for _, y in batch])
    B = len(batch)
    S = SH @ E.T
    m = S.max(axis=1, keepdims=True)
    ex = np.exp(S - m)
    pr = ex / ex.sum(axis=1, keepdims=True)
    loss = float(np.mean(np.log(ex.sum(axis=1)) + m[:, 0] - S[np.arange(B), Y]))
    A_ = np.abs if mag else (lambda a: a)
    pa = {k: A_(v) for k, v in p.items()}
    if mag:
        SHa = np.abs(np.array([c['cat'] for c in caches])) @ pa['W3'] + pa['b3']
        Sm = SHa @ np.abs(E).T
        dS = (pr * (1.0 + Sm + Sm.max(axis=1, keepdims=True)) + (np.arange(E.shape[0])[None, :] == Y[:, None])) / B
    else:
        dS = pr.copy()
        dS[np.arange(B), Y] -= 1.0
        dS /= B
        SHa = SH
    g = {k: np.zeros_like(v) for k, v in p.items()}
    dSH = dS @ pa['E']
    g['E'] += dS.T @ SHa
    for c, dsh in zip(caches, dSH):
        hs, u, alpha, cat = A_(c['hs']), c['u'], A_(c['alpha']), A_(c['cat'])
        g['W3'] += np.outer(cat, dsh)
        g['b3'] += dsh
        dcat = pa['W3'] @ dsh
        dsg, dsl = dcat[:d], dcat[d:].copy()
        da = hs @ dsg
        dhs = np.outer(alpha, dsg)
        dpre = da[:, None] * pa['q'][None, :] * u * (1.0 - u)
        g['q'] += u.T @ da
        g['W2'] += hs.T @ dpre
        g['b2'] += dpre.sum(axis=0)
        dhs += dpre @ pa['W2'].T
        dq1 = dpre.sum(axis=0)
        g['W1'] += np.outer(hs[-1], dq1)
        g['b1'] += dq1
        dsl += pa['W1'] @ dq1
        dhs[-1] += dsl
        dH = np.zeros((len(c['nodes']), d))
        np.add.at(dH, c['alias'], dhs)
        for s in reversed(c['steps']):
            H, A, r, z, n, ghn = A_(s['H']), A_(s['A']), s['r'], s['z'], s['n'], A_(s['ghn'])
            dz = dH * (H + np.abs(n) if mag else H - n)
            dn = dH * (1.0 - z)
            dpn = dn * (1.0 - n * n)
            dpr = dpn * ghn * r * (1.0 - r)
            dpz = dz * z * (1.0 - z)
            dgi = np.concatenate([dpr, dpz, dpn], axis=1)
            dgh = np.concatenate([dpr, dpz, dpn * r], axis=1)
            g['W_ih'] += A.T @ dgi
            g['b_ih'] += dgi.sum(axis=0)
            g['W_hh'] += H.T @ dgh
            g['b_hh'] += dgh.sum(axis=0)
            dA = dgi @ pa['W_ih'].T
            g['b_iah'] += dA[:, :d].sum(axis=0)
            g['b_oah'] += dA[:, d:].sum(axis=0)
            dXI, dXO = c['a_in'].T @ dA[:, :d], c['a_out'].T @ dA[:, d:]
            g['W_in'] += H.T @ dXI
            g['b_in'] += dXI.sum(axis=0)
            g['W_out'] += H.T @ dXO
            g['b_out'] += dXO.sum(axis=0)
            dH = dH * z + dgh @ pa['W_hh'].T + dXI @ pa['W_in'].T + dXO @ pa['W_out'].T
        g['E'][c['nodes']] += dH
    return loss, g


def train(th0, n_items, d, step, sample_list, orders, batch_size, lrs, l2):
    """the fit: per epoch (learning rate lrs[e]), mini-batches of batch_size samples in the order, one Adam step each on
    gradient + l2 theta.  Returns (theta, per-step losses)"""
    th = np.asarray(th0, dtype=np.float64)
    m, v = np.zeros_like(th), np.zeros_like(th)
    losses, t = [], 0
    for order, lr in zip(orders, lrs):
        for b0 in range(0, len(order), batch_size):
            loss, g = loss_and_grads(unpack(th, n_items, d), [sample_list[k] for k in order[b0:b0 + batch_size]], step)
            t += 1
            th, m, v = adam(th, pack(g) + l2 * th, m, v, t, lr)
            losses.append(loss)
    return th, losses


def encode(p, prefix, step, max_len):
    """eval-mode s_h of a prefix: the graph of its last max_len inputs"""
    return forward(p, list(prefix)[-max_len:], step)[1]


def encode_events(p, items, offsets, n_history, step, max_len):
    """every counted event's s_h in evaluate's order"""
    out = []
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for pos in range(st + max(h, 1) - 1, en - 1):
            out.append(encode(p, items[st:pos + 1], step, max_len))
    return np.array(out).reshape(-1, p['E'].shape[1])
