"""Float64 restatement of full-softmax training (full_softmax=True, DESIGN §3n) on top of the NumPy oracle
(oracle/gru4rec_oracle.py): the reference for the device's full-catalogue step in tests/test_gpu_full_softmax.py and
tests/test_host_full_softmax.py.

The score columns of a step are the catalogue 0..I-1, each item once; the target of lane b is column Y[b].  forward() already
takes an arbitrary column list; the loss, its gradient and the backward here take the target column instead of the diagonal.
The update is apply_updates() with C['Y'] = arange(I).  logq corrects a sampled softmax and is not applied.  Also the
per-element float64 bound of one step (full_step_reference, row_update_bounds) that tests/test_gpu_full_softmax_rows.py holds
the device to and tests/test_host_full_softmax_rows.py checks.  Test infrastructure only: the product path never imports it."""
import copy

import numpy as np

import gru4rec_oracle as orc


def loss_and_grad_target(loss, yhat, Y):
    """(loss sum, dL/dyhat) of the cross-entropy losses with lane b's target in column Y[b] (gru4rec.py:225-236)"""
    dt = yhat.dtype.type
    ar = np.arange(yhat.shape[0])
    t = yhat[ar, Y]
    g = np.zeros_like(yhat)
    if loss == 'cross-entropy':
        g[ar, Y] = -dt(1) / (t + dt(orc.EPS_LOG))
        return dt(np.sum(-np.log(t + dt(orc.EPS_LOG)))), g
    if loss == 'xe_logit':
        g[ar, Y] = dt(1)
        return dt(np.sum(t)), g
    raise NotImplementedError('full softmax: only the cross-entropy losses')


def backward_full(m, C, M, Y):
    """backward() of one full-catalogue step: cost and gradients as m.backward() returns them (dSy / dSBy over every item)"""
    dt = m.dtype
    L, dyhat = loss_and_grad_target(m.loss, C['yhat'], np.asarray(Y))
    cost = dt(L / dt(m.batch_size))
    do = orc.act_bwd(m.fact, C['o'], C['yhat'], dyhat / dt(m.batch_size))
    G = dict(dSy=do.T @ C['y_last'], dSBy=do.sum(axis=0).reshape(-1, 1), do=do)
    gru_backward(m, C, do @ C['Sy'], G)
    return cost, G


def gru_backward(m, C, dy, G):
    """the GRU backward of backward() from dL/dy of the last layer: fills dWx / dWh / dWrz / dBh / dvec of every layer and dSx"""
    dt = m.dtype
    nl = len(m.layers)
    for key in ('dWx', 'dWh', 'dWrz', 'dBh', 'dvec'):
        G[key] = [None] * nl
    G['dy_last'] = dy
    first = nl - len(C['layers'])
    for li in range(len(C['layers']) - 1, -1, -1):
        lc = C['layers'][li]
        i = first + li
        dh = dy * lc['mk'] if lc['mk'] is not None else dy
        H, r, z, ht = lc['H'], lc['r'], lc['z'], lc['ht']
        dz = dh * (ht - H)
        da_h = orc.act_bwd(m.hact, lc['a_h'], ht, dh * z)
        G['dWh'][i] = (H * r).T @ da_h
        dHr = da_h @ m.Wh[i].T
        da_rz = np.hstack([dHr * H * r * (dt(1) - r), dz * z * (dt(1) - z)])
        G['dWrz'][i] = H.T @ da_rz
        dvec = np.hstack([da_h, da_rz])
        G['dvec'][i] = dvec
        G['dBh'][i] = dvec.sum(axis=0)
        if lc['inp'] is not None:
            G['dWx'][i] = lc['inp'].T @ dvec
            dy = dvec @ m.Wx[i].T
        else:
            G['dSx'] = dvec
            dy = None
    if C['mode'] in ('shared', 'embed'):
        G['dSx'] = dy * C['mk_e'] if C['mk_e'] is not None else dy
    return G


def forward_full(m, X, M, R=None, masks=None, H=None):
    """forward() with the catalogue as the column list and without the logQ correction"""
    logq, m.logq = m.logq, 0.0
    try:
        return m.forward(np.asarray(X, dtype=np.int64), np.arange(m.n_items), M, R=R, samples=None, masks=masks, H=H)
    finally:
        m.logq = logq


def train_step_full(m, X, Y, R, slots=None, masks=None):
    """One full-catalogue training step: the schedule, slots, resets and dropout masks of train_step(), every item a score
    column, the update apply_updates() with C['Y'] = arange(I).  Returns the cost."""
    X = np.asarray(X, dtype=np.int64); Y = np.asarray(Y, dtype=np.int64)
    M = len(X)
    if masks is None:
        masks = m.make_masks(M)
    slots = np.arange(M) if slots is None else np.asarray(slots)
    _, C = forward_full(m, X, M, R=R, masks=masks, H=[h[slots] for h in m.H])
    cost, G = backward_full(m, C, M, Y)
    m.apply_updates(C, G, M)
    for i in range(len(m.layers)):
        m.H[i][slots] = C['H_new'][i]
    m.step_count += 1
    m.last_cache, m.last_grads = C, G
    return cost


# ---------------- per-element float64 bound of one full-catalogue step ----------------
# What a correct float32 step may differ from float64 by, element by element, so that every Wy / By row is held at its own scale
# (the rows of non-target items are 1e-3 .. 1e-4 of the target rows, and a bar scaled by the table's max does not see them).
# Built in float64 from the final-layer output y the step's row product used (the device's own, so no hidden-state term):
#   scores    |ds_bj| <= 2^-19 (|y_b|.|Wy_j| + |By_j|)            (fp32 tiles and 3xTF32 alike, as the scoring tests)
#   p         relative: ds_bj + sum_j p_bj ds_bj (the log-sum-exp) + 2^-17 (the merge tree of max / sum-exp)
#             + 2u |o_bj - m_b| (the argument of exp) + 4u (exp, divide); absolute floor 2^-126 (float32 underflow)
#   dL/do     fac_b (p_bj - [j = Y_b]) / B with fac_b = p_t / (p_t + EPS_LOG) (1 for xe_logit): the errors of p_bj, of fac_b
#             and 4u of the products; the reference itself is the chained form -1/(t + EPS_LOG) through act_bwd
#   rows      dWy_jk: sum_b e_bj |y_bk| + gamma_M sum_b |do_bj| |y_bk|; dBy_j likewise without y
#   dL/dy     sum_j e_bj |Wy_j| + gamma_n sum_j |do_bj| |Wy_j| (n: the summands of one element of k_full_dy's K split)
#   dvec, dSx the dL/dy bound through the GRU backward with every factor taken by magnitude, plus kappa u times the lane's
#             largest backward magnitude (float32 rounding of the backward and of the forward values it reads, per lane)
#   updates   the oracle's apply_updates evaluated from the same state at g + e, g - e and g - clip(g, -e, e): the largest
#             deviation from the update at g (no optimizer derived by hand), plus 8u of the update for the optimizer's own float32
#             arithmetic; the caller adds one fp32 rounding of the stored result per applied update
U32 = 2.0 ** -24                # float32 unit roundoff
SCORE_ULP = 2.0 ** -19          # score error per unit of |y|.|Wy| + |By|
LSE_ULP = 2.0 ** -17            # log-sum-exp error of the tile merges, besides the scores'
F32_TINY = 2.0 ** -126          # float32's smallest normal number: the absolute floor of p and dL/do


def gamma(n):
    """the worst-case relative error of an n-term float32 sum (Higham's gamma_n)"""
    return n * U32 / (1.0 - n * U32)


def dy_terms(n_items, B, L, n_sm=132):
    """summands of one dL/dy element: k_full_dy sums one K split of kchunk items in order, k_b1 the ks splits in order
    (g4r_lib.cu full_shape: 32 x 32 output tiles, 128-item slabs, about two CTAs per SM)"""
    mn = -(-B // 32) * -(-L // 32)
    slabs = -(-n_items // 128)
    ks = max(1, min(slabs, -(-2 * n_sm // mn)))
    kchunk = -(-slabs // ks) * 128
    return min(n_items, kchunk) + -(-n_items // kchunk)


def _probabilities(m, yhat):
    """softmax(o) from the final activation: softmax itself, or softmax_logit's -log softmax"""
    return yhat if m.fact[0] == 'softmax' else np.exp(-yhat)


def full_step_reference(m, X, Y, R, y, n_sm=132):
    """Float64 reference and per-element bound of one full step of m (its state before the step), the row product taken with
    the final-layer output y [M x L] the step used.  Returns (C, G, E): the forward cache of m, the gradients (dSy, dSBy, do,
    dy_last, dvec, dSx and the dense ones) from y, and the bounds of their errors (dSy, dSBy, e = dL/do, dy, dvec, dSx)."""
    X = np.asarray(X, dtype=np.int64); Y = np.asarray(Y, dtype=np.int64)
    M = len(X)
    y = np.asarray(y, np.float64)
    _, C = forward_full(m, X, M, R=R, masks=m.make_masks(M), H=[h[:M] for h in m.H])
    By = m.By.reshape(-1)
    o = y @ m.Wy.T + By
    yhat = orc.act_fwd(m.fact, o)
    _, dyhat = loss_and_grad_target(m.loss, yhat, Y)
    do = orc.act_bwd(m.fact, o, yhat, dyhat / m.batch_size)
    G = dict(dSy=do.T @ y, dSBy=do.sum(axis=0).reshape(-1, 1), do=do)
    gru_backward(m, C, do @ m.Wy, G)
    # scores, probabilities, dL/do
    ar = np.arange(M)
    ay, aW = np.abs(y), np.abs(m.Wy)
    ds = SCORE_ULP * (ay @ aW.T + np.abs(By))
    p = _probabilities(m, yhat)
    rel = ds + ((p * ds).sum(axis=1) + LSE_ULP)[:, None] + 2 * U32 * (o.max(axis=1, keepdims=True) - o) + 4 * U32
    dp = p * rel + F32_TINY
    t = np.zeros_like(p); t[ar, Y] = 1.0
    if m.loss == 'cross-entropy':
        pt = p[ar, Y]
        fac = pt / (pt + orc.EPS_LOG)
        dfac = dp[ar, Y] * orc.EPS_LOG / (pt + orc.EPS_LOG) ** 2 + 2 * U32 * fac
    else:
        fac, dfac = np.ones(M), np.zeros(M)
    e = (fac[:, None] * dp + np.abs(p - t) * (dfac[:, None] + 4 * U32 * fac[:, None])) / m.batch_size + F32_TINY
    ado = np.abs(do)
    E = dict(e=e, dSy=e.T @ ay + gamma(M) * (ado.T @ ay), dSBy=(e.sum(axis=0) + gamma(M) * ado.sum(axis=0)).reshape(-1, 1))
    n = dy_terms(m.n_items, m.batch_size, m.layers[-1], n_sm)
    E['dy'] = e @ aW + gamma(n) * (ado @ aW)
    E['dvec'], E['dSx'] = _gru_backward_bound(m, C, E['dy'], ado @ aW)
    return C, G, E


def _gru_backward_bound(m, C, e_dy, a_dy):
    """bounds of dvec of every layer and of dSx: e_dy through gru_backward with every factor by magnitude, plus kappa u times
    the largest magnitude of the lane's backward (a_dy: the magnitude of dL/dy, sum_j |do_bj| |Wy_j|)"""
    nl = len(m.layers)
    out = [None] * nl
    first = nl - len(C['layers'])
    e_sx = None
    for li in range(len(C['layers']) - 1, -1, -1):
        lc = C['layers'][li]
        i = first + li
        mk = np.abs(lc['mk']) if lc['mk'] is not None else 1.0
        H, r, z, ht = np.abs(lc['H']), lc['r'], lc['z'], lc['ht']
        dact = np.abs(orc.act_bwd(m.hact, lc['a_h'], ht, np.ones_like(ht)))
        aWh, Lw = np.abs(m.Wh[i]), m.layers[i]
        inp = lc['inp'].shape[1] if lc['inp'] is not None else 0       # no-embedding mode: layer 0's input is a row gather
        kappa = 8 * (inp + 3 * Lw) + 64

        def chain(d, dz_abs):
            dh = d * mk
            da_h = dh * z * dact
            return np.hstack([da_h, (da_h @ aWh.T) * H * r * (1 - r), dh * dz_abs * z * (1 - z)])
        a_vec = chain(a_dy, np.abs(ht) + H)
        e_vec = chain(e_dy, np.abs(ht - lc['H'])) + kappa * U32 * a_vec.max(axis=1, keepdims=True)
        out[i] = e_vec
        if lc['inp'] is not None:
            aWx = np.abs(m.Wx[i])
            e_dy = e_vec @ aWx.T + gamma(3 * Lw) * (a_vec @ aWx.T)
            a_dy = a_vec @ aWx.T
        else:
            e_sx = e_vec
    if C['mode'] in ('shared', 'embed'):
        e_sx = e_dy * (np.abs(C['mk_e']) if C['mk_e'] is not None else 1.0)
    return out, e_sx


def _apply_rows(m, lo, hi, xin, gx, gy, gby):
    """apply_updates() of m restricted to Wy / By rows lo..hi-1: the input occurrences xin first (shared mode, gradients gx), then
    every item's score column (gy, gby), from m's state, which stays unchanged.  {name: (before, after)} of the rows and state."""
    sub = copy.copy(m)
    sub.layers = []                             # no dense parameter
    n = hi - lo
    sub.Wy, sub.By = m.Wy[lo:hi].copy(), m.By[lo:hi].copy()
    sub.opt = {k: v[lo:hi].copy() for k, v in m.opt.items() if k[0] in ('Wy', 'By')}
    before = dict(Wy=m.Wy[lo:hi], By=m.By[lo:hi], **{'%s.%s' % k: m.opt[k][lo:hi] for k in sub.opt})
    Xc = np.concatenate([np.asarray(xin, np.int64) - lo, np.arange(n)])
    C = dict(mode='shared', X=None, Y=np.arange(n), Xc=Xc, S=sub.Wy[Xc])
    sub.apply_updates(C, dict(dSx=gx, dSy=gy, dSBy=gby), 0)
    after = dict(Wy=sub.Wy, By=sub.By, **{'%s.%s' % k: v for k, v in sub.opt.items()})
    return {k: (before.get(k, np.zeros_like(v)), v) for k, v in after.items()}


def row_update_bounds(m, C, G, E, chunk=8192):
    """The reference update of every Wy / By row and of its optimizer state, and its allowance, in chunks of rows: yields
    (lo, hi, counts, {name: (before, reference after, allowance)}); counts: the occurrences of each row in the step's Wy list
    (the shared-mode inputs, then the column).  m holds the state before the step and is not changed."""
    I, L = m.Wy.shape
    shared = C['mode'] == 'shared'
    xin = np.asarray(C['X'], np.int64) if shared else np.zeros(0, np.int64)
    gx = G['dSx'] if shared else np.zeros((0, L))
    ex = E['dSx'] if shared else np.zeros((0, L))
    for lo in range(0, I, chunk):
        hi = min(I, lo + chunk)
        sel = (xin >= lo) & (xin < hi)
        g = (gx[sel], G['dSy'][lo:hi], G['dSBy'][lo:hi])
        e = (ex[sel], E['dSy'][lo:hi], E['dSBy'][lo:hi])
        ref = _apply_rows(m, lo, hi, xin[sel], *g)
        allow = {k: np.zeros_like(v[1]) for k, v in ref.items()}
        for gv in ([a + b for a, b in zip(g, e)], [a - b for a, b in zip(g, e)], [a - np.clip(a, -b, b) for a, b in zip(g, e)]):
            for k, (_, v) in _apply_rows(m, lo, hi, xin[sel], *gv).items():
                allow[k] = np.maximum(allow[k], np.abs(v - ref[k][1]))
        counts = 1 + np.bincount(xin[sel] - lo, minlength=hi - lo)
        # plus the optimizer's own float32 arithmetic (g^2, acc + g^2, sqrt, divide, lr and momentum products): 8u of the update
        yield lo, hi, counts, {k: (b, a, allow[k] + 8 * U32 * np.abs(a - b)) for k, (b, a) in ref.items()}


def bound_ratio(dev, ref, allow):
    """max |dev - ref| / allow over the elements (0 where they agree exactly; inf for a non-finite element or an error where the
    allowance is 0): a value <= 1 meets the bound"""
    dev = np.asarray(dev, np.float64); ref = np.asarray(ref, np.float64).reshape(dev.shape)
    if not (np.isfinite(dev).all() and np.isfinite(ref).all()):
        return np.inf
    err = np.abs(dev - ref)
    allow = np.broadcast_to(np.asarray(allow, np.float64), err.shape)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.where(err > 0, err / allow, 0.0)
    return float(r.max()) if r.size else 0.0
