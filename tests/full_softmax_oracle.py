"""Float64 restatement of full-softmax training (full_softmax=True, DESIGN §3n) on top of the NumPy oracle
(oracle/gru4rec_oracle.py): the reference for the device's full-catalogue step in tests/test_gpu_full_softmax.py and
tests/test_host_full_softmax.py.

The score columns of a step are the catalogue 0..I-1, each item once; the target of lane b is column Y[b].  forward() already
takes an arbitrary column list; the loss, its gradient and the backward here take the target column instead of the diagonal.
The update is apply_updates() with C['Y'] = arange(I).  logq corrects a sampled softmax and is not applied.  Test
infrastructure only: the product path never imports it."""
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
    dy = do @ C['Sy']
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
    return cost, G


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
