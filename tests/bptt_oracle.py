"""Float64 restatement of truncated backpropagation through time (DESIGN §3l) on top of the NumPy oracle
(oracle/gru4rec_oracle.py): the reference for the device's window path in tests/test_gpu_bptt.py and tests/test_host_bptt.py.

Both functions take an OracleGRU4Rec `m` and use only its forward(), make_masks() and apply_updates(); a window of one step is
m.train_step() exactly.  Test infrastructure only: the product path never imports it."""
import numpy as np

import gru4rec_oracle as orc


def backward_through_time(m, C, M, dH_new=None):
    """backward() of one step of a BPTT window, with the gradient `dH_new[i]` (lanes of the step) that the later steps of the
    window send back to the state H_new layer i leaves (None: the window's last step).  It reaches h through the reset
    (H_new = 0 where the lane's session ended, C['R']) and the hidden-dropout mask.  Returns (cost, G, dH): G as backward()
    gives it, dH[i] the gradient on the state that entered the step (lanes of the step)."""
    dt = m.dtype
    L, dyhat = orc.loss_and_grad(m.loss, C['yhat'], M, m.n_sample, m.bpreg, m.smoothing)
    cost = dt(L / dt(m.batch_size))
    dyhat = dyhat / dt(m.batch_size)
    do = orc.act_bwd(m.fact, C['o'], C['yhat'], dyhat)
    G = dict(dSy=do.T @ C['y_last'], dSBy=do.sum(axis=0).reshape(-1, 1))
    dy = do @ C['Sy']
    nl = len(m.layers)
    for key in ('dWx', 'dWh', 'dWrz', 'dBh', 'dvec'):
        G[key] = [None] * nl
    dH = [None] * nl
    first = nl - len(C['layers'])
    for li in range(len(C['layers']) - 1, -1, -1):
        lc = C['layers'][li]
        i = first + li
        mk = lc['mk']
        dh = dy * mk if mk is not None else dy
        if dH_new is not None:
            carry = np.where(np.asarray(C['R'], dtype=bool).reshape(-1, 1), dt(0), dH_new[i])
            dh = dh + (carry * mk if mk is not None else carry)
        H, r, z, ht = lc['H'], lc['r'], lc['z'], lc['ht']
        dz = dh * (ht - H)
        da_h = orc.act_bwd(m.hact, lc['a_h'], ht, dh * z)
        G['dWh'][i] = (H * r).T @ da_h
        dHr = da_h @ m.Wh[i].T
        da_r = dHr * H * r * (dt(1) - r)
        da_rz = np.hstack([da_r, dz * z * (dt(1) - z)])
        G['dWrz'][i] = H.T @ da_rz
        dvec = np.hstack([da_h, da_rz])
        G['dvec'][i] = dvec
        G['dBh'][i] = dvec.sum(axis=0)
        dH[i] = dh * (dt(1) - z) + dHr * r + da_rz @ m.Wrz[i].T
        if lc['inp'] is not None:
            G['dWx'][i] = lc['inp'].T @ dvec
            dy = dvec @ m.Wx[i].T
        else:
            G['dSx'] = dvec
            dy = None
    if C['mode'] in ('shared', 'embed'):
        G['dSx'] = dy * C['mk_e'] if C['mk_e'] is not None else dy
    return cost, G, dH


def train_window(m, steps):
    """One update for a window of consecutive mini-batches (truncated BPTT).  `steps`: dicts with X, Y, R and optionally
    slots, samples, masks, as train_step() takes them.  Every step runs forward with the parameters of the window's start
    from the state the previous step left; the objective is the sum of the step costs, its gradient flows back through the
    carried states (the state entering the window is a constant); the update is apply_updates() of one merged step: dense
    gradients summed, the row lists of the steps concatenated in step order.  Returns the step costs.  A window of one step
    is train_step()."""
    Cs = []
    for st in steps:
        X = np.asarray(st['X'], dtype=np.int64); Y = np.asarray(st['Y'], dtype=np.int64)
        M = len(X)
        masks = st.get('masks')
        if masks is None:
            masks = m.make_masks(M)
        slots = np.arange(M) if st.get('slots') is None else np.asarray(st['slots'])
        R = np.zeros(M, dtype=bool) if st.get('R') is None else np.asarray(st['R'], dtype=bool)
        yhat, C = m.forward(X, Y, M, R=R, samples=st.get('samples'), masks=masks, H=[h[slots] for h in m.H])
        C['R'], C['slots'] = R, slots
        for i in range(len(m.layers)):
            m.H[i][slots] = C['H_new'][i]
        m.step_count += 1
        Cs.append(C)
    T = len(Cs)
    costs, Gs, dH_new = [None] * T, [None] * T, None
    for t in range(T - 1, -1, -1):
        costs[t], Gs[t], dH = backward_through_time(m, Cs[t], len(Cs[t]['X']), dH_new)
        if t > 0:          # lane b of step t holds physical slot slots_t[b]; step t - 1 left that slot's state
            dH_new = []
            for i, L in enumerate(m.layers):
                full = np.zeros((m.batch_size, L), dtype=m.dtype)
                full[Cs[t]['slots']] = dH[i]
                dH_new.append(full[Cs[t - 1]['slots']])
    if T == 1:
        Cm, Gm = Cs[0], Gs[0]
    else:
        cat = lambda key: np.concatenate([C[key] for C in Cs])
        Cm = dict(mode=Cs[0]['mode'], X=cat('X'), Y=cat('Y'), Sx=cat('Sx'), Sy=cat('Sy'))
        Gm = dict(dSx=np.concatenate([G['dSx'] for G in Gs]), dSy=np.concatenate([G['dSy'] for G in Gs]),
                  dSBy=np.concatenate([G['dSBy'] for G in Gs]))
        if Cm['mode'] == 'shared':
            # one Wy list X_t | Y_t | samples_t per step, in step order: apply_updates stacks dSx over dSy, so the rows of
            # every step go to dSx in that order and dSy is empty
            Cm.update(Xc=cat('Xc'), S=cat('S'))
            Gm['dSx'] = np.concatenate([np.vstack([G['dSx'], G['dSy']]) for G in Gs])
            Gm['dSy'] = Gm['dSy'][:0]
        for key in ('dWx', 'dWh', 'dWrz', 'dBh'):
            Gm[key] = []
            for i in range(len(m.layers)):
                acc = Gs[0][key][i]
                for G in Gs[1:]:
                    acc = None if acc is None else acc + G[key][i]
                Gm[key].append(acc)
    m.apply_updates(Cm, Gm, None)
    m.last_cache, m.last_grads, m.last_window = Cs[-1], Gs[-1], (Cm, Gm)
    return np.array(costs, dtype=m.dtype)
