"""Shared helpers for the -m gpu parity tests: build an Engine + an oracle with identical state."""
import numpy as np
import gru4rec_oracle as orc
from gru4rec_b200 import _lib


make_cfg = _lib.make_config


def param_names(m):
    names = []
    for i in range(len(m.layers)):
        names += ['Wx%d' % i, 'Wh%d' % i, 'Wrz%d' % i, 'Bh%d' % i]
    names += ['Wy', 'By']
    if m.E is not None:
        names.append('E')
    return names


def oracle_param(m, name):
    if name in ('Wy', 'By', 'E'):
        return getattr(m, name)
    kind, i = name.rstrip('0123456789'), int(name[len(name.rstrip('0123456789')):])
    return getattr(m, kind)[i]


def push_weights(eng, m):
    for name in param_names(m):
        eng.set(name, oracle_param(m, name))
    for i in range(len(m.layers)):
        eng.set('H%d' % i, m.H[i])


def compare_weights(eng, m, rtol, atol, what=''):
    for name in param_names(m):
        dev = eng.get(name)
        ref = np.asarray(oracle_param(m, name)).reshape(dev.shape)
        np.testing.assert_allclose(dev, ref, rtol=rtol, atol=atol, err_msg='%s %s' % (what, name))


def compare_opt_state(eng, m, rtol, atol):
    for (name, slot), val in m.opt.items():
        dev = eng.get('%s.%s' % (name, slot))
        np.testing.assert_allclose(dev, np.asarray(val).reshape(dev.shape), rtol=rtol, atol=atol, err_msg='%s.%s' % (name, slot))


def make_pair(n_items, mk, n_store_rows=0, seed=0, eval_lanes=0, randomize_state=True, step_mode=0):
    """Engine + oracle with identical random weights, hidden state, and (optionally) sample store."""
    rs = np.random.RandomState(seed)
    okw = dict(mk)
    m = orc.OracleGRU4Rec(**okw)
    m.init(n_items)
    if randomize_state:
        for h in m.H:
            h[:] = rs.randn(*h.shape).astype(np.float32) * 0.5
        m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
        for b in m.Bh:
            b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    S = mk.get('n_sample', 2048)
    cfg = make_cfg(n_items, mk, sample_store=n_store_rows * S, eval_lanes=eval_lanes, step_mode=step_mode)
    eng = _lib.Engine(cfg)
    push_weights(eng, m)
    store = None
    if n_store_rows > 1 and S > 0:
        store = rs.randint(0, n_items, size=(n_store_rows, S)).astype(np.int64)
        # make duplicates likely (inside samples and against targets)
        store[:, :max(1, S // 8)] = rs.randint(0, max(2, n_items // 10), size=(n_store_rows, max(1, S // 8)))
        eng.set_sample_store(store)
    if mk.get('logq', 0):
        P0 = rs.randint(1, 50, size=n_items).astype(np.float32)
        m.P0 = P0
        eng.set_logq_support(P0)
    return eng, m, store, rs


def oracle_multi_step(m, Hs, inputs):
    """One synchronous data-parallel step of R ranks on the oracle: every rank's forward/backward with the shared
    weights and its own hidden state, then ONE merged update -- row gradients of all ranks concatenated in
    (rank, position) order, dense gradients summed (the stated multi-GPU semantics, gru4rec_b200/csrc/g4r_multi.cuh)."""
    Cs, Gs, costs = [], [], []
    base_seed = m.dropout_seed
    for r, inp in enumerate(inputs):
        M = len(inp['X'])
        m.dropout_seed = (base_seed + r * 0x9E3779B1) & 0xffffffff      # independent dropout masks per rank (g4r_lib.cu layout())
        masks = m.make_masks(M)
        m.dropout_seed = base_seed
        Hr = [h[inp['slots']] for h in Hs[r]]
        X = np.asarray(inp['X'], dtype=np.int64); Y = np.asarray(inp['Y'], dtype=np.int64)
        yhat, C = m.forward(X, Y, M, R=inp['R'], samples=inp.get('samples'), masks=masks, H=Hr)
        cost, G = m.backward(C, M)
        Cs.append(C); Gs.append(G); costs.append(cost)
    nl = len(m.layers)
    Cm = dict(mode=Cs[0]['mode'], X=np.concatenate([C['X'] for C in Cs]), Y=np.concatenate([C['Y'] for C in Cs]),
              Sx=np.vstack([C['Sx'] for C in Cs]), Sy=np.vstack([C['Sy'] for C in Cs]))
    Gm = dict(dSx=np.vstack([G['dSx'] for G in Gs]), dSy=np.vstack([G['dSy'] for G in Gs]), dSBy=np.vstack([G['dSBy'] for G in Gs]))
    for key in ('dWx', 'dWh', 'dWrz', 'dBh'):
        Gm[key] = [None if Gs[0][key][i] is None else sum(G[key][i] for G in Gs) for i in range(nl)]
    m.apply_updates(Cm, Gm, sum(len(i['X']) for i in inputs))
    for r, inp in enumerate(inputs):
        for i in range(nl):
            Hs[r][i][inp['slots']] = Cs[r]['H_new'][i]
    m.step_count += 1
    return costs


# ---------------- product-level comparison with a float64 oracle ----------------
# The tensor-core kernels compute every fp32 product as 3xTF32 (~2^-21 relative per product); a product that lost one of its
# cross terms is 2xTF32 / 1xTF32 (~2^-11).  The bar sits between the two: per tensor max |dev - ref| <= F64_REL * max |ref|, and
# |dev - ref| <= F64_RTOL * |ref| on every element above 1 % of max |ref|.  The gradient chain (dL/dh sums 2048 score columns whose
# loss gradients cancel) needs more room than one product: a float32 run of the oracle itself is up to 9.1e-6 / 2.3e-4 away from
# float64 on the cases of TC_CASES, so the bar is 4x that.  The device and a 2xTF32 product, measured against it: see
# tests/test_gpu_tcstep.py::test_tc_step_products_match_float64.
F64_REL = 4e-5
F64_RTOL = 1e-3


def f64_errors(dev, ref, extra_atol=0.0):
    """(max |dev - ref| / max |ref|, max relative error over the elements above 1 % of max |ref|); `extra_atol` (scalar or per
    element) is an allowance subtracted from |dev - ref| first.  A non-finite element on either side gives (inf, inf)."""
    dev = np.asarray(dev, np.float64)
    ref = np.asarray(ref, np.float64).reshape(dev.shape)
    if not (np.isfinite(dev).all() and np.isfinite(ref).all()):
        return np.inf, np.inf
    scale = max(float(np.abs(ref).max()) if ref.size else 0.0, 1e-30)
    err = np.maximum(np.abs(dev - ref) - extra_atol, 0.0)
    big = np.abs(ref) > 0.01 * scale
    rel = float((err[big] / np.abs(ref[big])).max()) if big.any() else 0.0
    return float(err.max()) / scale if err.size else 0.0, rel


def assert_f64_close(dev, ref, what, extra_atol=0.0):
    a, r = f64_errors(dev, ref, extra_atol)
    assert a <= F64_REL and r <= F64_RTOL, '%s: max err / max |ref| = %.3g (bar %g), max relative err above 1%% of max = %.3g (bar %g)' % (
        what, a, F64_REL, r, F64_RTOL)


OPT_SLOTS = {None: (), 'adagrad': ('acc',), 'rmsprop': ('acc',), 'adadelta': ('acc', 'upd'), 'adam': ('acc', 'meang', 'countt')}


def opt_slots(m):
    """optimizer state tensors of every parameter, as g4r_lib.cu layout() registers them ('<param>.<slot>')"""
    return OPT_SLOTS[m.adapt] + (('vel',) if m.momentum > 0 else ())


def oracle_f64(eng, mk, n_items, step_count, P0=None, dtype=np.float64):
    """A float64 oracle holding the device's current float32 weights, hidden state and optimizer state, at dropout step
    `step_count`: the reference for one step of the device, free of the float32 rounding of a second implementation.  With
    dtype=np.float32, the same oracle in float32: what a second float32 implementation reaches on the same inputs.  The tables
    are taken from the device as they are (no random initialisation first: at 172,000 x 512 that alone takes seconds)."""
    m = orc.OracleGRU4Rec(dtype=dtype, **mk)
    nl = len(m.layers)
    m.n_items = n_items
    m.Wx, m.Wh, m.Wrz = ([eng.get('%s%d' % (kind, i)).astype(dtype) for i in range(nl)] for kind in ('Wx', 'Wh', 'Wrz'))
    m.Bh = [eng.get('Bh%d' % i).astype(dtype).reshape(-1) for i in range(nl)]
    m.H = [eng.get('H%d' % i).astype(dtype) for i in range(nl)]
    m.Wy = eng.get('Wy').astype(dtype)
    m.By = eng.get('By').astype(dtype).reshape(-1, 1)
    m.E = eng.get('E').astype(dtype) if (m.embedding and not m.constrained_embedding) else None
    m.init_opt_state()
    for name in param_names(m):
        p = oracle_param(m, name)
        for slot in opt_slots(m):
            m.opt[(name, slot)] = eng.get('%s.%s' % (name, slot)).reshape(p.shape).astype(dtype)
    m.step_count = step_count
    m.P0 = None if P0 is None else np.asarray(P0, dtype)
    return m


def random_opt_state(eng, m, rs):
    """Optimizer state in the range of a trained model: acc and upd positive, meang of both signs, countt small integers that
    differ per element (so does adam's bias correction), vel of both signs.  From zero state the first Adagrad / rmsprop / adam
    update is about +-lr whatever the size of the gradient; from this state it depends on the size."""
    for name in param_names(m):
        shape = eng.shape(name)
        for slot in opt_slots(m):
            if slot in ('acc', 'upd'):
                v = 10.0 ** rs.uniform(-4.0, -2.0, shape)
            elif slot == 'countt':
                v = rs.randint(1, 30, shape)
            else:
                v = rs.randn(*shape) * 1e-3
            eng.set('%s.%s' % (name, slot), v.astype(np.float32))


def _tc_mk(L, B, S, loss, fact, **kw):
    mk = dict(layers=[L], batch_size=B, n_sample=S, loss=loss, final_act=fact, constrained_embedding=True, adapt=None, learning_rate=0.5,
              momentum=0.0, sample_alpha=0.5)
    mk.update(kw)
    return mk


# shapes of the tensor-core training step and the edge each one covers: name -> (model keywords, n_items, step_mode)
TC_CASES = {
    # K padding of every operand
    'L16_B8_xe_logq': (_tc_mk(16, 8, 32, 'cross-entropy', 'softmax', logq=1.0), 300, 4),
    # Lk2 = 96 for 72 live values, Bk = 64, N = 93 (not a multiple of 4)
    'L36_B33_bpr': (_tc_mk(36, 33, 60, 'bpr', 'linear'), 500, 4),
    # the automatic switch (L >= 160); 2L = 320: the second N tile of the gates is 1/4 live
    'L160_B64_bprmax': (_tc_mk(160, 64, 2048, 'bpr-max', 'elu-0.5', bpreg=1.95), 4000, 2),
    # Lp = L, 3L = 768 = six full row tiles; both dropouts
    'L256_B128_top1max_drop': (_tc_mk(256, 128, 1024, 'top1-max', 'tanh', dropout_p_hidden=0.2, dropout_p_embed=0.3), 4000, 2),
    # Lp = 512: G8a column tiles with 4 live columns; two lane tiles; relu hidden activation
    'L260_B129_top1_relu': (_tc_mk(260, 129, 2048, 'top1', 'tanh', hidden_act='relu'), 4000, 2),
    # G7 K = 33 chunks on the 16-CTA cluster: five empty K splits
    'L344_B48_xe_logq': (_tc_mk(344, 48, 2048, 'cross-entropy', 'softmax', logq=1.0), 4000, 2),
    # the largest batch and the largest shipped L
    'L512_B256_xelogit': (_tc_mk(512, 256, 2048, 'xe_logit', 'softmax_logit'), 4000, 2),
    # the optimizer epilogues: Adagrad + momentum + L2
    'L224_B80_bprmax_adagrad': (_tc_mk(224, 80, 2048, 'bpr-max', 'elu-0.5', adapt='adagrad', momentum=0.4, lmbd=1e-3, learning_rate=0.05,
                                       bpreg=1.95), 4000, 2),
}


def f64_step_inputs(n_items, B, S, seed, per_item=None, input_in_scores=False, wide_group=0):
    """Sample store and (X, Y, R) of two steps: step 1 with M = B lanes; step 2 with M < B, a reset lane, a duplicated input item,
    a target that is also one of the samples, and half of the sample row heavily duplicated -- drawn from 8 items, or, with
    `per_item`, exactly `per_item` copies of each of S / 2 / per_item items (duplicate groups that fit one chunk of the
    role-specialised kernels).  `input_in_scores`: step 2 also feeds in the target of another lane and one of its samples
    (shared embedding: the input-row and the output-row update of one Wy row, once with a target column's large gradient).  `wide_group`: step 1's samples start with that many copies of
    one item."""
    rs = np.random.RandomState(seed)
    store = rs.randint(0, n_items, size=(4, S)).astype(np.int64)
    if per_item is None:
        store[1, :S // 2] = rs.randint(0, 8, size=S // 2)
    else:
        store[1, :S // 2] = rs.permutation(np.arange(S // 2) // per_item)
    X1, Y1 = rs.randint(0, n_items, B), rs.randint(0, n_items, B)
    M2 = B - max(1, B // 5)
    X2, Y2 = rs.randint(0, n_items, M2), rs.randint(0, n_items, M2)
    X2[-1] = X2[0]
    Y2[1] = store[1, 3]
    if input_in_scores:
        X2[2], X2[3] = Y2[4], store[1, S - 5]
    if wide_group:
        store[0, :wide_group] = store[0, S - 1]
    R2 = np.zeros(M2, bool)
    R2[M2 // 2] = True
    return store, [(X1, Y1, np.zeros(B, bool)), (X2, Y2, R2)]


def f64_setup(mk, n_items, step_mode, seed=0, torch_alloc=True, **inputs):
    """Engine with random weights, a random hidden state, biases, logQ support, random optimizer state and the sample store of
    f64_step_inputs(**inputs)."""
    rs = np.random.RandomState(seed)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    for h in m.H:
        h[:] = rs.randn(*h.shape).astype(np.float32) * 0.5
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    for b in m.Bh:
        b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    store, steps = f64_step_inputs(n_items, mk['batch_size'], mk['n_sample'], seed + 1, **inputs)
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=store.size, step_mode=step_mode), use_torch_allocator=torch_alloc)
    push_weights(eng, m)
    eng.set_sample_store(store)
    P0 = None
    if mk.get('logq', 0):
        P0 = rs.randint(1, 50, size=n_items).astype(np.float32)
        eng.set_logq_support(P0)
    random_opt_state(eng, m, np.random.RandomState(seed + 2))
    return eng, store, steps, P0


def dense_grads(m, G):
    """(name, gradient) of the dense parameters; Wx0 is a row table without an embedding"""
    nl = len(m.layers)
    wx0 = 0 if (m.embedding or m.constrained_embedding) else 1
    return ([('Wx%d' % i, G['dWx'][i]) for i in range(wx0, nl)] + [('Wh%d' % i, G['dWh'][i]) for i in range(nl)] +
            [('Wrz%d' % i, G['dWrz'][i]) for i in range(nl)] + [('Bh%d' % i, G['dBh'][i]) for i in range(nl)])


def sparse_grads(C, G):
    """(name, rows, per-position gradient) of the row tables a step updates (gru4rec_oracle.apply_updates)"""
    if C['mode'] == 'shared':
        out = [('Wy', C['Xc'], np.vstack([G['dSx'], G['dSy']]))]
    elif C['mode'] == 'embed':
        out = [('E', C['X'], G['dSx']), ('Wy', C['Y'], G['dSy'])]
    else:
        out = [('Wx0', C['X'], G['dSx']), ('Wy', C['Y'], G['dSy'])]
    return out + [('By', C['Y'], G['dSBy'])]


# The kernel a training step runs, told apart by the handle's counters (kernel launches, role-specialised windows, fallback
# windows) -- and by what it leaves in DSY, the dSy rows of the step:
#   'tc'          the tensor-core step (uses_tensor_cores()); writes every DSY row
#   'fast'        k_fast (step_mode 2) or its cluster variant (step_mode 3): one launch after the plan, +1 role-specialised
#                 window; keeps dSy in shared memory and never writes DSY, so the dSy rows are checked only through the Wy rows
#   'persistent'  k_persistent: one launch after the plan, +1 fallback window in step_modes 2 / 3
#   'phases'      the per-phase launch sequence (step_mode 0, and every mode with grad_cap / smoothing)
# The generic kernels keep the dSy rows of a chunk of <= 16 columns in shared memory (csrc/g4r_kernels.cuh, lossgrad) and write
# DSY only for wider chunks -- and, with grad_cap, for every chunk (the rows wait for the global norm): DSY is filled with NaN
# before the step; a row still all NaN was not written, every other row is compared (a partly non-finite row fails).  A chunk
# never splits a duplicate group, so the rows of a group wider than SC_CT columns must have been written.
STEP_PATHS = ('tc', 'fast', 'persistent', 'phases')
SC_CT = 16          # columns of one lossgrad sub tile (csrc/g4r_kernels.cuh)


def _counters(eng):
    return (eng.kernel_launches(),) + tuple(eng.fast_windows())


def _assert_path(path, before, after, step_mode, tag):
    launches, fast, fallback = (a - b for a, b in zip(after, before))
    if path == 'tc':
        return
    if path == 'fast':
        ok = launches == 2 and fast == 1 and fallback == 0
    elif path == 'persistent':
        ok = launches == 2 and fast == 0 and fallback == (1 if step_mode >= 2 else 0)
    else:
        ok = launches > 2 and fast == 0 and fallback == 0
    assert ok, '%sexpected the %s path; kernel launches +%d, role-specialised windows +%d, fallback windows +%d' % (
        tag, path, launches, fast, fallback)


def _f32_oracle_checks(m, ref_cost, m32, X, Y, R, store_row, lanes, tag, sgd):
    """The products and the gradients (plain SGD) or updates (any other optimizer) of a float32 oracle `m32`, which holds the
    state the float64 oracle `m` held before it took the step, against `m`'s on the same inputs -- the comparisons f64_run_steps
    makes for the device, so the two worst errors measure the same things.  Updates: at the touched rows of the row tables, with
    one fp32 rounding of the result per applied update."""
    names, slots = param_names(m32), opt_slots(m32)
    W0 = {n: np.array(oracle_param(m32, n)) for n in names}
    S0 = {(n, s): np.array(m32.opt[(n, s)]) for n in names for s in slots}
    cost = m32.train_step(X, Y, R, samples=store_row, slots=lanes)
    C, G, C32, G32 = m.last_cache, m.last_grads, m32.last_cache, m32.last_grads
    out = [(tag + 'cost', np.float64(cost), ref_cost, 0.0)]
    for i in range(len(m.layers)):
        out += [(tag + 'H%d' % i, C32['H_new'][i], C['H_new'][i], 0.0), (tag + 'dvec%d' % i, G32['dvec'][i], G['dvec'][i], 0.0)]
    out += [(tag + 'y%d' % i, a, b, 0.0) for i, (a, b) in enumerate(zip([lc['inp'] for lc in C32['layers'][1:]] + [C32['y_last']],
                                                                        [lc['inp'] for lc in C['layers'][1:]] + [C['y_last']]))]
    out += [(tag + 'dSx', G32['dSx'], G['dSx'], 0.0), (tag + 'dSy', G32['dSy'], G['dSy'], 0.0)]
    if sgd:
        out += [(tag + 'd' + n, g32, g, 0.0) for (n, g32), (_, g) in zip(dense_grads(m32, G32), dense_grads(m, G))]
        return out + [(tag + 'd' + n + ' rows', g32, g, 0.0) for (n, _, g32), (_, _, g) in zip(sparse_grads(C32, G32), sparse_grads(C, G))]
    touched = {n: np.unique(idx, return_counts=True) for n, idx, _ in sparse_grads(C, G)}
    for n in names:
        rows, mult = (touched[n][0], touched[n][1][:, None]) if n in touched else (slice(None), 1)
        pairs = [(n, W0[n], oracle_param(m32, n), oracle_param(m, n))] + [
            ('%s.%s' % (n, s), S0[(n, s)], m32.opt[(n, s)], m.opt[(n, s)]) for s in slots]
        for what, a0, a1, r1 in pairs:
            a0, a1, r1 = (np.asarray(a, np.float64) for a in (a0[rows], a1[rows], r1[rows]))
            out.append((tag + what + ' update', a1 - a0, r1 - a0, mult * 2.0 ** -23 * (np.abs(a0) + np.abs(a1))))
    return out


def f64_run_steps(eng, mk, n_items, store, steps, P0, path, run=None, keep_weights=True, f32_checks=None, require_dsy=True):
    """Runs `steps` through Engine.train_step on the kernel `path` (one of STEP_PATHS, or one per step; None: no counters are
    checked).  A step is (X, Y, R), or a step of orc.build_train_schedule (a dict that also holds `slots`, the H row of each
    lane: H is compared at those rows and the oracle runs with them); `run(k, X, Y, R)`, if given, runs step k on the device
    instead of Engine.train_step and returns its cost.  Step k takes sample-store row k and dropout step k.
    Before each step a float64 oracle is re-seeded from the device state (errors do not compound), after it every
    product the path keeps is paired with the oracle's: the cost, y, H and dvec = [da_h | da_r | da_z] of every layer, dSx
    (embedding modes) and the DSY rows the path wrote.  Plain SGD: every gradient is recovered from the update, W0 - W1 =
    lr * g (* the grad_cap scale): the dense ones, and the rows of Wx0 / E / Wy / By (one fp32 rounding per duplicate).  Any
    other optimizer: the updates W1 - W0 of every weight and every state tensor against the oracle's, with one fp32 rounding
    of the result per applied update.  Rows of the row tables that no position touched stay bit-identical (weights and state).
    The row tables are held as the device's float32 arrays and taken to float64 only at the touched rows, so a step costs a
    few float32 copies of each table besides the oracle's own float64 tables (at 172,000 x 512: 352 MB per copy).
    `keep_weights=False` leaves the parameters after each step out of the returned outputs (a long run on a large catalogue
    would hold one copy of every table per step).  `f32_checks`, if a list, receives the same comparisons for a float32 oracle
    run from the same state on the same inputs (_f32_oracle_checks).  `require_dsy`: a generic step after the first must have
    written some DSY row (true of f64_step_inputs' second step; the steps of a real schedule need not have a chunk wider than
    a sub tile, and then their dSy rows are checked through the Wy rows they update).
    Returns ([(what, dev, ref, extra_atol)], {output name: device array} for bitwise comparisons, [grad_cap scale per step])."""
    paths = [path] * len(steps) if path is None or isinstance(path, str) else list(path)
    assert eng.uses_tensor_cores() == (paths[0] == 'tc')
    lr = mk.get('learning_rate', 0.1)          # the default of make_config and of the oracle
    sgd = mk.get('adapt', 'adagrad') is None and not mk.get('momentum', 0) and not mk.get('lmbd', 0)
    ulp = lambda a, b: 2.0 ** -23 * (np.abs(a) + np.abs(b))        # rounding of one fp32 update
    f64 = lambda a: np.asarray(a, np.float64)
    checks, outs, scales = [], {}, []
    for k, st in enumerate(steps):
        X, Y, R, lanes = (st['X'], st['Y'], st['R'], st['slots']) if isinstance(st, dict) else tuple(st) + (None,)
        m = oracle_f64(eng, mk, n_items, k, P0)
        m32 = oracle_f64(eng, mk, n_items, k, None if P0 is None else np.asarray(P0, np.float32), np.float32) if f32_checks is not None else None
        names, slots = param_names(m), opt_slots(m)
        nl = len(m.layers)
        W0 = {n: eng.get(n) for n in names}
        S0 = {(n, s): eng.get('%s.%s' % (n, s)) for n in names for s in slots}
        dsy_all = paths[k] == 'tc' or (paths[k] == 'phases' and m.grad_cap > 0)
        if paths[k] != 'fast' and not dsy_all:
            eng.set('DSY', np.full(eng.shape('DSY'), np.nan, np.float32))
        tag = 'step %d (M=%d) ' % (k + 1, len(X))
        c0 = _counters(eng)
        cost = eng.train_step(X, Y, R) if run is None else run(k, X, Y, R)
        if paths[k] is not None:
            _assert_path(paths[k], c0, _counters(eng), eng.cfg.step_mode, tag)
        ref_cost = m.train_step(X, Y, R, samples=store[k], slots=lanes)
        C, G = m.last_cache, m.last_grads
        M, N = len(X), len(C['Y'])
        ys = [lc['inp'] for lc in C['layers'][1:]] + [C['y_last']]
        dev, ref = dict(cost=np.float64(cost)), dict(cost=ref_cost)
        hrows = slice(None, M) if lanes is None else np.asarray(lanes)
        for i in range(nl):
            for n, r in (('y', ys[i]), ('H', C['H_new'][i]), ('dvec', G['dvec'][i])):
                dev['%s%d' % (n, i)], ref['%s%d' % (n, i)] = eng.get('%s%d' % (n, i))[hrows if n == 'H' else slice(None, M)], r
        if C['mode'] != 'none':
            dev['dSx'], ref['dSx'] = eng.get('dSx')[:M], G['dSx']
        if paths[k] != 'fast':
            order = np.lexsort((np.arange(N), C['Y']))      # DSY rows: score columns sorted by (item, position) (k_plan)
            dsy = eng.get('DSY')[:N]
            wrote = ~np.isnan(dsy).all(axis=1)
            wide = np.bincount(C['Y'])[C['Y'][order]] > SC_CT
            assert wrote.all() or not dsy_all, tag + 'DSY: %d of %d rows not written' % ((~wrote).sum(), N)
            assert wrote[wide].all(), tag + 'DSY: %d rows of duplicate groups wider than a sub tile not written' % (~wrote[wide]).sum()
            # step 2 of f64_step_inputs has heavy duplicates: some chunk is wider than a sub tile
            assert wrote.any() or k == 0 or not require_dsy, tag + 'DSY: no row written'
            if wrote.any():
                dev['DSY'], ref['DSY'] = dsy[wrote], G['dSy'][order][wrote]
        W1 = {n: eng.get(n) for n in names}
        checks += [(tag + n, dev[n], ref[n], 0.0) for n in dev]
        outs.update({'%d_%s' % (k, n): v for n, v in dev.items()})
        if keep_weights:
            outs.update({'%d_%s' % (k, n): v for n, v in W1.items()})
        sc = float(m.last_gscale)
        scales.append(sc)
        sparse = sparse_grads(C, G)
        # the rows each row table's positions touched (ascending) and how many positions touched each
        touched = {n: np.unique(idx, return_inverse=True, return_counts=True) for n, idx, _ in sparse}

        def untouched_same(n, a0, a1, what):
            changed = (a0.view(np.uint32) != a1.view(np.uint32)).any(axis=1)
            changed[touched[n][0]] = False
            assert not changed.any(), tag + what + ': an untouched row changed'
        for n in touched:
            untouched_same(n, W0[n], W1[n], n)
        if sgd:
            for n, g in dense_grads(m, G):
                w0, w1 = f64(W0[n]), f64(W1[n])
                checks.append((tag + 'd' + n + ' recovered', (w0 - w1) / lr, g * sc, ulp(w0, w1) / lr))
            for n, idx, g in sparse:
                rows, inv, cnt = touched[n]
                w0, w1 = f64(W0[n][rows]), f64(W1[n][rows])
                gref = np.zeros((len(rows),) + W0[n].shape[1:])
                np.add.at(gref, inv.reshape(-1), g * sc)
                checks.append((tag + 'd' + n + ' rows recovered', (w0 - w1) / lr, gref, cnt[:, None] * (ulp(w0, w1) / lr)))
        else:
            for n in names:
                rows = touched[n][0] if n in touched else slice(None)
                mult = touched[n][2][:, None] if n in touched else 1
                pairs = [(n, W0[n], W1[n], oracle_param(m, n))]
                for s in slots:
                    S1 = eng.get('%s.%s' % (n, s))
                    if n in touched:
                        untouched_same(n, S0[(n, s)], S1, '%s.%s' % (n, s))
                    pairs.append(('%s.%s' % (n, s), S0[(n, s)], S1, m.opt[(n, s)]))
                for what, a0, a1, r1 in pairs:
                    r1 = np.asarray(r1).reshape(a0.shape)[rows]
                    a0, a1 = f64(a0[rows]), f64(a1[rows])
                    checks.append((tag + what + ' update', a1 - a0, r1 - a0, mult * ulp(a0, a1)))
        if m32 is not None:
            f32_checks += _f32_oracle_checks(m, ref_cost, m32, X, Y, R, store[k], lanes, tag, sgd)
    return checks, outs, scales


def f64_failures(checks):
    """the checks of f64_run_steps that miss the bar, as 'what: max err / max |ref|  /  max relative err above 1 % of max'"""
    out = []
    for what, dev, ref, extra in checks:
        a, r = f64_errors(dev, ref, extra)
        if not (a <= F64_REL and r <= F64_RTOL):
            out.append('%s: %.3g / %.3g' % (what, a, r))
    return out


def assert_step_costs(costs, ref, err_msg=''):
    """Per-mini-batch costs of a whole trajectory at the north-star tolerance (1e-4 relative, every step).  fp32 rounding alone
    stays two orders of magnitude below it (tests/test_oracle_grads.py::test_fp32_trajectory_noise_level)."""
    costs = np.asarray(costs); ref = np.asarray(ref)
    assert costs.shape == ref.shape, (costs.shape, ref.shape)
    np.testing.assert_allclose(costs, ref, rtol=1e-4, atol=1e-6, err_msg=err_msg)
