"""-m gpu parity tests: the CUDA path (through the C ABI) against the NumPy oracle on identical inputs.
Tolerances: integer / index work bit-exact; fp32 within 1e-4 relative (north_star), written per test."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gpu_utils import assert_step_costs, make_cfg, make_pair, compare_weights, compare_opt_state

pytestmark = pytest.mark.gpu


def small_engine(n_items=50, **mk):
    base = dict(layers=[8], batch_size=4, n_sample=8, loss='bpr-max', final_act='elu-0.5')
    base.update(mk)
    return _lib.Engine(make_cfg(n_items, base, sample_store=base['n_sample'] * 4))


# ---------------- K2': searchsorted, bit exact ----------------
@pytest.mark.parametrize('n_d,n_x,alpha', [(1000, 20000, 0.75), (37483, 200000, 0.0), (7, 1000, 1.0), (1, 10, 0.5)])
def test_searchsorted_bit_exact(n_d, n_x, alpha):
    rs = np.random.RandomState(1)
    supp = rs.randint(1, 1000, size=n_d)
    P = orc.sampling_cdf(supp, alpha).astype(np.float32)
    x = rs.rand(n_x).astype(np.float32)
    # edge values: exact hits of CDF entries, 0, just below 1, values above the max and at the min
    x[:min(n_d, 100)] = P[:min(n_d, 100)]
    x[100:104] = [0.0, np.nextafter(np.float32(1), np.float32(0)), 1.0, 1.5][:len(x[100:104])]
    eng = small_engine()
    y = eng.searchsorted(P, x)
    np.testing.assert_array_equal(y, orc.searchsorted_k2(P, x))
    np.testing.assert_array_equal(y[:300], orc.searchsorted_k2_loop(P, x[:300]))


# ---------------- K1': row gather ----------------
def test_gather_rows_and_bounds():
    rs = np.random.RandomState(2)
    eng = small_engine()
    for cols in (100, 300, 7):
        T = rs.randn(500, cols).astype(np.float32)
        idx = rs.randint(-500, 500, size=3000)
        out = eng.gather_rows(T, idx)
        np.testing.assert_array_equal(out, T[idx])
    with pytest.raises(IndexError):
        eng.gather_rows(T, np.array([0, 500]))
    with pytest.raises(IndexError):
        eng.gather_rows(T, np.array([-501]))
    assert eng.gather_rows(T, np.zeros(0, dtype=np.int64)).shape == (0, 7)


# ---------------- MRG31k3p + sample store ----------------
def test_mrg_uniform_and_store_bit_exact():
    n_items, S, rows = 300, 64, 40
    mk = dict(layers=[8], batch_size=4, n_sample=S, loss='bpr-max', final_act='elu-0.5')
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=S * rows))
    rs = np.random.RandomState(3)
    P = orc.sampling_cdf(rs.randint(1, 100, size=n_items), 0.5).astype(np.float32)
    eng.set_sampling_cdf(P)
    ref = orc.MRGStreams(12345)
    n = S * rows
    st = ref.substreams(ref.n_streams(n))
    for call in range(3):     # successive generate_samples() calls continue the same streams
        eng.generate_samples()
        u = ref.uniform_from_state(st, n)
        assert u.min() >= 0 and u.max() < 1
        np.testing.assert_array_equal(eng.get_sample_store(), orc.searchsorted_k2(P, u).reshape(rows, S))
    eng2 = _lib.Engine(make_cfg(n_items, mk, sample_store=S * rows))
    ref2 = orc.MRGStreams(12345)
    st2 = ref2.substreams(ref2.n_streams(n))
    np.testing.assert_array_equal(eng2.mrg_uniform(n), ref2.uniform_from_state(st2, n))


# ---------------- single / multi step training parity ----------------
CASES = {
    'bprmax_none_mom': dict(layers=[20], batch_size=8, n_sample=40, loss='bpr-max', final_act='elu-0.5', learning_rate=0.2, momentum=0.3, sample_alpha=0.0),
    'bprmax_none_L100_B32': dict(layers=[100], batch_size=32, n_sample=256, loss='bpr-max', final_act='elu-0.5', learning_rate=0.02, momentum=0.3),
    'xe_shared_logq_drop': dict(layers=[24], batch_size=8, n_sample=48, loss='cross-entropy', final_act='softmax', constrained_embedding=True,
                                learning_rate=0.2, momentum=0.2, logq=1.0, sample_alpha=0.5, dropout_p_hidden=0.4, dropout_p_embed=0.2, bpreg=0.0),
    'xe_embed_2layer': dict(layers=[12, 20], batch_size=6, n_sample=30, loss='cross-entropy', final_act='softmax', embedding=12,
                            learning_rate=0.1, dropout_p_embed=0.3, dropout_p_hidden=0.2, lmbd=0.001),
    'top1max_none_3layer': dict(layers=[12, 12, 12], batch_size=6, n_sample=20, loss='top1-max', final_act='tanh', learning_rate=0.1, momentum=0.1),
    'bprmax_shared_odd': dict(layers=[18], batch_size=7, n_sample=33, loss='bpr-max', final_act='elu-1', constrained_embedding=True,
                              learning_rate=0.05, momentum=0.4, bpreg=1.95, dropout_p_embed=0.5, dropout_p_hidden=0.05),
    'bpr_none': dict(layers=[16], batch_size=8, n_sample=24, loss='bpr', final_act='linear', learning_rate=0.05),
    'top1_embed': dict(layers=[16], batch_size=8, n_sample=24, loss='top1', final_act='tanh', embedding=10, learning_rate=0.05, momentum=0.2),
    'xelogit_none_sgd': dict(layers=[16], batch_size=8, n_sample=24, loss='xe_logit', final_act='softmax_logit', adapt=None, learning_rate=0.05),
    'bprmax_relu_hidden_selu': dict(layers=[16], batch_size=8, n_sample=24, loss='bpr-max', final_act='selu-1.05-1.67', hidden_act='relu', learning_rate=0.05),
    'bprmax_none_nosample': dict(layers=[16], batch_size=8, n_sample=0, loss='bpr-max', final_act='elu-0.5', learning_rate=0.1, momentum=0.2),
    'xe_none_L7_pad': dict(layers=[7], batch_size=5, n_sample=9, loss='cross-entropy', final_act='softmax', learning_rate=0.1, momentum=0.1),
}


@pytest.mark.parametrize('step_mode', [0, 1, 2, 3, 4])
@pytest.mark.parametrize('name', sorted(CASES))
def test_train_steps_match_oracle(name, step_mode):
    mk = CASES[name]
    n_items = 120
    B = mk['batch_size']
    rows = 12
    eng, m, store, rs = make_pair(n_items, mk, n_store_rows=rows if mk['n_sample'] else 0, seed=11, step_mode=step_mode)
    if step_mode == 4 and not eng.uses_tensor_cores():
        pytest.skip('the tensor-core step takes constrained embedding, one layer, L % 4 == 0, SGD / Adagrad')
    costs_d, costs_o = [], []
    for t in range(rows - 1 if mk['n_sample'] else 10):
        X = rs.randint(0, n_items, B); Y = rs.randint(0, n_items, B)
        if t % 2 == 0:      # duplicates inside the batch, and between inputs and targets
            X[1] = X[0]; Y[2] = Y[0]; Y[3] = X[0]
        if store is not None and t % 3 == 0:
            Y[4 % B] = store[t][0]        # a target that also appears among the samples
        R = rs.rand(B) < 0.3
        costs_d.append(eng.train_step(X, Y, R))
        costs_o.append(m.train_step(X, Y, R, samples=None if store is None else store[t]))
        if t == 0:
            compare_weights(eng, m, rtol=1e-4, atol=1e-6, what='after step 1')
            compare_opt_state(eng, m, rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(costs_d, costs_o, rtol=1e-4, atol=1e-6)
    compare_weights(eng, m, rtol=2e-3, atol=2e-5, what='after all steps')
    for i in range(len(m.layers)):
        np.testing.assert_allclose(eng.get('H%d' % i), m.H[i], rtol=1e-3, atol=1e-5)


@pytest.mark.parametrize('step_mode', [0, 1, 2, 3])
def test_shrinking_batch_and_slots(step_mode):
    """epoch tail: M < B with lane compaction (gru4rec.py:644-651) through a real schedule."""
    from gru4rec_b200.synth import make_sessions
    mk = dict(layers=[16], batch_size=8, n_sample=16, loss='bpr-max', final_act='elu-0.5', learning_rate=0.1, momentum=0.1)
    df = make_sessions(n_items=80, n_events=400, seed=5)
    d = orc.prepare_fit_data(df)
    eng, m, store, rs = make_pair(d['n_items'], mk, n_store_rows=400, seed=4, randomize_state=False, step_mode=step_mode)
    sched = _lib.Schedule(d['data_items'], d['offset_sessions'], d['base_order'], 8, 16, mode=0)
    steps = orc.build_train_schedule(d['data_items'], d['offset_sessions'], d['base_order'], 8, 16)
    assert sched.n_steps == len(steps) and steps[-1]['M'] < 8
    costs = eng.train_steps(sched, 0, sched.n_steps)
    ref = [m.train_step(st['X'], st['Y'], st['R'], samples=store[k], slots=st['slots']) for k, st in enumerate(steps)]
    assert_step_costs(costs, ref)
    compare_weights(eng, m, rtol=3e-3, atol=3e-5)


@pytest.mark.parametrize('loss,fact,alpha,extra', [('bpr-max', 'elu-0.5', 0.0, {}), ('cross-entropy', 'softmax', 0.75, {}), ('top1-max', 'tanh', 1.0, {}),
                                                   ('bpr-max', 'elu-1', 0.0, dict(dropout_p_hidden=0.25, lmbd=0.0005)),
                                                   ('cross-entropy', 'softmax', 0.0, dict(logq=1.0, momentum=0.0)),
                                                   ('bpr', 'linear', 0.0, dict(adapt=None, learning_rate=0.01)),
                                                   ('bpr-max', 'elu-0.5', 0.0, dict(layers=[128])),                    # widest GRU the kernel takes
                                                   ('top1', 'tanh', 0.25, dict(layers=[50], batch_size=13)),           # L not a multiple of 4, odd batch
                                                   ('xe_logit', 'softmax_logit', 0.0, dict(layers=[64], batch_size=16, momentum=0.0))])
@pytest.mark.parametrize('step_mode', [2, 3])
def test_headline_shape_role_specialised_kernel(loss, fact, alpha, extra, step_mode):
    """B=32, GRU(100), 2048 samples (BASELINE configs[1] shape) through step_mode 2 (48-CTA GRU group) and 3 (GRU on one
    thread-block cluster, weights resident in shared memory); two windows, so the resident weights are written back and
    re-read; heavy duplicates with alpha=1."""
    from gru4rec_b200.synth import make_session_arrays
    n_items = 3000
    mk = dict(layers=[100], batch_size=32, n_sample=2048, loss=loss, final_act=fact, learning_rate=0.05, momentum=0.3, sample_alpha=alpha,
              dropout_p_hidden=0.1 if loss == 'top1-max' else 0.0)
    mk.update(extra)
    items, offset, order, supports = make_session_arrays(n_items, 40000, seed=5)
    rows = 20
    eng, m, _, rs = make_pair(n_items, mk, n_store_rows=0, seed=3, randomize_state=False, step_mode=step_mode)
    eng.close()
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=rows * 2048, step_mode=step_mode))
    from gpu_utils import push_weights
    push_weights(eng, m)
    if mk.get('logq', 0):
        P0 = np.maximum(supports, 1).astype(np.float32)
        m.P0 = P0
        eng.set_logq_support(P0)
    P = orc.sampling_cdf(supports, alpha).astype(np.float32)
    u = rs.rand(rows * 2048).astype(np.float32)
    eng.set_sampling_cdf(P)
    eng.generate_samples_from_uniform(u)
    store = orc.searchsorted_k2(P, u).reshape(rows, 2048)
    np.testing.assert_array_equal(eng.get_sample_store(), store)
    sched = _lib.Schedule(items, offset, order, mk['batch_size'], 2048, mode=0)
    steps = orc.build_train_schedule(items, offset, order, mk['batch_size'], 2048)
    n = 14
    costs = np.concatenate([eng.train_steps(sched, 0, 9), eng.train_steps(sched, 9, n - 9)])
    ref = [m.train_step(st['X'], st['Y'], st['R'], samples=store[k], slots=st['slots']) for k, st in enumerate(steps[:n])]
    assert_step_costs(costs, ref)
    compare_weights(eng, m, rtol=2e-3, atol=2e-5, what='headline shape')
    fast, fallback = eng.fast_windows()
    if step_mode == 2 and mk['layers'][0] > 120:
        assert fast == 0 and fallback >= 1   # the 48-CTA GRU group covers 240 gate columns: wider layers run the generic persistent kernel
    elif alpha == 0.0:
        assert fast >= 1 and fallback == 0
    else:
        assert fast + fallback >= 1      # popularity sampling can create duplicate groups wider than a chunk -> generic kernel


@pytest.mark.parametrize('alpha', [0.0, 0.5])
def test_headline_workload_full_catalogue(alpha):
    """The benched workload itself: I = 37,483 items, B = 32, GRU(100), BPR-max, 2048 samples, momentum (BASELINE configs[1]),
    negatives drawn by the device sampler from the uniform (alpha = 0) and the popularity-based (alpha = 0.5) distribution."""
    from gru4rec_b200.synth import make_session_arrays
    from gpu_utils import push_weights
    n_items = 37483
    mk = dict(layers=[100], batch_size=32, n_sample=2048, loss='bpr-max', final_act='elu-0.5', learning_rate=0.2, momentum=0.3, sample_alpha=alpha, bpreg=1.0)
    items, offset, order, supports = make_session_arrays(n_items, 4 * n_items, seed=2)
    rows = 16
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=rows * 2048, step_mode=2))
    push_weights(eng, m)
    P = orc.sampling_cdf(supports, alpha).astype(np.float32)
    eng.set_sampling_cdf(P)
    eng.generate_samples()                          # MRG31k3p uniforms + binary search on the device
    store = eng.get_sample_store()
    assert store.min() >= 0 and store.max() < n_items
    sched = _lib.Schedule(items, offset, order, 32, 2048, mode=0)
    steps = orc.build_train_schedule(items, offset, order, 32, 2048)
    n = 10
    costs = eng.train_steps(sched, 0, n)
    ref = [m.train_step(st['X'], st['Y'], st['R'], samples=store[k], slots=st['slots']) for k, st in enumerate(steps[:n])]
    np.testing.assert_allclose(costs, ref, rtol=1e-4, atol=1e-6)
    compare_weights(eng, m, rtol=2e-3, atol=2e-5, what='headline workload')
    fast, fallback = eng.fast_windows()
    if alpha == 0.0:
        assert fast >= 1 and fallback == 0
    else:
        assert fast + fallback >= 1      # popularity sampling can create duplicate groups wider than a chunk -> generic kernel


def test_index_errors_and_nan():
    eng = small_engine()
    eng.set_sample_store(np.zeros((4, 8), dtype=np.int64))
    with pytest.raises(IndexError):
        eng.train_step([0, 1, 2, 50], [0, 1, 2, 3])
    with pytest.raises(IndexError):
        eng.set_sample_store(np.full((4, 8), 50, dtype=np.int64))
    eng.set('Wy', np.full((50, 8), np.nan, dtype=np.float32))
    with pytest.raises(_lib.NaNError):
        eng.train_step([0, 1, 2, 3], [4, 5, 6, 7])


def test_unsupported_configs_raise():
    for mk in (dict(loss='cross-entropy', final_act='linear'), dict(loss='bpr-max', final_act='softmax'), dict(adapt='adam', adapt_params=[0.9, 0.999], constrained_embedding=True)):
        with pytest.raises(NotImplementedError):
            small_engine(**mk)


# ---------------- scoring path ----------------
@pytest.mark.parametrize('mode_kw', [dict(), dict(constrained_embedding=True), dict(embedding=10)])
def test_eval_matches_oracle(mode_kw):
    from gru4rec_b200.synth import make_sessions
    mk = dict(layers=[16, 12], batch_size=8, n_sample=16, loss='bpr-max', final_act='elu-0.5')
    mk.update(mode_kw)
    df = make_sessions(n_items=90, n_events=900, seed=7)
    d = orc.prepare_fit_data(df)
    eng, m, store, rs = make_pair(d['n_items'], mk, n_store_rows=0, seed=9, eval_lanes=11)
    sched = _lib.Schedule(d['data_items'], d['offset_sessions'], None, 11, 0, mode=1)
    for mode, code in (('standard', 0), ('conservative', 1), ('median', 2)):
        rec, mrr, n = eng.eval_schedule(sched, [1, 5, 20], code)
        r0, m0 = m.evaluate(d['data_items'], d['offset_sessions'], batch_size=11, cut_off=(1, 5, 20), mode=mode)
        assert n == sched.n_events
        np.testing.assert_allclose(rec / n, r0, rtol=1e-4, atol=1e-9)
        np.testing.assert_allclose(mrr / n, m0, rtol=1e-4, atol=1e-9)
    # candidate subset with duplicates and items that never occur as targets (evaluate_gpu(items=...))
    sub = np.concatenate([np.arange(0, d['n_items'], 4), [3, 3, 7]])
    eng.set_eval_items(sub)
    for mode, code in (('standard', 0), ('conservative', 1), ('median', 2)):
        rec, mrr, n = eng.eval_schedule(sched, [1, 5, 20], code)
        r0, m0 = m.evaluate(d['data_items'], d['offset_sessions'], batch_size=11, cut_off=(1, 5, 20), mode=mode, items=sub)
        np.testing.assert_allclose(rec / n, r0, rtol=1e-4, atol=1e-9)
        np.testing.assert_allclose(mrr / n, m0, rtol=1e-4, atol=1e-9)
    with pytest.raises(IndexError):
        eng.set_eval_items([0, d['n_items']])
    eng.set_eval_items(None)
    rec, mrr, n = eng.eval_schedule(sched, [1, 5, 20], 0)
    r0, m0 = m.evaluate(d['data_items'], d['offset_sessions'], batch_size=11, cut_off=(1, 5, 20), mode='standard')
    np.testing.assert_allclose(rec / n, r0, rtol=1e-4, atol=1e-9)


def test_predict_matches_oracle():
    mk = dict(layers=[16], batch_size=8, n_sample=16, loss='cross-entropy', final_act='softmax')
    eng, m, store, rs = make_pair(70, mk, seed=13, eval_lanes=6)
    H = [np.zeros((6, 16), dtype=np.float32)]
    for t in range(3):
        X = rs.randint(0, 70, 6)
        zero = np.array([t == 0] * 6) | (rs.rand(6) < 0.3)
        out = eng.predict(X, zero.astype(np.uint8))
        ref = m.predict_step(X, H, zero=zero)
        np.testing.assert_allclose(out, ref, rtol=1e-4, atol=1e-7)
