"""-m gpu: Engine.predict_topk (g4r_predict_topk, csrc/g4r_topk.cuh) against predict() plus a stable sort on a twin engine with
the same weights and inputs.  Items must match exactly and scores bit for bit, on the fp32 FFMA tiles (eval_tc=False) and on
the wgmma 3xTF32 tiles (eval_tc=True)."""
import ctypes as C

import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
from gpu_utils import param_names, push_weights

pytestmark = pytest.mark.gpu


def _model(n_items, act, layers, seed, by=None, wy_scale=1.0, **mk_extra):
    loss = {'softmax': 'cross-entropy', 'softmax_logit': 'xe_logit'}.get(act, 'bpr-max')
    mk = dict(layers=layers, batch_size=8, n_sample=0, loss=loss, final_act=act, **mk_extra)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1 if by is None else by
    m.Wy[:] = (m.Wy * np.float32(wy_scale)).astype(np.float32)
    return mk, m


def _engine(n_items, mk, m, lanes, tc=None):
    eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=tc))
    push_weights(eng, m)
    return eng


def _sorted_predict(p, k):
    order = np.argsort(-p, axis=1, kind='stable')[:, :k]
    return order.astype(np.int32), np.take_along_axis(p, order, axis=1)


def _assert_topk(items, scores, p, k, what=''):
    e_items, e_scores = _sorted_predict(p, k)
    np.testing.assert_array_equal(items, e_items, err_msg=what)
    np.testing.assert_array_equal(scores.view(np.uint32), e_scores.view(np.uint32), err_msg=what)


def _inputs(rs, n_items, lanes):
    return rs.randint(0, n_items, lanes).astype(np.int32)


# n_items, layers, lanes, act, k, By, Wy scale, extra model arguments
CASES = [
    (200, [32], 8, 'linear', 200, None, 1.0, {}),                     # k = n_items, catalogue under one tile
    (2049, [64], 40, 'relu', 20, -0.35, 1.0, {}),                     # zero ties straddle position k; padded last tile
    (2049, [64], 40, 'relu', 1024, -0.35, 1.0, {}),
    (256, [64], 40, 'relu', 100, -0.35, 1.0, {}),
    (3000, [48], 129, 'leaky-0.1', 20, None, 1.0, {}),                # two lane blocks
    (5000, [100], 1, 'elu-0.5', 100, None, 1.0, {}),                  # one lane
    (4100, [40], 33, 'selu-1.05-1.67', 1, None, 1.0, {}),             # lanes not a multiple of 32
    (3000, [32], 70, 'tanh', 100, None, 60.0, {}),                    # saturated tanh: exact +-1 ties
    (2500, [48, 24], 64, 'elu-0.5', 20, None, 1.0, {}),               # two layers
    (3000, [64], 96, 'linear', 20, None, 1.0, dict(constrained_embedding=True)),   # shared embedding
]


@pytest.mark.parametrize('n_items,layers,lanes,act,k,by,wys,extra',
                         [pytest.param(*c, id='%d-%s-%d-%s-k%d' % (c[0], 'x'.join(map(str, c[1])), c[2], c[3], c[4])) for c in CASES])
def test_topk_equals_sorted_predict(n_items, layers, lanes, act, k, by, wys, extra):
    mk, m = _model(n_items, act, layers, seed=1, by=by, wy_scale=wys, **extra)
    ref = _engine(n_items, mk, m, lanes)
    engs = {tc: _engine(n_items, mk, m, lanes, tc) for tc in (False, True)}
    rs = np.random.RandomState(2)
    for step in range(2):                 # the second call carries the hidden state, with two lanes reset
        X = _inputs(rs, n_items, lanes)
        reset = None if step == 0 else (np.arange(lanes) % 3 == 1).astype(np.uint8)
        p = ref.predict(X, reset)
        for tc, eng in engs.items():
            items, scores = eng.predict_topk(X, k, reset)
            _assert_topk(items, scores, p, k, 'eval_tc=%s step %d' % (tc, step))
    for e in [ref] + list(engs.values()):
        e.close()


@pytest.mark.parametrize('act', ['softmax', 'softmax_logit'])
def test_topk_softmax_orders_by_preactivation(act):
    n_items, lanes, k = 3000, 80, 50
    mk, m = _model(n_items, act, [64], seed=4)
    mk_lin = dict(mk, final_act='linear', loss='bpr-max')
    ref_pre = _engine(n_items, mk_lin, m, lanes)             # predict() of a linear model = the pre-activation scores
    ref_p = _engine(n_items, mk, m, lanes)
    engs = {tc: _engine(n_items, mk, m, lanes, tc) for tc in (False, True)}
    rs = np.random.RandomState(5)
    for step in range(2):
        X = _inputs(rs, n_items, lanes)
        pre = ref_pre.predict(X)
        p = ref_p.predict(X)
        e_items, _ = _sorted_predict(pre, k)
        for tc, eng in engs.items():
            items, scores = eng.predict_topk(X, k)
            np.testing.assert_array_equal(items, e_items, err_msg='eval_tc=%s' % tc)
            np.testing.assert_allclose(scores, np.take_along_axis(p, e_items, axis=1), rtol=1e-5, atol=0, err_msg='eval_tc=%s' % tc)


@pytest.mark.parametrize('tc', [False, True])
def test_topk_overflow_fallback(tc):
    """scores rising with the item index: the prefix bound lets through almost the whole catalogue, every lane overflows its
    survivor list and takes the exact whole-row path (one extra kernel launch); the result is still the sorted predict()"""
    n_items, lanes, k = 20000, 16, 20
    mk, m = _model(n_items, 'linear', [16], seed=6, by=np.linspace(-1, 1, n_items, dtype=np.float32).reshape(-1, 1), wy_scale=1e-3)
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(7)
    X = _inputs(rs, n_items, lanes)
    n0 = eng.kernel_launches()
    items, scores = eng.predict_topk(X, k, np.ones(lanes, np.uint8))
    d_overflow = eng.kernel_launches() - n0
    p = ref.predict(X, np.ones(lanes, np.uint8))
    _assert_topk(items, scores, p, k)
    # falling scores: the prefix holds the best items, nothing overflows
    for e in (ref, eng):
        e.set('By', m.By[::-1].copy())
    n0 = eng.kernel_launches()
    items, scores = eng.predict_topk(X, k, np.ones(lanes, np.uint8))
    d_plain = eng.kernel_launches() - n0
    _assert_topk(items, scores, ref.predict(X, np.ones(lanes, np.uint8)), k)
    assert d_overflow == d_plain + 1, (d_overflow, d_plain)


@pytest.mark.parametrize('tc', [False, True])
def test_topk_alternates_with_predict(tc):
    """predict and predict_topk advance the same hidden state: alternating them on one engine, with resets and fewer lanes than
    the engine reserves, gives what a predict-only twin gives"""
    n_items, lanes, k = 2600, 100, 30
    mk, m = _model(n_items, 'elu-0.5', [40], seed=8)
    a = _engine(n_items, mk, m, lanes, tc)
    b = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(9)
    for step in range(6):
        batch = 70 if step < 4 else 100
        X = _inputs(rs, n_items, batch)
        reset = (rs.rand(batch) < 0.2).astype(np.uint8)
        p = b.predict(X, reset)
        if step % 2 == 0:
            items, scores = a.predict_topk(X, k, reset)
            _assert_topk(items, scores, p, k, 'step %d' % step)
        else:
            np.testing.assert_array_equal(a.predict(X, reset), p)


def test_topk_split_cache_follows_the_weights():
    """the wgmma tiles of top-k and evaluation share one split item table, kept between calls: set('Wy'), set('By') and training
    must all be seen, also when an evaluation made the split that top-k then uses"""
    n_items, lanes, k = 3000, 128, 20
    mk, m = _model(n_items, 'linear', [32], seed=10)
    a = _engine(n_items, mk, m, lanes, True)
    b = _engine(n_items, mk, m, lanes)
    rs = np.random.RandomState(11)
    ones = np.ones(lanes, np.uint8)
    d = orc.prepare_fit_data(make_sessions(n_items=n_items, n_events=3000, seed=12))
    esched = _lib.Schedule(d['data_items'] % n_items, d['offset_sessions'], None, lanes, 0, mode=1)
    m_last = int(esched.export()['M'][-1])

    def check(what):
        X = _inputs(rs, n_items, lanes)
        items, scores = a.predict_topk(X, k, ones)
        _assert_topk(items, scores, b.predict(X, ones), k, what)

    def check_eval(what):
        twin = _engine(n_items, mk, m, lanes, True)     # a fresh engine: its split is made from the current weights
        for name in param_names(m):
            twin.set(name, a.get(name))
        for call in range(2):                           # the first call on `a` splits the new table, the second reuses it
            got = [tuple(e.eval_schedule(esched, [1, 5, 20], 0)) + (e.eval_counts(m_last),) for e in (a, twin)]
            for x, y in zip(*got):
                np.testing.assert_array_equal(x, y, err_msg='%s, call %d' % (what, call))
        twin.close()

    check('initial')
    Wy = (rs.randn(*m.Wy.shape) * 0.2).astype(np.float32)
    a.set('Wy', Wy); b.set('Wy', Wy)
    check_eval('evaluation after set Wy')
    check('after set Wy and an evaluation')
    By = (rs.randn(*m.By.shape) * 0.5).astype(np.float32)
    a.set('By', By); b.set('By', By)
    check('after set By')
    sched = _lib.Schedule(d['data_items'] % n_items, d['offset_sessions'], None, 8, 0, mode=0)
    a.train_steps(sched)
    for name in param_names(m):                # the twin takes the trained weights (its own split is never cached)
        b.set(name, a.get(name))
    check_eval('evaluation after train_steps')
    check('after train_steps and an evaluation')


@pytest.mark.parametrize('tc', [False, True])
def test_topk_deterministic_and_errors(tc):
    n_items, lanes, k = 4000, 96, 100
    mk, m = _model(n_items, 'relu', [48], seed=13, by=-0.35)
    a = _engine(n_items, mk, m, lanes, tc)
    b = _engine(n_items, mk, m, lanes, tc)
    X = _inputs(np.random.RandomState(14), n_items, lanes)
    ones = np.ones(lanes, np.uint8)
    r = [a.predict_topk(X, k, ones), a.predict_topk(X, k, ones), b.predict_topk(X, k, ones)]
    for items, scores in r[1:]:
        np.testing.assert_array_equal(items, r[0][0])
        np.testing.assert_array_equal(scores.view(np.uint32), r[0][1].view(np.uint32))
    for bad in (0, n_items + 1, _lib.G4R_TOPK_MAX + 1):
        with pytest.raises(ValueError):
            a.predict_topk(X, bad)
        out_i = np.empty((lanes, max(bad, 1)), np.int32); out_s = np.empty((lanes, max(bad, 1)), np.float32)
        rc = a.lib.g4r_predict_topk(a.h, X.ctypes.data_as(C.c_void_p), lanes, None, bad, out_i.ctypes.data_as(C.c_void_p), out_s.ctypes.data_as(C.c_void_p))
        assert rc == _lib.G4R_ERR_INVALID
    with pytest.raises(NotImplementedError):
        a.predict_topk(_inputs(np.random.RandomState(15), n_items, lanes + 1), k)
    bad_x = X.copy(); bad_x[3] = n_items
    with pytest.raises(IndexError):
        a.predict_topk(bad_x, k)
    # the rejected calls left the state alone
    items, scores = a.predict_topk(X, k, ones)
    np.testing.assert_array_equal(items, r[0][0])


def test_topk_non_finite_weights_return():
    """non-finite weights have no ordering requirement, but the call must come back with a result of the right shape"""
    n_items, lanes, k = 3000, 64, 20
    mk, m = _model(n_items, 'tanh', [32], seed=16)
    Wy = m.Wy.copy(); Wy[5] = np.nan; Wy[7] = np.inf
    for tc in (False, True):
        eng = _engine(n_items, mk, m, lanes, tc)
        eng.set('Wy', Wy)
        items, scores = eng.predict_topk(_inputs(np.random.RandomState(17), n_items, lanes), k)
        assert items.shape == (lanes, k) and scores.shape == (lanes, k)
        eng.close()
