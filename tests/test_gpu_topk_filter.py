"""-m gpu: Engine.predict_topk with filters (g4r_predict_topk_filtered, csrc/g4r_topk.cuh): a candidate set and per-lane
exclusions, against predict() on a twin engine with the same weights and inputs, masked and stable-sorted.  Items must match
exactly and scores bit for bit, on the fp32 FFMA tiles (eval_tc=1) and on the wgmma 3xTF32 tiles (eval_tc=2)."""
import ctypes as C

import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gpu_utils import push_weights

pytestmark = pytest.mark.gpu

TC = [False, True]


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


def _inputs(rs, n_items, lanes):
    return rs.randint(0, n_items, lanes).astype(np.int32)


def _eligible(shape, cand=None, excl=None):
    ok = np.ones(shape, bool)
    if cand is not None:
        ok[:] = False
        ok[:, np.asarray(cand)] = True
    for b, e in enumerate(excl or []):
        if e is not None and len(e):
            ok[b, np.asarray(e)] = False
    return ok


def _ref(key, k, cand=None, excl=None):
    """stable descending order of `key` over each lane's eligible items: (items, positions live)"""
    ok = _eligible(key.shape, cand, excl)
    order = np.argsort(-np.where(ok, key, -np.inf), axis=1, kind='stable')[:, :k]
    live = np.take_along_axis(ok, order, axis=1)
    return np.where(live, order, -1).astype(np.int32), live


def _assert_filtered(items, scores, p, k, cand=None, excl=None, what=''):
    e_items, live = _ref(p, k, cand, excl)
    np.testing.assert_array_equal(items, e_items, err_msg=what)
    e_scores = np.take_along_axis(p, np.maximum(e_items, 0), axis=1)
    np.testing.assert_array_equal(scores[live].view(np.uint32), e_scores[live].view(np.uint32), err_msg=what)
    assert np.isnan(scores[~live]).all(), what


def _raw_filtered(eng, X, k, cand, off, ex, reset=None):
    """g4r_predict_topk_filtered through ctypes: (return code, items, scores)"""
    out_i = np.empty((len(X), max(k, 1)), np.int32); out_s = np.empty((len(X), max(k, 1)), np.float32)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    rc = eng.lib.g4r_predict_topk_filtered(eng.h, p(X), len(X), p(reset), k, p(cand), 0 if cand is None else len(cand), p(off), p(ex),
                                           p(out_i), p(out_s))
    return rc, out_i, out_s


@pytest.mark.parametrize('k', [20, 1024])
def test_half_catalogue_candidates(k):
    """(a) a random 50 % candidate set of the RSC15 catalogue, 129 lanes (two lane blocks of the wgmma tiles)"""
    n_items, lanes = 37483, 129
    mk, m = _model(n_items, 'elu-0.5', [48], seed=1)
    ref = _engine(n_items, mk, m, lanes)
    engs = {tc: _engine(n_items, mk, m, lanes, tc) for tc in TC}
    rs = np.random.RandomState(2)
    cand = np.sort(rs.choice(n_items, n_items // 2, replace=False)).astype(np.int32)
    for step in range(2):
        X = _inputs(rs, n_items, lanes)
        reset = None if step == 0 else (np.arange(lanes) % 3 == 1).astype(np.uint8)
        p = ref.predict(X, reset)
        for tc, eng in engs.items():
            items, scores = eng.predict_topk(X, k, reset, items=rs.permutation(cand))
            _assert_filtered(items, scores, p, k, cand, what='eval_tc=%s step %d' % (tc, step))


@pytest.mark.parametrize('tc', TC)
def test_candidates_avoid_the_catalogue_prefix(tc):
    """(b) no candidate in [0, P): a tau taken from the catalogue's own prefix would be above the best candidates"""
    n_items, lanes, k = 37483, 64, 50
    mk, m = _model(n_items, 'tanh', [40], seed=3, by=np.r_[np.full(6000, 2.0), np.zeros(n_items - 6000)].astype(np.float32).reshape(-1, 1))
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(4)
    cand = (6000 + rs.choice(n_items - 6000, 9000, replace=False)).astype(np.int32)
    X = _inputs(rs, n_items, lanes)
    items, scores = eng.predict_topk(X, k, items=cand)
    _assert_filtered(items, scores, ref.predict(X), k, cand)


@pytest.mark.parametrize('tc', TC)
def test_small_candidate_set_runs_no_tile(tc):
    """(c) 300 candidates of 20,000: the exact prefix holds them all, so no catalogue tile kernel runs"""
    n_items, lanes, k = 20000, 96, 40
    mk, m = _model(n_items, 'leaky-0.1', [32], seed=5)
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    twin = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(6)
    cand = rs.choice(n_items, 300, replace=False).astype(np.int32)
    ones = np.ones(lanes, np.uint8)
    X = _inputs(rs, n_items, lanes)
    twin.predict_topk(X, k, ones)
    n0 = twin.kernel_launches(); twin.predict_topk(X, k, ones); d_plain = twin.kernel_launches() - n0
    eng.predict_topk(X, k, ones, items=cand)
    n0 = eng.kernel_launches()
    items, scores = eng.predict_topk(X, k, ones, items=cand)
    d_filt = eng.kernel_launches() - n0
    _assert_filtered(items, scores, ref.predict(X, ones), k, cand)
    assert d_filt < d_plain, (d_filt, d_plain)


@pytest.mark.parametrize('tc', TC)
def test_k_equals_candidates_and_k_above_errors(tc):
    """(d) k == the number of distinct candidates returns them all in order; k above it is an error"""
    n_items, lanes = 5000, 40
    mk, m = _model(n_items, 'relu', [32], seed=7, by=-0.35)
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(8)
    cand = rs.choice(n_items, 64, replace=False).astype(np.int32)
    ones = np.ones(lanes, np.uint8)
    X = _inputs(rs, n_items, lanes)
    items, scores = eng.predict_topk(X, 64, ones, items=np.r_[cand, cand[:9]])
    _assert_filtered(items, scores, ref.predict(X, ones), 64, cand)
    with pytest.raises(ValueError):
        eng.predict_topk(X, 65, ones, items=cand)
    rc, _, _ = _raw_filtered(eng, X, 65, cand, None, None, ones)
    assert rc == _lib.G4R_ERR_INVALID


@pytest.mark.parametrize('n_items', [2049, 4097])
@pytest.mark.parametrize('k', [20, 100])
def test_relu_zero_ties_and_padded_last_tile(n_items, k):
    """(e) relu with By = -0.35: zero ties across position k; candidates in the padded last tile (4097 items: the tiles run)"""
    lanes = 40
    mk, m = _model(n_items, 'relu', [64], seed=9, by=-0.35)
    ref = _engine(n_items, mk, m, lanes)
    engs = {tc: _engine(n_items, mk, m, lanes, tc) for tc in TC}
    rs = np.random.RandomState(10)
    cand = np.r_[rs.choice(n_items - 1, int(0.9 * n_items), replace=False), n_items - 1].astype(np.int32)
    X = _inputs(rs, n_items, lanes)
    p = ref.predict(X)
    assert (p == 0).sum(axis=1).min() > k
    for tc, eng in engs.items():
        items, scores = eng.predict_topk(X, k, items=cand)
        _assert_filtered(items, scores, p, k, cand, what='eval_tc=%s' % tc)


def _exclusions(rs, p, k, sizes, P, n_items):
    """per lane: sizes[b % len] items, unsorted, with duplicates, holding the lane's unfiltered top k; lane 3 excludes the best
    items of the catalogue prefix [0, P)"""
    top = np.argsort(-p, axis=1, kind='stable')
    out = []
    for b in range(len(p)):
        n = sizes[b % len(sizes)]
        if n == 0:
            out.append(None if b % 2 else np.zeros(0, np.int64))
            continue
        e = list(top[b, :min(n, k)]) + list(rs.randint(0, n_items, max(0, n - k)))
        if b == 3:
            e = list(np.argsort(-p[b, :P], kind='stable')[:n])
        e = np.array(e + e[: n // 4])
        out.append(rs.permutation(e))
    return out


@pytest.mark.parametrize('tc', TC)
@pytest.mark.parametrize('with_cand', [False, True])
def test_exclusions_per_lane(tc, with_cand):
    """(f) 0, 1, 50 and 3,000 exclusions per lane (unsorted, duplicated, holding the lane's unfiltered top k); one lane excludes
    the best items of the prefix, so a tau computed before the exclusions would drop real winners"""
    n_items, lanes, k = 37483, 64, 100
    mk, m = _model(n_items, 'elu-0.5', [48], seed=11)
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(12)
    cand = rs.choice(n_items, n_items // 2, replace=False).astype(np.int32) if with_cand else None
    ones = np.ones(lanes, np.uint8)
    X = _inputs(rs, n_items, lanes)
    p = ref.predict(X, ones)
    key = p if cand is None else np.where(_eligible(p.shape, cand), p, -np.inf)
    excl = _exclusions(rs, key, k, [0, 1, 50, 3000], 2368, n_items)
    items, scores = eng.predict_topk(X, k, ones, items=cand, exclude=excl)
    _assert_filtered(items, scores, p, k, cand, excl)


@pytest.mark.parametrize('tc', TC)
def test_short_lanes(tc):
    """(g) fewer eligible items than k: the eligible ones best first, then item -1 / NaN"""
    n_items, lanes, k = 6000, 8, 30
    mk, m = _model(n_items, 'tanh', [32], seed=13)
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(14)
    cand = rs.choice(n_items, 40, replace=False).astype(np.int32)
    excl = [cand[:n] for n in (0, 5, 10, 20, 35, 40, 39, 1)]
    X = _inputs(rs, n_items, lanes)
    items, scores = eng.predict_topk(X, k, items=cand, exclude=excl)
    _assert_filtered(items, scores, ref.predict(X), k, cand, excl)
    assert (items[5] == -1).all() and (items[4, 5:] == -1).all() and (items[3, :20] >= 0).all() and (items[3, 20:] == -1).all()


@pytest.mark.parametrize('tc', TC)
def test_overflow_fallback_respects_the_mask(tc):
    """(h) rising scores overflow every survivor list; the fallback row must keep to the candidates: the single best item of the
    catalogue is not one and must not appear"""
    n_items, lanes, k = 20000, 16, 20
    by = np.linspace(-1, 1, n_items, dtype=np.float32).reshape(-1, 1)
    mk, m = _model(n_items, 'linear', [16], seed=15, by=by, wy_scale=1e-3)
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(16)
    cand = rs.choice(n_items - 1, 12000, replace=False).astype(np.int32)
    ones = np.ones(lanes, np.uint8)
    X = _inputs(rs, n_items, lanes)
    excl = [np.array([cand.max()]) if b % 2 else None for b in range(lanes)]
    n0 = eng.kernel_launches()
    items, scores = eng.predict_topk(X, k, ones, items=cand, exclude=excl)
    d_overflow = eng.kernel_launches() - n0
    p = ref.predict(X, ones)
    assert p.argmax(axis=1).tolist() == [n_items - 1] * lanes
    _assert_filtered(items, scores, p, k, cand, excl)
    assert not (items == n_items - 1).any()
    for e in (ref, eng):
        e.set('By', by[::-1].copy())
    n0 = eng.kernel_launches()
    items, scores = eng.predict_topk(X, k, ones, items=cand, exclude=excl)
    d_plain = eng.kernel_launches() - n0
    _assert_filtered(items, scores, ref.predict(X, ones), k, cand, excl)
    assert d_overflow == d_plain + 1, (d_overflow, d_plain)


@pytest.mark.parametrize('act', ['softmax', 'softmax_logit'])
@pytest.mark.parametrize('n_cand', [300, 2500])
def test_softmax_normalised_over_candidates(act, n_cand):
    """(i) softmax: order of the linear twin's pre-activations over the candidates, probabilities within 1e-5 of a float64
    softmax over the distinct candidates, and the same probabilities with or without exclusions"""
    n_items, lanes, k = 3000, 80, 50
    mk, m = _model(n_items, act, [64], seed=17)
    ref_pre = _engine(n_items, dict(mk, final_act='linear', loss='bpr-max'), m, lanes)
    rs = np.random.RandomState(18)
    cand = rs.choice(n_items, n_cand, replace=False).astype(np.int32)
    X = _inputs(rs, n_items, lanes)
    pre = ref_pre.predict(X).astype(np.float64)
    z = pre[:, cand]
    prob = np.exp(pre - z.max(axis=1, keepdims=True)) / np.exp(z - z.max(axis=1, keepdims=True)).sum(axis=1, keepdims=True)
    excl = [cand[rs.choice(n_cand, 30, replace=False)] if b % 2 else None for b in range(lanes)]
    for tc in TC:
        a = _engine(n_items, mk, m, lanes, tc)
        b = _engine(n_items, mk, m, lanes, tc)
        ia, sa = a.predict_topk(X, k, items=np.r_[cand, cand[:7]])
        ib, sb = b.predict_topk(X, k, items=cand, exclude=excl)
        for items, scores, ex in ((ia, sa, None), (ib, sb, excl)):
            e_items, _ = _ref(pre, k, cand, ex)
            np.testing.assert_array_equal(items, e_items, err_msg='eval_tc=%s' % tc)
            np.testing.assert_allclose(scores, np.take_along_axis(prob, e_items, axis=1), rtol=1e-5, atol=0, err_msg='eval_tc=%s' % tc)
        for lane in range(lanes):                       # an item's probability does not depend on the exclusions
            da = dict(zip(ia[lane], sa[lane].view(np.uint32)))
            for it, s in zip(ib[lane], sb[lane].view(np.uint32)):
                if it in da:
                    assert da[it] == s, (tc, lane, it)


@pytest.mark.parametrize('tc', TC)
def test_no_filter_equals_predict_topk_and_alternates(tc):
    """(j) the filtered entry point without filters is bitwise g4r_predict_topk; filtered, unfiltered and predict calls
    alternate on one engine with resets and fewer lanes than reserved, and follow a predict-only twin"""
    n_items, lanes, k = 2600, 100, 30
    mk, m = _model(n_items, 'elu-0.5', [40], seed=19)
    a = _engine(n_items, mk, m, lanes, tc)
    b = _engine(n_items, mk, m, lanes, tc)
    c = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(20)
    cand = rs.choice(n_items, 1800, replace=False).astype(np.int32)
    for step in range(8):
        batch = 70 if step < 5 else 100
        X = _inputs(rs, n_items, batch)
        reset = (rs.rand(batch) < 0.2).astype(np.uint8)
        p = b.predict(X, reset)
        if step % 4 == 0:
            rc, items, scores = _raw_filtered(a, X, k, None, None, None, reset)
            assert rc == 0
            i2, s2 = c.predict_topk(X, k, reset)
            np.testing.assert_array_equal(items, i2)
            np.testing.assert_array_equal(scores.view(np.uint32), s2.view(np.uint32))
            _assert_filtered(items, scores, p, k, what='step %d' % step)
            continue
        c.predict(X, reset)
        if step % 4 == 1:
            excl = [rs.choice(n_items, 20) for _ in range(batch)]
            items, scores = a.predict_topk(X, k, reset, items=cand, exclude=excl)
            _assert_filtered(items, scores, p, k, cand, excl, 'step %d' % step)
        elif step % 4 == 2:
            items, scores = a.predict_topk(X, k, reset)
            _assert_filtered(items, scores, p, k, what='step %d' % step)
        else:
            np.testing.assert_array_equal(a.predict(X, reset), p)


@pytest.mark.parametrize('tc', TC)
def test_candidate_cache_follows_content_and_weights(tc):
    """(k) a second candidate list of the same length replaces the cached one; set('Wy') is seen with a cached list"""
    n_items, lanes, k = 12000, 64, 20
    mk, m = _model(n_items, 'linear', [32], seed=21)
    a = _engine(n_items, mk, m, lanes, tc)
    b = _engine(n_items, mk, m, lanes)
    rs = np.random.RandomState(22)
    ones = np.ones(lanes, np.uint8)
    c1 = rs.choice(n_items, 5000, replace=False).astype(np.int32)
    c2 = rs.choice(n_items, 5000, replace=False).astype(np.int32)
    for cand in (c1, c2, c2, c1):
        X = _inputs(rs, n_items, lanes)
        items, scores = a.predict_topk(X, k, ones, items=cand)
        _assert_filtered(items, scores, b.predict(X, ones), k, cand)
    Wy = (rs.randn(*m.Wy.shape) * 0.2).astype(np.float32)
    a.set('Wy', Wy); b.set('Wy', Wy)
    X = _inputs(rs, n_items, lanes)
    items, scores = a.predict_topk(X, k, ones, items=c1)
    _assert_filtered(items, scores, b.predict(X, ones), k, c1, what='after set Wy')


@pytest.mark.parametrize('tc', TC)
def test_errors_leave_the_hidden_state(tc):
    """(l) out-of-range candidates or exclusions, bad offsets and bad k are refused before the hidden state moves"""
    n_items, lanes, k = 4000, 32, 20
    mk, m = _model(n_items, 'elu-0.5', [32], seed=23)
    a = _engine(n_items, mk, m, lanes, tc)
    b = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(24)
    X = _inputs(rs, n_items, lanes)
    a.predict(X); b.predict(X)                                     # a non-zero hidden state
    cand = rs.choice(n_items, 500, replace=False).astype(np.int32)
    X = _inputs(rs, n_items, lanes)
    bad_c = cand.copy(); bad_c[7] = n_items
    with pytest.raises(IndexError):
        a.predict_topk(X, k, items=bad_c)
    with pytest.raises(IndexError):
        a.predict_topk(X, k, exclude=[np.array([-1])] + [None] * (lanes - 1))
    with pytest.raises(ValueError):
        a.predict_topk(X, 501, items=cand)
    off = np.zeros(lanes + 1, np.int64); ex = np.arange(10, dtype=np.int32)
    for bad_off in (np.r_[1, np.full(lanes, 10)], np.r_[0, 5, 3, np.full(lanes - 2, 10)]):
        rc, _, _ = _raw_filtered(a, X, k, cand, bad_off.astype(np.int64), ex)
        assert rc == _lib.G4R_ERR_INVALID
    rc, _, _ = _raw_filtered(a, X, k, bad_c, off, ex)
    assert rc == _lib.G4R_ERR_INDEX
    off[1:] = 10; ex[4] = n_items + 3
    rc, _, _ = _raw_filtered(a, X, k, cand, off, ex)
    assert rc == _lib.G4R_ERR_INDEX
    for bad_k in (0, 501, _lib.G4R_TOPK_MAX + 1):
        rc, _, _ = _raw_filtered(a, X, bad_k, cand, None, None)
        assert rc == _lib.G4R_ERR_INVALID
    np.testing.assert_array_equal(a.predict(X), b.predict(X))


@pytest.mark.parametrize('tc', TC)
def test_filtered_calls_are_deterministic(tc):
    """(m) two identical calls give bitwise identical results"""
    n_items, lanes, k = 30000, 128, 100
    mk, m = _model(n_items, 'softmax', [48], seed=25)
    a = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(26)
    cand = rs.choice(n_items, 20000, replace=False).astype(np.int32)
    excl = [rs.choice(n_items, 50) for _ in range(lanes)]
    X = _inputs(rs, n_items, lanes)
    ones = np.ones(lanes, np.uint8)
    r = [a.predict_topk(X, k, ones, items=cand, exclude=excl) for _ in range(2)]
    np.testing.assert_array_equal(r[0][0], r[1][0])
    np.testing.assert_array_equal(r[0][1].view(np.uint32), r[1][1].view(np.uint32))


@pytest.mark.parametrize('tc', TC)
def test_shared_embedding_model(tc):
    """(n) a constrained_embedding model (the item table doubles as the input embedding)"""
    n_items, lanes, k = 8000, 96, 40
    mk, m = _model(n_items, 'linear', [64], seed=27, constrained_embedding=True)
    ref = _engine(n_items, mk, m, lanes)
    eng = _engine(n_items, mk, m, lanes, tc)
    rs = np.random.RandomState(28)
    cand = rs.choice(n_items, 5000, replace=False).astype(np.int32)
    for step in range(2):
        X = _inputs(rs, n_items, lanes)
        excl = [X[b:b + 1] for b in range(lanes)]
        items, scores = eng.predict_topk(X, k, None, items=cand, exclude=excl)
        _assert_filtered(items, scores, ref.predict(X), k, cand, excl, 'step %d' % step)
