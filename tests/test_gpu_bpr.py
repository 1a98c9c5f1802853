"""BPR-MF on the device (DESIGN §3k).  The fit: the dataflow SGD bitwise equal to its strictly sequential run (max_warps = 1) on
data built for long chains (one item in most events, p == n draws, sessions of 1 to 3,000 events) at n_factors 1, 7, 100, 130
and 1024; two fits bitwise equal; U and I within 1e-12 of oracle/bpr_oracle.py and within 1e-10 of the reference's recorded runs;
the largest level equal to the oracle's longest chain.  The evaluation: per-event counts, sums and top-k lists bitwise the
oracle's in all four modes x items= (with duplicates) x exclude_seen x history, on a small catalogue and on 172,000 items (several
blocks of events, sessions across block boundaries).  A GRU4Rec and an ItemKNN evaluation in the same process stay bitwise
unchanged."""
import contextlib
import io
import itertools
import os

import numpy as np
import pandas as pd
import pytest

import baselines_oracle as bo
import bpr_oracle as bpo
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'baselines')


def _chain_data(n_items=40, seed=0):
    """sessions of 1 .. 3,000 events, item 0 in most events: the draws give long chains on I[0] and p == n often"""
    rs = np.random.RandomState(seed)
    lens = np.r_[1, 1, 2, 5, rs.randint(1, 40, 150), 700, 3000]
    rows_s = np.repeat(np.arange(len(lens)), lens).astype(np.int32)
    rows_i = np.where(rs.rand(len(rows_s)) < 0.7, 0, rs.randint(0, n_items, len(rows_s))).astype(np.int32)
    rows_i[:n_items] = np.arange(n_items)
    return rows_s, rows_i, len(lens), n_items


def _device_fit(rows_s, rows_i, S, NI, F, draws, U0, I0, bI, hyper, max_warps=1 << 30):
    dev = _lib.Baselines('bpr', NI, F)
    dev.bpr_begin(rows_s, rows_i, S, U0, I0, bI)
    stats = [dev.bpr_iterate(p, n, *hyper, max_warps=max_warps) for p, n in draws]
    U, I = dev.bpr_export()
    return U, I, stats


@pytest.mark.parametrize('F', [1, 7, 100, 130, 1024])
def test_dataflow_fit_equals_the_sequential_run_bitwise(F):
    rows_s, rows_i, S, NI = _chain_data()
    rs = np.random.RandomState(F)
    U0, I0, bI = rs.randn(S, F) * 0.1, rs.randn(NI, F) * 0.1, rs.randn(NI) * 0.01
    draws = [(rs.permutation(len(rows_s)), rs.randint(NI, size=len(rows_s))) for _ in range(3)]
    assert any((rows_i[n] == rows_i[p]).sum() > 100 for p, n in draws)
    hyper = (0.05, 0.01, 0.02)
    U1, I1, st1 = _device_fit(rows_s, rows_i, S, NI, F, draws, U0, I0, bI, hyper, max_warps=1)
    U2, I2, st2 = _device_fit(rows_s, rows_i, S, NI, F, draws, U0, I0, bI, hyper)
    U3, I3, st3 = _device_fit(rows_s, rows_i, S, NI, F, draws, U0, I0, bI, hyper)
    assert U1.tobytes() == U2.tobytes() == U3.tobytes() and I1.tobytes() == I2.tobytes() == I3.tobytes()
    assert [s[:2] for s in st1] == [s[:2] for s in st2] == [s[:2] for s in st3]
    if F in (7, 130):                                   # the oracle's per-event loop; its level is the longest chain
        Uo, Io, means, levels = bpo.fit(rows_s, rows_i, U0, I0, bI, draws, *hyper)
        eu, ei = np.abs(U2 - Uo).max(), np.abs(I2 - Io).max()
        print('F=%d: worst |U - oracle| %.3g, |I - oracle| %.3g' % (F, eu, ei))
        assert eu <= 1e-12 and ei <= 1e-12
        assert [s[1] for s in st2] == levels
        np.testing.assert_allclose([s[0] for s in st2], means, rtol=1e-12, atol=0)


@pytest.mark.parametrize('case,tag', [(c, t) for c in ('int_ids', 'str_messy') for t in ('f16_uniform', 'f100_normal')])
def test_class_fit_against_the_oracle_and_the_reference(case, tag):
    import baselines
    from test_host_bpr import PARAMS
    g = dict(np.load(os.path.join(GOLDEN, 'bpr_%s_%s.npz' % (case, tag))))
    tr = pd.DataFrame({'SessionId': g['train_sid'], 'ItemId': g['train_iid'], 'Time': g['train_time']})
    np.random.seed(int(g['seed']))
    m = baselines.BPR(**PARAMS[tag])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        m.fit(tr)
    er = max(np.abs(m.U - g['U']).max(), np.abs(m.I - g['I']).max())
    # the oracle on the same inputs: the reference's merge, init and draws
    np.random.seed(int(g['seed']))
    o = baselines.BPR(**PARAMS[tag])
    o.n_items, o.n_sessions = m.n_items, m.n_sessions
    o.init(None)
    merged = pd.merge(tr, pd.DataFrame({'ItemId': m.itemidmap.index.values, 'ItemIdx': np.arange(m.n_items)}), on='ItemId', how='inner')
    merged = pd.merge(merged, pd.DataFrame({'SessionId': tr.SessionId.unique(), 'SessionIdx': np.arange(m.n_sessions)}), on='SessionId', how='inner')
    draws = [bpo.iteration_draws(len(merged), m.n_items) for _ in range(3)]
    Uo, Io, means, levels = bpo.fit(merged.SessionIdx.values, merged.ItemIdx.values, o.U, o.I, o.bI, draws, o.learning_rate,
                                    o.lambda_session, o.lambda_item)
    eo = max(np.abs(m.U - Uo).max(), np.abs(m.I - Io).max())
    print('%s %s: worst |device - oracle| %.3g, |device - reference| %.3g' % (case, tag, eo, er))
    assert eo <= 1e-12 and er <= 1e-10
    assert [s[1] for s in m.fit_stats] == levels
    np.testing.assert_allclose([float(x.split()[1]) for x in buf.getvalue().splitlines()], g['means'], rtol=0, atol=1e-12)


@pytest.fixture(scope='module')
def small():
    n, F = 300, 24
    rs = np.random.RandomState(4)
    I, bI = rs.randn(n, F) * 0.3, rs.randn(n) * 0.05
    I[5] = I[6]; bI[5] = bI[6]                                    # an exact tie between two items
    dev = _lib.Baselines('bpr', n, F)
    dev.bpr_import(I, bI)
    items, off, _, _ = make_session_arrays(n, 900, seed=7, max_len=30)
    items = items.astype(np.int32)
    rep = np.flatnonzero(rs.rand(len(items)) < 0.25)
    items[rep[rep > 0]] = items[rep[rep > 0] - 1]
    nh = np.minimum(rs.randint(0, 4, len(off) - 1), np.diff(off)).astype(np.int32)
    return dev, I, bI, items, off.astype(np.int64), nh


def test_event_counts_sums_and_lists_equal_the_oracle(small):
    dev, I, bI, items, off, nh = small
    n = I.shape[0]
    cand = np.r_[np.arange(0, n, 4), [0, 0, 8]]
    cand = cand[cand != items[off[0] + 1]]                        # an unlisted target
    cuts = [1, 5, 20]
    for mode, cd, ex, hist in itertools.product(['standard', 'conservative', 'median', 'tiebreaking'], [None, cand], [False, True], [None, nh]):
        what = (mode, cd is not None, ex, hist is not None)
        wc, wi, ws = bpo.rank_events(I, bI, items, off, hist, mode, cd, ex, k=7)
        rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, hist, cuts, bo.MODES[mode], cd, ex, k=7)
        rec0, mrr0, _, cnt0, _, _ = dev.evaluate(items, off, hist, cuts, bo.MODES[mode], cd, ex, k=0)
        assert nc == len(wc), what
        np.testing.assert_array_equal(cnt, wc, err_msg=str(what))
        np.testing.assert_array_equal(cnt0, wc, err_msg=str(what))
        np.testing.assert_array_equal(ti, wi, err_msg=str(what))
        np.testing.assert_array_equal(ts, ws, err_msg=str(what))
        hits, rrs = bo.sums(wc, mode, cuts)
        assert list(rec) == hits and list(rec0) == hits, what
        for a, b in zip(list(mrr) + list(mrr0), rrs + rrs):
            assert a == b or abs(a - b) <= 1e-12 * abs(b), (what, a, b)
        if ex:
            assert (cnt[:, 0] < 0).any(), what


def test_lists_padded_when_fewer_than_k_items_are_eligible(small):
    dev, I, bI, items, off, nh = small
    cand = np.r_[np.bincount(items, minlength=I.shape[0]).argsort()[-4:]]
    cand = np.r_[cand, cand[0]]
    rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, None, [2], 0, cand, True, k=4)
    wc, wi, ws = bpo.rank_events(I, bI, items, off, None, 'standard', cand, True, k=4)
    assert (ti == -1).any() and np.isnan(ts[ti == -1]).all() and not np.isnan(ts[ti >= 0]).any()
    np.testing.assert_array_equal(cnt, wc)
    np.testing.assert_array_equal(ti, wi)
    np.testing.assert_array_equal(ts, ws)


def test_172k_items_over_several_blocks():
    """172,000 items, k = 5: 390 events per block of list scratch, sessions across block boundaries; k = 1024 once"""
    n, F = 172000, 8
    rs = np.random.RandomState(9)
    I, bI = rs.randn(n, F) * 0.2, np.zeros(n)
    dev = _lib.Baselines('bpr', n, F)
    dev.bpr_import(I, bI)
    items, off, _, _ = make_session_arrays(500, 800, seed=3, max_len=60)
    items = (items * 343 + 1).astype(np.int32)                    # spread over the catalogue
    items[::7] = items[::7] % 50                                  # repeats of a few items
    off = off.astype(np.int64)
    nh = np.minimum(rs.randint(0, 3, len(off) - 1), np.diff(off)).astype(np.int32)
    for mode, ex, k in (('standard', True, 5), ('tiebreaking', False, 5), ('median', False, 1024)):
        wc, wi, ws = bpo.rank_events(I, bI, items, off, nh, mode, None, ex, k=k)
        rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, nh, [20], bo.MODES[mode], None, ex, k=k)
        assert len(wc) > 400
        np.testing.assert_array_equal(cnt, wc)
        np.testing.assert_array_equal(ti, wi)
        np.testing.assert_array_equal(ts, ws)


def test_begin_refuses_fewer_rows_than_items_in_the_library():
    """the C entry point itself, below the binding's check: 4 rows, 5 items, so a negative draw could name a missing row"""
    import ctypes as C
    dev = _lib.Baselines('bpr', 5, 3)
    rs, ri = np.array([0, 1, 0, 1], np.int32), np.array([0, 1, 2, 3], np.int32)
    U, I, bI = np.zeros((2, 3)), np.zeros((5, 3)), np.zeros(5)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert dev.lib.g4r_bl_bpr_begin(dev.h, p(rs), p(ri), 4, 2, p(U), p(I), p(bI)) == _lib.G4R_ERR_INVALID
    assert b'n_rows >= n_items' in dev.lib.g4r_bl_last_error(dev.h)
    rs, ri = np.r_[rs, 1].astype(np.int32), np.r_[ri, 4].astype(np.int32)
    assert dev.lib.g4r_bl_bpr_begin(dev.h, p(rs), p(ri), 5, 2, p(U), p(I), p(bI)) == _lib.G4R_OK


def test_evaluate_through_the_python_surface():
    import baselines
    import evaluation
    train = make_sessions(n_items=200, n_events=6000, seed=1)
    test = make_sessions(n_items=200, n_events=1500, seed=2)
    test['SessionId'] += 100000
    np.random.seed(0)
    m = baselines.BPR(n_factors=32, n_iterations=2)
    with contextlib.redirect_stdout(io.StringIO()):
        m.fit(train.copy())
    with pytest.raises(RuntimeError):                  # fit ended: U and the per-row buffers are off the device
        m._dev.bpr_export()
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(m, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
        rec = evaluation.evaluate_gpu(m, test.copy(), cut_off=[5, 20], mode='median', exclude_seen=True)
    assert rec == (res['recall'], res['mrr'])
    import pickle
    m2 = pickle.loads(pickle.dumps(m))
    with contextlib.redirect_stdout(io.StringIO()):
        res2 = evaluation.evaluate_events(m2, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
    pd.testing.assert_frame_equal(res['events'], res2['events'])
    assert res['topk_scores'].tobytes() == res2['topk_scores'].tobytes()


def test_other_evaluations_are_untouched_by_bpr_calls():
    import baselines
    import evaluation
    import gru4rec
    train = make_sessions(n_items=150, n_events=4000, seed=3)
    test = make_sessions(n_items=150, n_events=1000, seed=4)
    test['SessionId'] += 100000
    gru = gru4rec.GRU4Rec(layers=[32], batch_size=32, n_epochs=1, n_sample=64, loss='bpr-max', final_act='elu-0.5')
    knn = baselines.ItemKNN(n_sims=20)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
        knn.fit(train.copy())
        before = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in (gru, knn)]
        np.random.seed(2)
        bpr = baselines.BPR(n_factors=16, n_iterations=2)
        bpr.fit(train.copy())
        evaluation.evaluate_events(bpr, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5, exclude_seen=True)
        after = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in (gru, knn)]
    for b, a in zip(before, after):
        pd.testing.assert_frame_equal(b['events'], a['events'])
        assert b['recall'] == a['recall'] and b['mrr'] == a['mrr']
        assert b['topk_scores'].tobytes() == a['topk_scores'].tobytes()
