"""The session baselines on the device (DESIGN §3j) against oracle/baselines_oracle.py and the reference's recorded runs: ItemKNN
rows (indices and float64 sims bitwise; the device and the oracle share the (sim desc, index asc) order, so the rows are equal
entry for entry) at catalogue sizes up to 172,000 items, with a heavy item, n_sims past the positive count and n_sims = 1, every
alpha / lmbd pair; determinism; the per-event counts, sums and top-k lists of all three baselines in every combination of mode,
items=, exclude_seen and history; and a GRU4Rec evaluation left bitwise unchanged by baseline calls in the same process."""
import contextlib
import io
import itertools

import numpy as np
import pandas as pd
import pytest

import baselines_oracle as bo
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions

pytestmark = pytest.mark.gpu


def _knn_device(off, items, n_items, n_sims, lmbd, alpha):
    dev = _lib.Baselines('itemknn', n_items, n_sims)
    a, b = bo.norm_factors(np.bincount(items, minlength=n_items), lmbd, alpha)
    stats = dev.knn_fit(off, items, a, b)
    return dev, dev.rows_export(), stats


def _check_rows(rows, off, items, n_items, n_sims, lmbd, alpha, sample=None):
    idx, sim, ln = rows
    want = bo.knn_rows(off, items, n_items, n_sims, lmbd, alpha, rows=sample)
    for i, (j, v) in want.items():
        assert ln[i] == len(j), (i, ln[i], len(j))
        np.testing.assert_array_equal(idx[i, :ln[i]], j)
        np.testing.assert_array_equal(sim[i, :ln[i]], v)            # float64, bitwise
        assert np.all(idx[i, ln[i]:] == -1) and np.all(sim[i, ln[i]:] == 0.0)


@pytest.mark.parametrize('lmbd,alpha', list(itertools.product([0, 20], [0.0, 0.5, 1.0])))
@pytest.mark.parametrize('n_sims', [1, 20, 500])
def test_knn_rows_small_catalogue(n_sims, lmbd, alpha):
    """300 items with repeated items inside sessions: n_sims = 500 keeps every positive sim of every row"""
    items, off, _, _ = make_session_arrays(300, 6000, seed=5, max_len=30)
    rs = np.random.RandomState(1)
    rep = np.flatnonzero(rs.rand(len(items)) < 0.2)
    items[rep[rep > 0]] = items[rep[rep > 0] - 1]
    items = items.astype(np.int32)
    _, rows, _ = _knn_device(off, items, 300, n_sims, lmbd, alpha)
    _check_rows(rows, off, items, 300, n_sims, lmbd, alpha)


def test_knn_rows_long_sessions():
    """sessions of 1 to 6,000 events with many repeats: the warp sort (<= 64 events) and the CTA sort of longer sessions"""
    rs = np.random.RandomState(8)
    lens = np.r_[rs.randint(1, 70, 400), 65, 128, 129, 1000, 4097, 6000]
    items = np.concatenate([rs.randint(0, 200 if l > 500 else 400, l) for l in lens]).astype(np.int32)
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    dev, rows, (pairs, scratch, ms) = _knn_device(off, items, 400, 50, 20, 0.5)
    assert pairs == sum(int(l) * len(np.unique(items[off[s]:off[s + 1]])) for s, l in enumerate(lens))
    _check_rows(rows, off, items, 400, 50, 20, 0.5)


def test_rows_import_refuses_bad_rows():
    n, k = 10, 3
    dev = _lib.Baselines('itemknn', n, k)
    idx = np.full((n, k), -1, np.int32); sim = np.zeros((n, k)); ln = np.zeros(n, np.int32)
    idx[0, :2] = [4, 4]; sim[0, :2] = [0.5, 0.25]; ln[0] = 2                 # falling sims, the same item twice
    with pytest.raises(ValueError):
        dev.rows_import(idx, sim, ln)
    idx[0, 1] = 5
    dev.rows_import(idx, sim, ln)
    np.testing.assert_array_equal(dev.rows_export()[0], idx)


def test_knn_rows_rsc15_shape_heavy_item_and_determinism():
    """37,483 items, sessions up to 200 events, item 7 in more than half of the sessions: 500 sampled rows (the heaviest
    included) equal the oracle; a second fit is bitwise equal"""
    n = 37483
    items, off, _, _ = make_session_arrays(n, 600000, seed=2, max_len=200)
    items = items.astype(np.int32)
    rs = np.random.RandomState(3)
    heavy = rs.rand(len(off) - 1) < 0.6
    items[off[:-1][heavy]] = 7
    assert np.mean([7 in items[off[s]:off[s + 1]] for s in range(0, len(off) - 1, 50)]) > 0.5
    dev, rows, (pairs, scratch, ms) = _knn_device(off, items, n, 100, 20, 0.5)
    lens = np.diff(off)
    assert pairs == sum(int(lens[s]) * len(np.unique(items[off[s]:off[s + 1]])) for s in range(len(lens)))
    sample = np.unique(np.r_[7, rs.choice(n, 499, replace=False)])
    _check_rows(rows, off, items, n, 100, 20, 0.5, sample=sample)
    rows2 = _knn_device(off, items, n, 100, 20, 0.5)[1]
    for a, b in zip(rows, rows2):
        assert a.tobytes() == b.tobytes()


def test_knn_rows_172k_items_within_the_scratch_budget():
    n = 172000
    items, off, _, _ = make_session_arrays(n, 1500000, seed=4, max_len=50)
    items = items.astype(np.int32)
    dev, rows, (pairs, scratch, ms) = _knn_device(off, items, n, 100, 20, 0.5)
    assert scratch <= 512 << 20
    supp = np.bincount(items, minlength=n)
    rs = np.random.RandomState(0)
    sample = np.unique(np.r_[np.argmax(supp), rs.choice(n, 499, replace=False)])
    _check_rows(rows, off, items, n, 100, 20, 0.5, sample=sample)


def test_knn_rows_equal_the_reference_fixtures():
    import os
    from test_host_baselines import GOLDEN, KNN, _train_csr, _tie_aware
    for case in ('int_ids', 'str_messy'):
        g = dict(np.load(os.path.join(GOLDEN, case + '.npz')))
        off, items, n = _train_csr(g)
        for tag, (n_sims, lmbd, alpha) in KNN.items():
            idx, sim, ln = _knn_device(off, items.astype(np.int32), n, n_sims, lmbd, alpha)[1]
            for i in range(n):
                wi, ws = g[tag + '_idx'][i], g[tag + '_sim'][i]
                _tie_aware(idx[i, :ln[i]], sim[i, :ln[i]], wi[wi >= 0], ws[wi >= 0])


@pytest.fixture(scope='module')
def models():
    n = 300
    items, off, _, _ = make_session_arrays(n, 8000, seed=6, max_len=25)
    items = items.astype(np.int32)
    supp = np.bincount(items, minlength=n)
    out = {}
    dev, rows, _ = _knn_device(off, items, n, 30, 20, 0.5)
    idx, sim, ln = rows
    out['itemknn'] = (dev, (n, {i: (idx[i, :ln[i]].astype(np.int64), sim[i, :ln[i]]) for i in range(n)}))
    for kind in ('pop', 'sessionpop'):
        dev = _lib.Baselines(kind, n, 40)
        dense = bo.pop_scores(supp, 40)
        dev.set_pop(dense)
        out[kind] = (dev, dense)
    te_items, te_off, _, _ = make_session_arrays(n, 900, seed=7, max_len=30)
    te_items = te_items.astype(np.int32)
    rs = np.random.RandomState(2)
    rep = np.flatnonzero(rs.rand(len(te_items)) < 0.25)
    te_items[rep[rep > 0]] = te_items[rep[rep > 0] - 1]
    nh = np.minimum(rs.randint(0, 4, len(te_off) - 1), np.diff(te_off)).astype(np.int32)
    return out, n, te_items, te_off.astype(np.int64), nh


@pytest.mark.parametrize('kind', ['pop', 'sessionpop', 'itemknn'])
def test_event_counts_sums_and_lists_equal_the_oracle(models, kind):
    out, n, items, off, nh = models
    dev, model = out[kind]
    cand = np.r_[np.arange(0, n, 4), [0, 0, 8]]
    cand = cand[cand != items[off[0] + 1]]                        # an unlisted target
    cuts = [1, 5, 20]
    for mode, cd, ex, hist in itertools.product(['standard', 'conservative', 'median', 'tiebreaking'], [None, cand], [False, True], [None, nh]):
        rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, hist, cuts, bo.MODES[mode], cd, ex, k=7)
        wc, wi, ws = bo.rank_events(kind, model, n, items, off, hist, mode, cd, ex, k=7)
        what = (kind, mode, cd is not None, ex, hist is not None)
        assert nc == len(wc), what
        np.testing.assert_array_equal(cnt, wc, err_msg=str(what))
        np.testing.assert_array_equal(ti, wi, err_msg=str(what))
        np.testing.assert_array_equal(ts, ws, err_msg=str(what))
        hits, rrs = bo.sums(wc, mode, cuts)
        assert list(rec) == hits, what
        for a, b in zip(mrr, rrs):
            assert a == b or abs(a - b) <= 1e-12 * abs(b), (what, a, b)
        if ex:
            assert (cnt[:, 0] < 0).any(), what


@pytest.mark.parametrize('kind', ['pop', 'sessionpop', 'itemknn'])
def test_lists_padded_when_fewer_than_k_items_are_eligible(models, kind):
    """items= of 4 distinct ids (one listed twice), k = 4, exclude_seen: events whose session has input one of them get -1 / NaN"""
    out, n, items, off, nh = models
    dev, model = out[kind]
    cand = np.r_[np.bincount(items, minlength=n).argsort()[-4:], items[0]]
    cand = np.r_[cand[:4], cand[0]]
    rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, None, [2], 0, cand, True, k=4)
    wc, wi, ws = bo.rank_events(kind, model, n, items, off, None, 'standard', cand, True, k=4)
    assert (ti == -1).any() and np.isnan(ts[ti == -1]).all() and not np.isnan(ts[ti >= 0]).any()
    np.testing.assert_array_equal(cnt, wc)
    np.testing.assert_array_equal(ti, wi)
    np.testing.assert_array_equal(ts, ws)


def test_evaluate_through_the_python_surface_and_batch_size():
    import baselines
    import evaluation
    train = make_sessions(n_items=200, n_events=6000, seed=1)
    test = make_sessions(n_items=200, n_events=1500, seed=2)
    test['SessionId'] += 100000
    for m in (baselines.Pop(top_n=30), baselines.SessionPop(top_n=30), baselines.ItemKNN(n_sims=50)):
        m.fit(train.copy())
        with contextlib.redirect_stdout(io.StringIO()):
            res = [evaluation.evaluate_events(m, test.copy(), cut_off=[5, 20], batch_size=bs, mode='median', k=10, exclude_seen=True)
                   for bs in (1, 100, 512)]
            rec = evaluation.evaluate_gpu(m, test.copy(), cut_off=[5, 20], mode='median', exclude_seen=True)
        for r in res[1:]:
            pd.testing.assert_frame_equal(r['events'], res[0]['events'])
            np.testing.assert_array_equal(r['topk_scores'], res[0]['topk_scores'])
        assert rec == (res[0]['recall'], res[0]['mrr'])
        assert res[0]['topk_scores'].dtype == np.float64


def test_gru_evaluation_is_untouched_by_baseline_calls():
    import baselines
    import evaluation
    import gru4rec
    train = make_sessions(n_items=150, n_events=4000, seed=3)
    test = make_sessions(n_items=150, n_events=1000, seed=4)
    test['SessionId'] += 100000
    gru = gru4rec.GRU4Rec(layers=[32], batch_size=32, n_epochs=1, n_sample=64, loss='bpr-max', final_act='elu-0.5')
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
        before = evaluation.evaluate_events(gru, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5)
        knn = baselines.ItemKNN(n_sims=20)
        knn.fit(train.copy())
        evaluation.evaluate_events(knn, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5)
        after = evaluation.evaluate_events(gru, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5)
    pd.testing.assert_frame_equal(before['events'], after['events'])
    assert before['recall'] == after['recall'] and before['mrr'] == after['mrr']
    assert before['topk_scores'].tobytes() == after['topk_scores'].tobytes()
