"""Session-based kNN on the device (DESIGN §3o): per-event counts, top-k items and float64 top-k scores exactly equal to
oracle/sknn_oracle.py, and Recall / MRR sums within 1e-12, for both similarities in all four modes x {plain, items= with duplicates,
exclude_seen, history}; a stress set (200,000 training sessions, one item in about 50,000 of them, many equal session times,
300-event histories of distinct items, sample_size 8192, k 1024) checked on 300 events per similarity; a 172,000-item catalogue
(the zero-score closed form, zero-score targets); padded lists; bitwise repeatability; and GRU4Rec / ItemKNN evaluations
unchanged by SessionKNN calls in between."""
import contextlib
import io
import itertools
import pickle

import numpy as np
import pandas as pd
import pytest

import baselines_oracle as bo
import sknn_oracle as sko
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions

pytestmark = pytest.mark.gpu


def _device(ix, k, sample_size, similarity):
    off, items, rank = ix.csr()
    dev = _lib.Baselines('sknn', ix.n_items, k)
    dev.sknn_fit(off, items, rank, sample_size, similarity)
    return dev


def _check(dev, ix, k_nb, S, sim, items, off, hist, mode, cand, ex, k, cuts=(1, 5, 20), only=None):
    what = (sim, mode, cand is not None, ex, hist is not None, k)
    rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, hist, list(cuts), bo.MODES[mode], cand, ex, k=k)
    wc, wi, ws = sko.rank_events(ix, k_nb, S, sim, items, off, hist, mode, cand, ex, k, only=only)
    sel = slice(None) if only is None else np.asarray(only)
    np.testing.assert_array_equal(cnt[sel], wc, err_msg=str(what))
    if k:
        np.testing.assert_array_equal(ti[sel], wi, err_msg=str(what))
        np.testing.assert_array_equal(ts[sel], ws, err_msg=str(what))
    if only is None:
        hits, rrs = bo.sums(wc, mode, list(cuts))
        assert list(rec) == hits, what
        for a, b in zip(mrr, rrs):
            assert a == b or abs(a - b) <= 1e-12 * abs(b), (what, a, b)
    return cnt, ti, ts


@pytest.fixture(scope='module')
def small():
    n = 300
    tr_items, tr_off, _, _ = make_session_arrays(n, 6000, seed=5, max_len=12)
    rs = np.random.RandomState(2)
    sess = np.repeat(np.arange(len(tr_off) - 1), np.diff(tr_off))
    times = rs.randint(0, 40, len(tr_off) - 1)[sess]                     # many equal session times
    ix = sko.Index(sess, tr_items, times, n)
    items, off, _, _ = make_session_arrays(n, 700, seed=7, max_len=25)
    items = items.astype(np.int32)
    rep = np.flatnonzero(rs.rand(len(items)) < 0.25)
    items[rep[rep > 0]] = items[rep[rep > 0] - 1]                         # repeated inputs
    nh = np.minimum(rs.randint(0, 4, len(off) - 1), np.diff(off)).astype(np.int32)
    return ix, items, off.astype(np.int64), nh


@pytest.mark.parametrize('similarity', ['cosine', 'vector'])
def test_counts_sums_and_lists_equal_the_oracle(small, similarity):
    ix, items, off, nh = small
    k_nb, S = 20, 60
    dev = _device(ix, k_nb, S, similarity)
    n = ix.n_items
    cand = np.r_[np.arange(0, n, 3), [0, 0, 9]]
    cand = cand[cand != items[off[0] + 1]]                                # an unlisted target
    for mode, (cd, ex, hist) in itertools.product(['standard', 'conservative', 'median', 'tiebreaking'],
                                                  [(None, False, None), (cand, False, None), (None, True, None), (None, False, nh)]):
        cnt = _check(dev, ix, k_nb, S, similarity, items, off, hist, mode, cd, ex, 7)[0]
        cnt0 = dev.evaluate(items, off, hist, [5], bo.MODES[mode], cd, ex, k=0)[3]
        np.testing.assert_array_equal(cnt0, cnt)
        if ex:
            assert (cnt[:, 0] < 0).any()


def test_lists_padded_when_fewer_than_k_items_are_eligible(small):
    ix, items, off, nh = small
    dev = _device(ix, 10, 50, 'vector')
    cand = np.bincount(items, minlength=ix.n_items).argsort()[-4:]
    cand = np.r_[cand, cand[0]]
    cnt, ti, ts = _check(dev, ix, 10, 50, 'vector', items, off, None, 'standard', cand, True, 4)
    assert (ti == -1).any() and np.isnan(ts[ti == -1]).all() and not np.isnan(ts[ti >= 0]).any()


def test_two_evaluations_are_bitwise_equal(small):
    ix, items, off, nh = small
    dev = _device(ix, 20, 100, 'cosine')
    a = dev.evaluate(items, off, nh, [5, 20], 3, None, True, k=9)
    b = dev.evaluate(items, off, nh, [5, 20], 3, None, True, k=9)
    for x, y in zip(a, b):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()


@pytest.fixture(scope='module')
def stress():
    rs = np.random.RandomState(11)
    n_items, S = 20000, 200000
    lens = rs.randint(2, 7, S)
    sess = np.repeat(np.arange(S), lens)
    items = rs.randint(1, n_items, len(sess))
    hot = np.flatnonzero(rs.rand(S) < 0.25)                               # item 0 in about 50,000 sessions
    items[np.r_[0, np.cumsum(lens)[:-1]][hot]] = 0
    times = rs.randint(0, 60, S)[sess]                                     # many sessions share T
    ix = sko.Index(sess, items, times, n_items)
    n_test, H, L = 25, 300, 13
    seqs = []
    for q in range(n_test):
        h = rs.choice(np.arange(1, n_items), H, replace=False)
        h[rs.randint(H)] = 0
        seqs.append(np.r_[h, rs.randint(0, n_items, L)])
    t_items = np.concatenate(seqs).astype(np.int32)
    t_off = np.r_[0, np.cumsum([len(x) for x in seqs])].astype(np.int64)
    nh = np.full(n_test, H, np.int32)
    return ix, t_items, t_off, nh


@pytest.mark.parametrize('similarity', ['cosine', 'vector'])
def test_stress_sample_8192_k_1024_long_histories(stress, similarity):
    ix, items, off, nh = stress
    assert np.diff(ix.post.indptr)[0] > 45000
    dev = _device(ix, 1024, 8192, similarity)
    n_ev = int((np.diff(off) - nh).sum())
    only = np.sort(np.random.RandomState(3).choice(n_ev, 300, replace=False))
    cnt, ti, ts = _check(dev, ix, 1024, 8192, similarity, items, off, nh, 'median', None, False, 5, only=only)
    assert len(cnt) == n_ev


def test_172k_catalogue_zero_score_targets():
    n = 172000
    tr_items, tr_off, _, _ = make_session_arrays(n, 420000, seed=3, max_len=10)
    sess = np.repeat(np.arange(len(tr_off) - 1), np.diff(tr_off))
    ix = sko.Index(sess, tr_items, sess // 50, n)
    rs = np.random.RandomState(4)
    items, off, _, _ = make_session_arrays(300, 900, seed=8, max_len=12)
    items = (items * 571 + 5).astype(np.int32)                             # spread over the catalogue
    items[::5] = rs.randint(0, 30, len(items[::5]))                        # repeats of popular items
    off = off.astype(np.int64)
    dev = _device(ix, 50, 500, 'cosine')
    zero_targets = 0
    for mode, k in (('conservative', 0), ('median', 5)):
        cnt, ti, ts = _check(dev, ix, 50, 500, 'cosine', items, off, None, mode, None, False, k)
        zero_targets = int((cnt[:, 1] > 100000).sum())
        assert zero_targets > 10, mode
    dev = _device(ix, 50, 500, 'vector')
    _check(dev, ix, 50, 500, 'vector', items, off, None, 'conservative', None, True, 3)


def test_class_evaluation_pickle_and_other_models_untouched():
    import baselines
    import evaluation
    import gru4rec
    train = make_sessions(n_items=150, n_events=4000, seed=3)
    test = make_sessions(n_items=150, n_events=1000, seed=4)
    test['SessionId'] += 100000
    test = test[test.ItemId.isin(train.ItemId.unique())]
    gru = gru4rec.GRU4Rec(layers=[32], batch_size=32, n_epochs=1, n_sample=64, loss='bpr-max', final_act='elu-0.5')
    knn = baselines.ItemKNN(n_sims=20)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
        knn.fit(train.copy())
        before = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in (gru, knn)]
        sk = baselines.SessionKNN(k=30, sample_size=200, similarity='vector')
        sk.fit(train.copy())
        res = evaluation.evaluate_events(sk, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
        rec = evaluation.evaluate_gpu(sk, test.copy(), cut_off=[5, 20], mode='median', exclude_seen=True)
        after = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in (gru, knn)]
    for b, a in zip(before, after):
        pd.testing.assert_frame_equal(b['events'], a['events'])
        assert b['recall'] == a['recall'] and b['mrr'] == a['mrr']
        assert b['topk_scores'].tobytes() == a['topk_scores'].tobytes()
    assert rec == (res['recall'], res['mrr'])
    # the device's top-k list of the first event equals predict_next's host scores
    first = test.sort_values(['SessionId', 'Time']).iloc[0]
    ids = sk.itemidmap.index.values
    host = sk.predict_next(first.SessionId, first.ItemId, ids).values
    top = res['topk_items'][0]
    assert np.array_equal(res['topk_scores'][0], host[sk.itemidmap[top].values])
    sk2 = pickle.loads(pickle.dumps(sk))
    with contextlib.redirect_stdout(io.StringIO()):
        res2 = evaluation.evaluate_events(sk2, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
    pd.testing.assert_frame_equal(res['events'], res2['events'])
    assert res['topk_scores'].tobytes() == res2['topk_scores'].tobytes()
