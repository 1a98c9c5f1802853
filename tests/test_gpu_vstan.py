"""VSTAN-style session kNN on the device (DESIGN §3r): per-event counts, top-k items and float64 top-k scores exactly equal to
tests/vstan_oracle.py, and Recall / MRR sums within 1e-12, for both similarities with finite lambdas and lambda_idf > 0 in all four
modes x {plain, items= with duplicates and an unlisted target, exclude_seen, history}; each addition alone; the reduction setting
bitwise equal to the device STAN; an underflow set (each item listed once); STAN's stress set (200,000 sessions, sample_size 8192,
k 1024, 300-event histories) on 300 events; a 172,000-item catalogue; the W4-table and set-before-evaluate refusals; bitwise
repeatability; the Python surface with pickles; and SessionKNN / STAN / GRU4Rec evaluations unchanged by VSTAN calls in between."""
import contextlib
import io
import itertools
import pickle

import numpy as np
import pandas as pd
import pytest

import baselines_oracle as bo
import vstan_oracle as vso
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions

pytestmark = pytest.mark.gpu
INF = float('inf')
LAM = dict(lambda_spw=1.02, lambda_snh=10.0, lambda_inh=2.05)


def _fit(kind, ix, k, sample_size, n_w1):
    off, items, rank = ix.csr()
    pos = np.concatenate([[ix.q[rank[s]][j] for j in items[off[s]:off[s + 1]].tolist()] for s in range(len(rank))]).astype(np.int32)
    dev = _lib.Baselines(kind, ix.n_items, k)
    dev.stan_fit(off, items, pos, rank, ix.w2[rank], ix.w3, sample_size)
    dev.stan_set_w1(ix.w1(n_w1))
    return dev


def _device(ix, k, sample_size, n_w1, n_w4=None):
    dev = _fit('vstan', ix, k, sample_size, n_w1)
    dev.vstan_set(ix.similarity, ix.f, ix.w4(n_w1 if n_w4 is None else n_w4))
    return dev


def _check(dev, ix, k_nb, S, items, off, hist, mode, cand, ex, k, cuts=(1, 5, 20), only=None):
    what = (ix.similarity, mode, cand is not None, ex, hist is not None, k)
    rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, hist, list(cuts), bo.MODES[mode], cand, ex, k=k)
    wc, wi, ws = vso.rank_events(ix, k_nb, S, items, off, hist, mode, cand, ex, k, only=only)
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


def _small_train(n=300, seed=5):
    tr_items, tr_off, _, _ = make_session_arrays(n, 6000, seed=seed, max_len=12)
    rs = np.random.RandomState(2)
    sess = np.repeat(np.arange(len(tr_off) - 1), np.diff(tr_off))
    times = rs.randint(0, 40, len(tr_off) - 1)[sess] + rs.randint(0, 3, len(sess))   # ties across and inside sessions
    tr_items = tr_items.copy()
    rep = np.flatnonzero(rs.rand(len(tr_items)) < 0.15)
    tr_items[rep[rep > 0]] = tr_items[rep[rep > 0] - 1]                      # repeated training items
    return sess, tr_items, times


@pytest.fixture(scope='module')
def small():
    n = 300
    sess, tr_items, times = _small_train(n)
    rs = np.random.RandomState(3)
    items, off, _, _ = make_session_arrays(n, 700, seed=7, max_len=25)
    items = items.astype(np.int32)
    rep = np.flatnonzero(rs.rand(len(items)) < 0.25)
    items[rep[rep > 0]] = items[rep[rep > 0] - 1]                         # repeated inputs
    nh = np.minimum(rs.randint(0, 4, len(off) - 1), np.diff(off)).astype(np.int32)
    return (sess, tr_items, times, n), items, off.astype(np.int64), nh


@pytest.mark.parametrize('similarity', ['cosine', 'vector'])
def test_counts_sums_and_lists_equal_the_oracle(small, similarity):
    (sess, tr_items, times, n), items, off, nh = small
    ix = vso.Index(sess, tr_items, times, n, similarity, lambda_ipw=1.02, lambda_idf=0.7, **LAM)
    k_nb, S = 20, 60
    dev = _device(ix, k_nb, S, int(np.diff(off).max()))
    cand = np.r_[np.arange(0, n, 3), [0, 0, 9]]
    cand = cand[cand != items[off[0] + 1]]                                # an unlisted target
    for mode, (cd, ex, hist) in itertools.product(['standard', 'conservative', 'median', 'tiebreaking'],
                                                  [(None, False, None), (cand, False, None), (None, True, None), (None, False, nh)]):
        cnt = _check(dev, ix, k_nb, S, items, off, hist, mode, cd, ex, 7)[0]
        cnt0 = dev.evaluate(items, off, hist, [5], bo.MODES[mode], cd, ex, k=0)[3]
        np.testing.assert_array_equal(cnt0, cnt)
        if ex:
            assert (cnt[:, 0] < 0).any()


@pytest.mark.parametrize('extra', [dict(similarity='vector'), dict(lambda_ipw=0.8), dict(lambda_idf=2.0)])
def test_each_addition_alone_equals_the_oracle(small, extra):
    (sess, tr_items, times, n), items, off, nh = small
    ix = vso.Index(sess, tr_items, times, n, **dict(LAM, **extra))
    dev = _device(ix, 15, 50, int(np.diff(off).max()))
    for mode, (ex, hist) in (('standard', (False, None)), ('median', (True, nh))):
        _check(dev, ix, 15, 50, items, off, hist, mode, None, ex, 6)


def test_reduction_is_bitwise_the_device_stan(small):
    (sess, tr_items, times, n), items, off, nh = small
    ix = vso.Index(sess, tr_items, times, n, 'cosine', lambda_ipw=INF, lambda_idf=0.0, **LAM)
    assert (ix.f == 1.0).all() and (ix.w4(5) == 1.0).all()
    L = int(np.diff(off).max())
    dev = _device(ix, 20, 60, L)
    st = _fit('stan', ix, 20, 60, L)
    cand = np.r_[np.arange(0, n, 4), [1, 1]]
    for mode, (cd, ex, hist) in itertools.product(['standard', 'conservative', 'median', 'tiebreaking'],
                                                  [(None, False, None), (cand, True, nh)]):
        a = dev.evaluate(items, off, hist, [1, 5, 20], bo.MODES[mode], cd, ex, k=9)
        b = st.evaluate(items, off, hist, [1, 5, 20], bo.MODES[mode], cd, ex, k=9)
        for x, y in zip(a, b):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (mode, cd is not None)


def test_underflow_exact_zeros_listed_once_by_index(small):
    (sess, tr_items, times, n), items, off, nh = small
    ix = vso.Index(sess, tr_items, times, n, 'vector', lambda_spw=1.02, lambda_snh=1e-300, lambda_inh=1e-300, lambda_ipw=1e-300,
                   lambda_idf=0.5)
    assert ix.w4(2)[1] == 0.0 and ix.w3[1] == 0.0
    dev = _device(ix, 20, 60, int(np.diff(off).max()))
    for mode, ex in (('conservative', False), ('median', True)):
        cnt, ti, ts = _check(dev, ix, 20, 60, items, off, None, mode, None, ex, 12)
        for row_i, row_s in zip(ti, ts):
            live = row_i[row_i >= 0]
            assert len(np.unique(live)) == len(live)
            z = row_s[row_i >= 0] == 0.0
            assert (np.diff(live[z]) > 0).all() and not (row_s[row_i >= 0][~z] <= 0.0).any()
    zero_scored = 0
    for p in range(0, 40):                                                # zero-score items the neighbours do hold
        s = vso.scores(ix, items[:p + 1], 20, 60)
        zero_scored += int(((s == 0.0) & (ix.qm[vso.neighbours(ix, items[:p + 1], 20, 60)[0]].getnnz(axis=0) > 0)).sum())
    assert zero_scored > 0


def test_refusals_w4_table_and_evaluate_before_set(small):
    (sess, tr_items, times, n), items, off, nh = small
    ix = vso.Index(sess, tr_items, times, n, 'vector', lambda_ipw=1.02, lambda_idf=0.7, **LAM)
    L = int(np.diff(off).max())
    dev = _fit('vstan', ix, 10, 50, L)
    with pytest.raises(RuntimeError, match='vstan_set'):                  # G4R_ERR_STATE
        dev.evaluate(items, off, None, [5], 0)
    dev.vstan_set('vector', ix.f, ix.w4(L - 2))
    with pytest.raises(ValueError, match='W4'):
        dev.evaluate(items, off, None, [5], 0)
    dev.vstan_set('vector', ix.f, ix.w4(L - 1))                           # the longest prefix is L - 1
    _check(dev, ix, 10, 50, items, off, None, 'standard', None, False, 3)
    a = dev.evaluate(items, off, nh, [5, 20], 3, None, True, k=9)
    b = dev.evaluate(items, off, nh, [5, 20], 3, None, True, k=9)
    for x, y in zip(a, b):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    o, it, rank = ix.csr()                                                # a fit clears the settings
    pos = np.concatenate([[ix.q[rank[s]][j] for j in it[o[s]:o[s + 1]].tolist()] for s in range(len(rank))]).astype(np.int32)
    dev.stan_fit(o, it, pos, rank, ix.w2[rank], ix.w3, 50)
    with pytest.raises(RuntimeError, match='vstan_set'):
        dev.evaluate(items, off, None, [5], 0)


@pytest.fixture(scope='module')
def stress():
    rs = np.random.RandomState(11)
    n_items, S = 20000, 200000
    lens = rs.randint(2, 7, S)
    sess = np.repeat(np.arange(S), lens)
    items = rs.randint(1, n_items, len(sess))
    hot = np.flatnonzero(rs.rand(S) < 0.25)                               # item 0 in about 50,000 sessions
    items[np.r_[0, np.cumsum(lens)[:-1]][hot]] = 0
    times = rs.randint(0, 60, S)[sess] * 100 + rs.randint(0, 3, len(sess))   # many sessions share T; ties inside sessions
    ix = vso.Index(sess, items, times, n_items, 'vector', lambda_spw=1.02, lambda_snh=2000.0, lambda_inh=2.05, lambda_ipw=1.02,
                   lambda_idf=1.0)
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


def test_stress_sample_8192_k_1024_long_histories(stress):
    ix, items, off, nh = stress
    assert np.diff(ix.post.indptr)[0] > 45000
    dev = _device(ix, 1024, 8192, int(np.diff(off).max()))
    n_ev = int((np.diff(off) - nh).sum())
    only = np.sort(np.random.RandomState(3).choice(n_ev, 300, replace=False))
    cnt, ti, ts = _check(dev, ix, 1024, 8192, items, off, nh, 'median', None, False, 5, only=only)
    assert len(cnt) == n_ev


def test_172k_catalogue_zero_score_targets():
    n = 172000
    tr_items, tr_off, _, _ = make_session_arrays(n, 420000, seed=3, max_len=10)
    sess = np.repeat(np.arange(len(tr_off) - 1), np.diff(tr_off))
    ix = vso.Index(sess, tr_items, sess // 50, n, 'cosine', lambda_spw=1.02, lambda_snh=5000.0, lambda_inh=2.05, lambda_ipw=1.02,
                   lambda_idf=1.0)
    rs = np.random.RandomState(4)
    items, off, _, _ = make_session_arrays(300, 900, seed=8, max_len=12)
    items = (items * 571 + 5).astype(np.int32)                             # spread over the catalogue
    items[::5] = rs.randint(0, 30, len(items[::5]))                        # repeats of popular items
    off = off.astype(np.int64)
    dev = _device(ix, 50, 500, int(np.diff(off).max()))
    for mode, k in (('conservative', 0), ('median', 5)):
        cnt, ti, ts = _check(dev, ix, 50, 500, items, off, None, mode, None, False, k)
        assert int((cnt[:, 1] > 100000).sum()) > 10, mode
    _check(dev, ix, 50, 500, items, off, None, 'conservative', None, True, 3)


def test_python_surface_pickle_and_other_models_untouched():
    import baselines
    import evaluation
    import gru4rec
    train = make_sessions(n_items=150, n_events=4000, seed=3)
    test = make_sessions(n_items=150, n_events=1000, seed=4)
    test['SessionId'] += 100000
    test = test[test.ItemId.isin(train.ItemId.unique())]
    gru = gru4rec.GRU4Rec(layers=[32], batch_size=32, n_epochs=1, n_sample=64, loss='bpr-max', final_act='elu-0.5')
    sk = baselines.SessionKNN(k=30, sample_size=200, similarity='cosine')
    st = baselines.STAN(k=30, sample_size=200, lambda_spw=1.02, lambda_snh=600.0, lambda_inh=2.05)
    lam = dict(lambda_spw=1.02, lambda_snh=600.0, lambda_inh=2.05, lambda_ipw=1.5, lambda_idf=0.8)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
        sk.fit(train.copy())
        st.fit(train.copy())
        before = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in (gru, sk, st)]
        vs = baselines.VSTAN(k=30, sample_size=200, similarity='vector', **lam)
        vs.fit(train.copy())
        res = evaluation.evaluate_events(vs, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
        rec = evaluation.evaluate_gpu(vs, test.copy(), cut_off=[5, 20], mode='median', exclude_seen=True)
        after = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in (gru, sk, st)]
    for b, a in zip(before, after):
        pd.testing.assert_frame_equal(b['events'], a['events'])
        assert b['recall'] == a['recall'] and b['mrr'] == a['mrr']
        assert b['topk_scores'].tobytes() == a['topk_scores'].tobytes()
    assert rec == (res['recall'], res['mrr'])
    # the frame's ranks equal the oracle's on the sorted test frame
    ix = vso.Index(train.SessionId.values, vs.itemidmap[train.ItemId.values].values, train.Time.values, vs.n_items, 'vector', **lam)
    assert ix.f.tobytes() == vs.f.tobytes()
    df = test.assign(ItemIdx=vs.itemidmap[test.ItemId.values].values).sort_values(['SessionId', 'Time', 'ItemId'])
    off = np.r_[0, np.cumsum(df.groupby('SessionId', sort=True).size().values)]
    cnt = vso.rank_events(ix, 30, 200, df.ItemIdx.values, off, None, 'median', None, True)[0]
    np.testing.assert_array_equal(res['events']['rank'].values, bo.ranks(cnt, 'median'))
    # the device's top-k list of the first event equals predict_next's host scores
    first = df.iloc[0]
    ids = vs.itemidmap.index.values
    host = vs.predict_next(first.SessionId, first.ItemId, ids).values
    top = res['topk_items'][0]
    assert np.array_equal(res['topk_scores'][0], host[vs.itemidmap[top].values])
    vs2 = pickle.loads(pickle.dumps(vs))
    with contextlib.redirect_stdout(io.StringIO()):
        res2 = evaluation.evaluate_events(vs2, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
    pd.testing.assert_frame_equal(res['events'], res2['events'])
    assert res['topk_scores'].tobytes() == res2['topk_scores'].tobytes()
