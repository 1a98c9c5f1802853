"""The rule-based baselines on the device (DESIGN §3q): fitted rows (indices, float64 weight bits, lengths) bitwise equal to
tests/rules_oracle.py for SR at steps 1, 3, 10, 20 x 'div' / 'same', at pruning 1, 20 and 1024, and for AR; two fits bitwise equal
and rows that survive export / import; a session of more than 2,000 events and an item holding 30 % of the events; a 172,000-item
catalogue within the fit's scratch budget; per-event counts, sums and k lists equal to baselines_oracle.rank_events on the rows in
all four modes with items=, exclude_seen and history; the Python surface; and ItemKNN / SessionKNN / GRU4Rec evaluations unchanged
by SR / AR calls in between."""
import contextlib
import io
import itertools
import pickle

import numpy as np
import pandas as pd
import pytest

import baselines_oracle as bo
import rules_oracle as ro
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions

pytestmark = pytest.mark.gpu
SCRATCH = 512 << 20


def _fit(kind, off, items, n, pruning, steps=None, weighting=None):
    dev = _lib.Baselines(kind, n, pruning)
    stats = dev.rules_fit(off, items, steps, weighting)
    return dev, stats


def _check_rows(dev, off, items, n, pruning, steps=None, weighting=None):
    rows = ro.rows(off, items, n, pruning, steps, weighting)
    got = dev.rows_export()
    for what, a, b in zip(('idx', 'w', 'len'), got, ro.dense(rows, n, pruning)):
        assert a.tobytes() == b.tobytes(), (what, steps, weighting, pruning)
    return got, rows


@pytest.fixture(scope='module')
def small():
    n = 200
    items, off, _, _ = make_session_arrays(n, 6000, seed=5, max_len=15)
    rs = np.random.RandomState(2)
    items = items.astype(np.int32).copy()
    rep = np.flatnonzero(rs.rand(len(items)) < 0.15)
    items[rep[rep > 0]] = items[rep[rep > 0] - 1]                          # repeats: i = j pairs to drop
    items[rs.rand(len(items)) < 0.1] = 7                                   # a popular item
    return n, off.astype(np.int64), items


@pytest.mark.parametrize('steps, weighting', list(itertools.product([1, 3, 10, 20], ['div', 'same'])))
def test_sr_rows_bitwise_the_oracle(small, steps, weighting):
    n, off, items = small
    dev, (pw, sb, ms) = _fit('sr', off, items, n, 20, steps, weighting)
    _check_rows(dev, off, items, n, 20, steps, weighting)
    lens = np.diff(off)
    assert pw == int(sum(min(steps, L - 1 - p) for L in lens for p in range(L)))
    assert 0 < sb <= SCRATCH and ms > 0


@pytest.mark.parametrize('kind, pruning', list(itertools.product(['sr', 'ar'], [1, 20, 1024])))
def test_pruning_and_ar_rows_bitwise_the_oracle(small, kind, pruning):
    n, off, items = small
    steps, weighting = (10, 'div') if kind == 'sr' else (None, None)
    dev, (pw, _, _) = _fit(kind, off, items, n, pruning, steps, weighting)
    (idx, w, ln), _ = _check_rows(dev, off, items, n, pruning, steps, weighting)
    assert ln.max() == pruning if pruning < 1024 else ln.max() > 20
    if kind == 'ar':
        assert pw == int((np.diff(off) * (np.diff(off) - 1)).sum())


def test_two_fits_bitwise_and_export_import_round_trip(small):
    n, off, items = small
    for kind, st, wt in (('sr', 10, 'div'), ('ar', None, None)):
        a, _ = _fit(kind, off, items, n, 20, st, wt)
        b, _ = _fit(kind, off, items, n, 20, st, wt)
        ra, rb = a.rows_export(), b.rows_export()
        for x, y in zip(ra, rb):
            assert x.tobytes() == y.tobytes()
        c = _lib.Baselines(kind, n, 20)
        c.rows_import(*ra)
        for x, y in zip(ra, c.rows_export()):
            assert x.tobytes() == y.tobytes()
        ev_items, ev_off, _, _ = make_session_arrays(n, 500, seed=9, max_len=12)
        r1 = a.evaluate(ev_items, ev_off, None, [5, 20], 2, None, True, k=6)
        r2 = c.evaluate(ev_items, ev_off, None, [5, 20], 2, None, True, k=6)
        for x, y in zip(r1, r2):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes()


def test_long_session_and_heavy_item():
    rs = np.random.RandomState(7)
    n = 120
    lens = np.r_[2300, rs.randint(2, 12, 1500)]
    items = rs.randint(1, n, lens.sum()).astype(np.int32)
    items[rs.rand(len(items)) < 0.3] = 0                                   # item 0: 30 % of the events
    items[100:140] = 5                                                     # a run of one item inside the long session
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    assert 0.28 < np.mean(items == 0) < 0.32
    for kind, st, wt in (('sr', 20, 'div'), ('sr', 4, 'same'), ('ar', None, None)):
        dev, (pw, sb, ms) = _fit(kind, off, items, n, 64, st, wt)
        _check_rows(dev, off, items, n, 64, st, wt)


def test_172k_catalogue_within_the_scratch_budget():
    n = 172000
    items, off, _, _ = make_session_arrays(n, 420000, seed=3, max_len=10)
    items = items.astype(np.int32)
    off = off.astype(np.int64)
    dev, (pw, sb, ms) = _fit('sr', off, items, n, 20, 10, 'div')
    assert sb <= SCRATCH
    _, rows = _check_rows(dev, off, items, n, 20, 10, 'div')
    t_items, t_off, _, _ = make_session_arrays(300, 600, seed=8, max_len=12)
    t_items = (t_items * 571 + 5).astype(np.int32)
    cnt = dev.evaluate(t_items, t_off, None, [20], 1)[3]
    want = bo.rank_events('itemknn', (n, rows), n, t_items, t_off[:11], None, 'conservative')[0]   # the first ten sessions
    np.testing.assert_array_equal(cnt[:len(want)], want)
    assert (want[:, 1] > 100000).any()                                     # zero-score targets tie most of the catalogue


@pytest.fixture(scope='module')
def fitted(small):
    n, off, items = small
    out = {}
    for kind, st, wt in (('sr', 5, 'div'), ('ar', None, None)):
        dev, _ = _fit(kind, off, items, n, 15, st, wt)
        out[kind] = dev, (n, ro.rows(off, items, n, 15, st, wt))
    rs = np.random.RandomState(3)
    t_items, t_off, _, _ = make_session_arrays(n, 700, seed=7, max_len=25)
    t_items = t_items.astype(np.int32).copy()
    rep = np.flatnonzero(rs.rand(len(t_items)) < 0.25)
    t_items[rep[rep > 0]] = t_items[rep[rep > 0] - 1]
    nh = np.minimum(rs.randint(0, 4, len(t_off) - 1), np.diff(t_off)).astype(np.int32)
    return out, t_items, t_off.astype(np.int64), nh


@pytest.mark.parametrize('kind', ['sr', 'ar'])
def test_counts_sums_and_lists_equal_the_oracle(fitted, kind):
    out, items, off, nh = fitted
    dev, model = out[kind]
    n = model[0]
    cand = np.r_[np.arange(0, n, 3), [0, 0, 7]]
    cand = cand[cand != items[off[0] + 1]]                                # an unlisted target
    for mode, (cd, ex, hist) in itertools.product(['standard', 'conservative', 'median', 'tiebreaking'],
                                                  [(None, False, None), (cand, False, None), (None, True, None), (None, False, nh)]):
        what = (kind, mode, cd is not None, ex, hist is not None)
        rec, mrr, nc, cnt, ti, ts = dev.evaluate(items, off, hist, [1, 5, 20], bo.MODES[mode], cd, ex, k=7)
        wc, wi, ws = bo.rank_events('itemknn', model, n, items, off, hist, mode, cd, ex, 7)
        np.testing.assert_array_equal(cnt, wc, err_msg=str(what))
        np.testing.assert_array_equal(ti, wi, err_msg=str(what))
        np.testing.assert_array_equal(ts, ws, err_msg=str(what))
        hits, rrs = bo.sums(wc, mode, [1, 5, 20])
        assert list(rec) == hits and nc == len(wc), what
        for a, b in zip(mrr, rrs):
            assert a == b or abs(a - b) <= 1e-12 * abs(b), what
        if ex:
            assert (cnt[:, 0] < 0).any()


def test_python_surface_pickle_and_other_models_untouched():
    import baselines
    import evaluation
    import gru4rec
    train = make_sessions(n_items=150, n_events=4000, seed=3)
    test = make_sessions(n_items=150, n_events=1000, seed=4)
    test['SessionId'] += 100000
    test = test[test.ItemId.isin(train.ItemId.unique())]
    gru = gru4rec.GRU4Rec(layers=[32], batch_size=32, n_epochs=1, n_sample=64, loss='bpr-max', final_act='elu-0.5')
    knn = baselines.ItemKNN(n_sims=20)
    sk = baselines.SessionKNN(k=30, sample_size=200, similarity='cosine')
    others = (gru, knn, sk)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
        knn.fit(train.copy())
        sk.fit(train.copy())
        before = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in others]
        res = {}
        for name, m in (('sr', baselines.SR(steps=10, weighting='div', pruning=20)), ('ar', baselines.AR(pruning=20))):
            m.fit(train.copy())
            r = evaluation.evaluate_events(m, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
            assert evaluation.evaluate_gpu(m, test.copy(), cut_off=[5, 20], mode='median', exclude_seen=True) == (r['recall'], r['mrr'])
            res[name] = m, r
        after = [evaluation.evaluate_events(x, test.copy(), cut_off=[5, 20], mode='tiebreaking', k=5) for x in others]
    for b, a in zip(before, after):
        pd.testing.assert_frame_equal(b['events'], a['events'])
        assert b['recall'] == a['recall'] and b['mrr'] == a['mrr']
        assert b['topk_scores'].tobytes() == a['topk_scores'].tobytes()
    for name, (m, r) in res.items():
        steps, weighting = m._steps()
        off, items = ro.sequences(train.SessionId.values, m.itemidmap[train.ItemId.values].values, train.Time.values)
        rows = ro.rows(off, items, m.n_items, 20, steps, weighting)
        for a, b in zip(m.rows, ro.dense(rows, m.n_items, 20)):
            assert a.tobytes() == b.tobytes(), name
        df = test.assign(ItemIdx=m.itemidmap[test.ItemId.values].values).sort_values(['SessionId', 'Time', 'ItemId'])
        toff = np.r_[0, np.cumsum(df.groupby('SessionId', sort=True).size().values)]
        cnt = bo.rank_events('itemknn', (m.n_items, rows), m.n_items, df.ItemIdx.values, toff, None, 'median', None, True)[0]
        np.testing.assert_array_equal(r['events']['rank'].values, bo.ranks(cnt, 'median'))
        first = df.iloc[0]
        ids = m.itemidmap.index.values
        host = m.predict_next(first.SessionId, first.ItemId, ids).values
        assert np.array_equal(r['topk_scores'][0], host[m.itemidmap[r['topk_items'][0]].values])
        m2 = pickle.loads(pickle.dumps(m))
        assert '_dev' not in m2.__dict__
        with contextlib.redirect_stdout(io.StringIO()):
            r2 = evaluation.evaluate_events(m2, test.copy(), cut_off=[5, 20], mode='median', k=10, exclude_seen=True)
        pd.testing.assert_frame_equal(r['events'], r2['events'])
        assert r['topk_scores'].tobytes() == r2['topk_scores'].tobytes()
