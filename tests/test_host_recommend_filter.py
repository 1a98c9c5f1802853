"""CPU tests of recommend_next_batch's filters (items=, exclude=, exclude_seen=) on the engine double (tests/oracle_engine.py),
extended here by a filtered predict_topk made of the double's own predict(), a mask and a stable sort: item-ID mapping of the
candidates and exclusions, the per-lane history behind exclude_seen and where it is cleared, None / NaN padding of short lanes,
and that savemodel's pickle carries no history.  The device kernels are tested in test_gpu_topk_filter.py."""
import contextlib
import io
import pickle

import numpy as np
import pytest

from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
import oracle_engine


class FilterOracleEngine(oracle_engine.OracleEngine):
    """the engine double plus Engine.predict_topk with filters: predict(), softmax renormalised over the distinct candidates,
    ineligible items masked out, then a stable sort; slots past a lane's eligible items are -1 / NaN"""

    calls = []

    def predict_topk(self, X, k, reset_mask=None, items=None, exclude=None):
        FilterOracleEngine.calls.append((items is not None, exclude is not None))
        n_items = int(self.cfg.n_items)
        cand = np.arange(n_items) if items is None else np.unique(np.asarray(items, dtype=np.int64))
        k = _lib.check_topk(k, len(cand))
        p = self.predict(X, reset_mask).astype(np.float64)
        if items is not None and self.mk.get('final_act') in ('softmax', 'softmax_logit'):
            p[:, cand] /= p[:, cand].sum(axis=1, keepdims=True)
        ok = np.zeros(p.shape, bool)
        ok[:, cand] = True
        for b, e in enumerate(exclude if exclude is not None else []):
            if e is not None and len(e):
                ok[b, np.asarray(e, dtype=np.int64)] = False
        key = np.where(ok, p, -np.inf)
        order = np.argsort(-key, axis=1, kind='stable')[:, :k]
        live = np.take_along_axis(ok, order, axis=1)
        out = np.where(live, order, -1).astype(np.int32)
        sc = np.where(live, np.take_along_axis(p, order, axis=1), np.nan).astype(np.float32)
        return out, sc


def _install(monkeypatch, gru):
    def make(cfg, device=0):
        return FilterOracleEngine(cfg, oracle_engine.model_kwargs_of(gru), device)
    monkeypatch.setattr(_lib, 'Engine', make)


def _twins(monkeypatch, tmp_path, mk, n=2):
    import gru4rec
    df = make_sessions(n_items=60, n_events=800, seed=5, item_as_str=True)
    gru = gru4rec.GRU4Rec(**mk)
    _install(monkeypatch, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(df.copy(), sample_store=mk['n_sample'] * 8)
    fn = str(tmp_path / 'model.pickle')
    gru.savemodel(fn)
    out = []
    for _ in range(n):
        g = gru4rec.GRU4Rec.loadmodel(fn)
        _install(monkeypatch, g)
        out.append(g)
    return out


MK = dict(loss='bpr-max', final_act='elu-0.5', layers=[12], batch_size=8, n_epochs=1, n_sample=16)


def _expected(preds, k, cand_ids=None, excl=None):
    """top k of predict_next_batch's frame (items x batch) restricted to cand_ids, minus excl[b] per lane"""
    ids = preds.index.to_numpy()
    v = preds.values.T.astype(np.float64)
    ok = np.ones(v.shape, bool) if cand_ids is None else np.isin(ids, list(cand_ids))[None, :].repeat(len(v), 0)
    for b, e in enumerate(excl or []):
        ok[b] &= ~np.isin(ids, list(e))
    order = np.argsort(-np.where(ok, v, -np.inf), axis=1, kind='stable')[:, :k]
    live = np.take_along_axis(ok, order, axis=1)
    items = np.where(live, ids[order], None)
    return items, np.where(live, np.take_along_axis(v, order, axis=1), np.nan).astype(np.float32)


def test_items_and_exclude_map_original_ids(monkeypatch, tmp_path):
    a, b = _twins(monkeypatch, tmp_path, MK)
    ids = a.itemidmap.index.values
    rs = np.random.RandomState(0)
    sess = np.arange(4)
    cand = list(ids[rs.choice(len(ids), 25, replace=False)])
    cand_dup = cand + cand[:5]                                  # duplicates are ignored
    excl = [list(rs.choice(cand, 3, replace=False)) + ['no-such-item'], None, [], list(cand[:10])]
    inp = ids[rs.randint(0, len(ids), 4)]
    ref = b.predict_next_batch(sess, inp, batch=4)
    items, scores = a.recommend_next_batch(sess, inp, k=8, batch=4, items=cand_dup, exclude=excl)
    e_items, e_scores = _expected(ref, 8, cand, [e or [] for e in excl])
    assert set(items.reshape(-1)) <= set(cand)
    np.testing.assert_array_equal(items, e_items.astype(items.dtype))
    np.testing.assert_array_equal(scores, e_scores)
    for lane, e in enumerate(excl):
        assert not set(items[lane]) & set(e or [])


def test_unknown_candidate_raises_and_k_bound(monkeypatch, tmp_path):
    a, = _twins(monkeypatch, tmp_path, MK, n=1)
    ids = a.itemidmap.index.values
    with pytest.raises(KeyError):
        a.recommend_next_batch(np.arange(3), ids[:3], k=2, batch=3, items=list(ids[:5]) + ['no-such-item'])
    with pytest.raises(ValueError):
        a.recommend_next_batch(np.arange(3), ids[:3], k=4, batch=3, items=list(ids[:3]) * 2)
    with pytest.raises(ValueError):
        a.recommend_next_batch(np.arange(3), ids[:3], k=2, batch=3, exclude=[None, None])


def test_unfiltered_call_is_unchanged(monkeypatch, tmp_path):
    """no filter: the engine's plain predict_topk, IDs of the catalogue's dtype"""
    a, b = _twins(monkeypatch, tmp_path, MK)
    ids = a.itemidmap.index.values
    FilterOracleEngine.calls.clear()
    items, scores = a.recommend_next_batch(np.arange(3), ids[:3], k=5, batch=3)
    assert FilterOracleEngine.calls == [(False, False)]
    e_items, e_scores = _expected(b.predict_next_batch(np.arange(3), ids[:3], batch=3), 5)
    np.testing.assert_array_equal(items, e_items.astype(items.dtype))
    np.testing.assert_array_equal(scores, e_scores)


def test_short_lanes_padded_with_none_and_nan(monkeypatch, tmp_path):
    import gru4rec
    df = make_sessions(n_items=40, n_events=500, seed=7, item_as_str=False)
    gru = gru4rec.GRU4Rec(**MK)
    _install(monkeypatch, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(df.copy(), sample_store=MK['n_sample'] * 8)
    ids = gru.itemidmap.index.values
    cand = list(ids[:6])
    items, scores = gru.recommend_next_batch(np.arange(2), ids[:2], k=5, batch=2, items=cand, exclude=[cand[:3], None])
    assert items.dtype == object
    assert list(items[0, 3:]) == [None, None] and np.isnan(scores[0, 3:]).all()
    assert all(x is not None for x in items[0, :3]) and not np.isnan(scores[0, :3]).any()
    assert set(items[0, :3]) == set(cand[3:])
    assert all(x is not None for x in items[1]) and set(items[1]) <= set(cand)


def test_exclude_seen_follows_the_session(monkeypatch, tmp_path):
    """exclude_seen: items fed into a lane since its session began, across alternating predict_next_batch /
    recommend_next_batch calls; cleared on a new session id and on a batch-size change"""
    a, b = _twins(monkeypatch, tmp_path, MK)
    ids = a.itemidmap.index.values
    rs = np.random.RandomState(3)
    sess = np.arange(4)
    seen = [[] for _ in range(4)]
    for step in range(7):
        if step == 4:
            sess = sess.copy(); sess[1] = 77; seen[1] = []
        inp = ids[rs.randint(0, len(ids), 4)]
        for lane in range(4):
            seen[lane].append(inp[lane])
        ref = b.predict_next_batch(sess, inp, batch=4)
        if step % 2 == 0:
            items, scores = a.recommend_next_batch(sess, inp, k=10, batch=4, exclude_seen=True)
            e_items, e_scores = _expected(ref, 10, None, seen)
            np.testing.assert_array_equal(items, e_items.astype(items.dtype), err_msg='step %d' % step)
            np.testing.assert_array_equal(scores, e_scores)
        else:
            np.testing.assert_array_equal(a.predict_next_batch(sess, inp, batch=4).values, ref.values)
    assert list(a._seen_n) == [7, 3, 7, 7]
    # a new batch size clears every lane
    inp = ids[:3]
    items, _ = a.recommend_next_batch(np.arange(3), inp, k=10, batch=3, exclude_seen=True)
    e_items, _ = _expected(b.predict_next_batch(np.arange(3), inp, batch=3), 10, None, [[x] for x in inp])
    np.testing.assert_array_equal(items, e_items.astype(items.dtype))
    assert list(a._seen_n) == [1, 1, 1]


def test_history_grows_past_its_capacity(monkeypatch, tmp_path):
    a, = _twins(monkeypatch, tmp_path, MK, n=1)
    ids = a.itemidmap.index.values
    for step in range(20):
        a.predict_next_batch(np.arange(2), ids[[step, step + 20]], batch=2)
    assert list(a._seen_n) == [20, 20]
    assert list(a._seen[0, :20]) == list(a.itemidmap[ids[:20]].values)
    items, _ = a.recommend_next_batch(np.arange(2), ids[[20, 40]], k=5, batch=2, exclude_seen=True)
    assert not set(items[0]) & set(ids[:21])


def test_savemodel_has_no_history(monkeypatch, tmp_path):
    a, = _twins(monkeypatch, tmp_path, MK, n=1)
    ids = a.itemidmap.index.values
    a.recommend_next_batch(np.arange(3), ids[:3], k=3, batch=3, exclude_seen=True)
    assert a._seen_n.sum() == 3
    fn = str(tmp_path / 'again.pickle')
    a.savemodel(fn)
    with open(fn, 'rb') as f:
        st = pickle.load(f).__dict__
    assert '_seen' not in st and '_seen_n' not in st
