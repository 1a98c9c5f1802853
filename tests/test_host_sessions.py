"""CPU tests of the session-keyed serving surface of GRU4Rec (recommend_sessions, feed_sessions, end_sessions, export_sessions,
import_sessions) on the engine double (tests/oracle_engine.py), extended here by a session store made of the double's own
predict(): a table of hidden-state rows addressed by slot, a least-recently-used key map and per-session histories, as the
library keeps them (DESIGN §3e).  Covered: item-ID mapping, argument errors, the store's lifetime across engine rebuilds,
fit() and loadmodel(), capacity changes, and pickles that do not change.  The device store is tested in test_gpu_sessions.py."""
import contextlib
import io
import pickle
from collections import OrderedDict

import numpy as np
import pytest

from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
import oracle_engine


class SessionOracleEngine(oracle_engine.OracleEngine):
    """the engine double plus Engine.sessions_*: hidden states in a [capacity x L] table per layer, advanced by the oracle's
    predict_step through slots; top-k by a stable sort of its scores"""
    session_capacity = None

    def sessions_open(self, capacity):
        self.session_capacity = int(capacity)
        self._tab = [np.zeros((self.session_capacity, L), np.float32) for L in self.m.layers]
        self._lru = OrderedDict()                  # key -> slot, least recently used first
        self._hist = {}
        self._free = list(range(self.session_capacity))[::-1]

    def _use(self, keys):
        call = set(int(k) for k in keys)
        if len(call) > self.session_capacity:
            raise NotImplementedError('more distinct sessions than the capacity')
        slots, fresh = [], []
        for key in (int(k) for k in keys):
            if key in self._lru:
                self._lru.move_to_end(key)
                fresh.append(False)
            else:
                if not self._free:
                    victim = next(k for k in self._lru if k not in call)
                    self._free.append(self._lru.pop(victim)); self._hist.pop(victim)
                self._lru[key] = self._free.pop(); self._hist[key] = []
                fresh.append(True)
            slots.append(self._lru[key])
        return np.array(slots), np.array(fresh)

    def _step(self, keys, X, slots, fresh):
        for key, x in zip(keys, X):
            self._hist[int(key)].append(int(x))
        return self.m.predict_step(np.asarray(X, np.int64), self._tab, slots=slots, zero=fresh)

    def sessions_count(self):
        return len(self._lru), sum(len(h) for h in self._hist.values())

    def sessions_feed(self, keys, X):
        self._check_items(X)
        slots, fresh = self._use(keys)
        for i in range(len(keys)):                  # events of a key in call order
            self._step(keys[i:i + 1], X[i:i + 1], slots[i:i + 1], fresh[i:i + 1])

    def sessions_topk(self, keys, X, k, items=None, exclude=None, exclude_seen=False):
        self._check_items(X)
        assert len(set(int(x) for x in keys)) == len(keys)
        slots, fresh = self._use(keys)
        p = self._step(keys, X, slots, fresh)
        ok = np.ones(p.shape, bool)
        if items is not None:
            ok[:] = False
            ok[:, np.asarray(items)] = True
        for b, key in enumerate(keys):
            if exclude is not None and len(exclude[b]):
                ok[b, np.asarray(exclude[b])] = False
            if exclude_seen:
                ok[b, self._hist[int(key)]] = False
        order = np.argsort(-np.where(ok, p, -np.inf), axis=1, kind='stable')[:, :k]
        live = np.take_along_axis(ok, order, axis=1)
        return np.where(live, order, -1).astype(np.int32), np.where(live, np.take_along_axis(p, order, axis=1), np.nan).astype(np.float32)

    def sessions_end(self, keys=None):
        for key in (list(self._lru) if keys is None else [int(k) for k in keys]):
            if key in self._lru:
                self._free.append(self._lru.pop(key)); self._hist.pop(key)

    def sessions_export(self):
        keys = np.array(list(self._lru), np.int64)
        slots = np.array([self._lru[k] for k in keys], np.int64)
        states = np.concatenate([t[slots] for t in self._tab], axis=1) if len(keys) else np.zeros((0, sum(self.m.layers)), np.float32)
        hs = [self._hist[k] for k in keys]
        off = np.concatenate([[0], np.cumsum([len(h) for h in hs])]).astype(np.int64)
        return keys, states, off, np.array(sum(hs, []), np.int32)

    def sessions_import(self, keys, states, hist_off=None, hist_items=None):
        slots, _ = self._use(keys)
        c = 0
        for li, t in enumerate(self._tab):
            t[slots] = states[:, c:c + t.shape[1]]
            c += t.shape[1]
        for i, key in enumerate(keys):
            self._hist[int(key)] = [] if hist_off is None else [int(x) for x in hist_items[hist_off[i]:hist_off[i + 1]]]

    def _check_items(self, X):
        if len(X) and (np.min(X) < 0 or np.max(X) >= int(self.cfg.n_items)):
            raise IndexError('Index out of bounds')


def _install(monkeypatch, gru):
    made = []

    def make(cfg, device=0):
        eng = SessionOracleEngine(cfg, oracle_engine.model_kwargs_of(gru), device)
        made.append(eng)
        return eng
    monkeypatch.setattr(_lib, 'Engine', make)
    return made


MK = dict(loss='bpr-max', final_act='elu-0.5', layers=[12], batch_size=8, n_epochs=1, n_sample=16)


def _trained(monkeypatch, tmp_path, mk=MK, n=2):
    """n models with the same trained weights and no serving state, each on its own engine double"""
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
    return out, df, fn


def _stream(ids, rs, n_sessions=12, n_events=60):
    sess = np.unique(rs.randint(0, 2 ** 62, n_sessions, dtype=np.int64))
    assert len(sess) == n_sessions
    return sess[rs.randint(0, n_sessions, n_events)], ids[rs.randint(0, len(ids), n_events)]


def test_recommend_sessions_equals_per_session_replay(monkeypatch, tmp_path):
    """original item IDs out, and every event's list equals that session replayed alone through recommend_next_batch"""
    (a, b), _, _ = _trained(monkeypatch, tmp_path)
    ids = a.itemidmap.index.values
    rs = np.random.RandomState(0)
    keys, inp = _stream(ids, rs)
    got_i, got_s = np.empty((len(keys), 6), object), np.empty((len(keys), 6), np.float32)
    i = 0
    while i < len(keys):                               # calls of distinct keys
        j = i
        while j < len(keys) and keys[j] not in keys[i:j] and j - i < 5:
            j += 1
        r = a.recommend_sessions(keys[i:j], inp[i:j], k=6)
        assert isinstance(r[0][0, 0], str)
        got_i[i:j], got_s[i:j] = r
        i = j
    for key in np.unique(keys):                        # the replay: one lane, reset when the session changes
        for e in np.flatnonzero(keys == key):
            p = b.predict_next_batch([key], [inp[e]], batch=1)[0].values
            order = np.argsort(-p, kind='stable')[:6]
            np.testing.assert_array_equal(got_i[e], ids[order])
            np.testing.assert_allclose(got_s[e], p[order], rtol=1e-5, atol=1e-7)
    n = len(np.unique(keys))
    assert a._engine.sessions_count() == (n, len(keys))
    sid, states, hist = a.export_sessions()
    assert states.shape == (n, 12) and set(sid) == set(keys)
    for s, h in zip(sid, hist):
        np.testing.assert_array_equal(h, inp[keys == s])


def test_filters_feed_and_end(monkeypatch, tmp_path):
    (a, _), _, _ = _trained(monkeypatch, tmp_path)
    ids = a.itemidmap.index.values
    a.feed_sessions([1, 2, 1, 1], ids[[3, 4, 5, 6]])                # keys may repeat in a feed
    sid, _, hist = a.export_sessions()
    assert list(sid) == [2, 1]                                      # least recently used first
    np.testing.assert_array_equal(hist[1], ids[[3, 5, 6]])
    items, scores = a.recommend_sessions([1], [ids[7]], k=4, exclude_seen=True)
    assert not set(items[0]) & set(ids[[3, 5, 6, 7]])
    items, scores = a.recommend_sessions([2], [ids[8]], k=3, items=ids[:3], exclude=[[ids[0], ids[1], 'unknown id']])
    assert items[0, 0] == ids[2] and items[0, 1] is None and items[0, 2] is None and np.isnan(scores[0, 1:]).all()
    a.end_sessions([1, 12345])
    assert list(a.export_sessions()[0]) == [2]
    a.end_sessions()
    assert len(a.export_sessions()[0]) == 0


def test_argument_errors(monkeypatch, tmp_path):
    (a, _), _, _ = _trained(monkeypatch, tmp_path)
    ids = a.itemidmap.index.values
    for bad in (['a', 'b'], [1.5, 2.0], [True, False]):
        with pytest.raises(TypeError):
            a.recommend_sessions(bad, ids[:2])
        with pytest.raises(TypeError):
            a.feed_sessions(bad, ids[:2])
    with pytest.raises(ValueError):
        a.recommend_sessions([3, 3], ids[:2])
    with pytest.raises(ValueError):
        a.recommend_sessions([3, 4], ids[:3])
    with pytest.raises(ValueError):
        a.recommend_sessions([3], ids[:1], k=0)
    with pytest.raises(ValueError):
        a.recommend_sessions([3], ids[:1], k=3, items=ids[:2])
    with pytest.raises(KeyError):
        a.recommend_sessions([3], ['no such item'])
    with pytest.raises(KeyError):
        a.feed_sessions([3], ['no such item'])
    with pytest.raises(ValueError):
        a.import_sessions([1, 1], np.zeros((2, 12), np.float32))
    with pytest.raises(ValueError):
        a.import_sessions([1], np.zeros((1, 11), np.float32))
    with pytest.raises(KeyError):
        a.import_sessions([1], np.zeros((1, 12), np.float32), [['no such item']])
    assert len(a.export_sessions()[0]) == 0           # nothing reached the store
    a.error_during_train = True
    with pytest.raises(Exception):
        a.recommend_sessions([3], ids[:1])


def test_store_lifetime(monkeypatch, tmp_path):
    """kept across scoring-engine rebuilds and set_value, dropped by fit() and loadmodel(), never pickled; a capacity change
    keeps the most recent sessions that fit"""
    (a, b), df, fn = _trained(monkeypatch, tmp_path)
    ids = a.itemidmap.index.values
    plain = pickle.dumps(a)
    rs = np.random.RandomState(1)
    keys, inp = _stream(ids, rs, 30, 200)
    a.feed_sessions(keys, inp)
    before = a.export_sessions()
    assert pickle.dumps(a) == plain
    # a wider predict_next_batch rebuilds the engine and carries the store
    eng0 = a._engine
    a.predict_next_batch(np.arange(a.eval_lanes + 4), ids[rs.randint(0, len(ids), a.eval_lanes + 4)], batch=a.eval_lanes + 4)
    assert a._engine is not eng0
    after = a.export_sessions()
    np.testing.assert_array_equal(before[0], after[0]); np.testing.assert_array_equal(before[1], after[1])
    # set_value keeps the states
    a.By.set_value(a.By.get_value())
    np.testing.assert_array_equal(a.export_sessions()[1], before[1])
    # a smaller capacity keeps the most recent sessions
    a.session_capacity = 10
    a.recommend_sessions([keys[-1]], [ids[0]], k=2)
    sid = a.export_sessions()[0]
    assert len(sid) == 10 and sid[-1] == keys[-1]
    np.testing.assert_array_equal(sid[:9], [k for k in before[0] if k != keys[-1]][-9:])
    assert pickle.dumps(a) == plain
    # the same events continue identically on a model that imports the exported store
    b.import_sessions(*a.export_sessions())
    r1 = a.recommend_sessions(sid[:3], ids[:3], k=5)
    r2 = b.recommend_sessions(sid[:3], ids[:3], k=5)
    np.testing.assert_array_equal(r1[0], r2[0]); np.testing.assert_array_equal(r1[1], r2[1])
    # fit() and loadmodel() start without sessions
    c = type(a).loadmodel(fn)
    assert len(c.export_sessions()[0]) == 0
    with contextlib.redirect_stdout(io.StringIO()):
        a.fit(df.copy(), sample_store=MK['n_sample'] * 8)
    assert len(a.export_sessions()[0]) == 0
