"""-m gpu: the session store (g4r_sessions_*, csrc/g4r_sessions.cuh; DESIGN §3e) through Engine.sessions_* and
GRU4Rec.recommend_sessions.  The reference for every result is a replay: a twin engine with the same weights runs each session
alone through predict_topk with batch 1, reset on the session's first event.  Items must match exactly and scores bit for bit
for the elementwise final activations, on the fp32 tiles (eval_tc=1) and the wgmma tiles (eval_tc=2); softmax / softmax_logit
scores within 1e-5 relative (the normaliser partials depend on the tile kind and the lanes of a chunk, DESIGN §3d).  Exported
states are checked against a float64 GRU forward of each session's events."""
import contextlib
import io

import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
from gpu_utils import push_weights, f64_errors
from test_gpu_scoring_f64 import _oracle, _gru, HID_REL, HID_RTOL

pytestmark = pytest.mark.gpu

N_ITEMS = 3001
TC = [False, True]


def _model(act, layers=(48,), seed=0, **kw):
    loss = {'softmax': 'cross-entropy', 'softmax_logit': 'xe_logit'}.get(act, 'bpr-max')
    mk = dict(layers=list(layers), batch_size=8, n_sample=0, loss=loss, final_act=act, **kw)
    m = orc.OracleGRU4Rec(**mk)
    m.init(N_ITEMS)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    for b in m.Bh:
        b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    return mk, m


def _engine(mk, m, lanes, tc=None, capacity=None):
    eng = _lib.Engine(_lib.make_config(N_ITEMS, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=tc))
    push_weights(eng, m)
    if capacity:
        eng.sessions_open(capacity)
    return eng


def _stream(rs, n_sessions, n_events):
    """an interleaved event stream: (keys, items), session keys sparse int64"""
    ids = np.unique(rs.randint(0, 2 ** 62, n_sessions, dtype=np.int64))
    assert len(ids) == n_sessions
    keys = ids[rs.randint(0, n_sessions, n_events)]
    return keys, rs.randint(0, N_ITEMS, n_events).astype(np.int32)


def _calls(rs, keys, sizes=(1, 5, 8, 13, 30), distinct=True):
    """cut the stream into calls of mixed sizes; with `distinct`, a call ends before a key would repeat in it"""
    calls, i = [], 0
    while i < len(keys):
        n = sizes[rs.randint(len(sizes))]
        j = i
        seen = set()
        while j < len(keys) and j - i < n and not (distinct and keys[j] in seen):
            seen.add(keys[j]); j += 1
        calls.append((i, j))
        i = j
    return calls


class Replay(object):
    """each session alone through predict_topk (batch 1) on a twin engine: results of event i, in any order of sessions"""

    def __init__(self, mk, m, tc):
        self.eng = _engine(mk, m, 1, tc)
        self.hist = {}

    def run(self, keys, X, k, items=None, exclude=None, exclude_seen=False):
        out_i = np.empty((len(keys), k), np.int32); out_s = np.empty((len(keys), k), np.float32)
        by_key = {}
        for i, key in enumerate(keys):
            by_key.setdefault(key, []).append(i)
        for key, evs in by_key.items():      # one session at a time: its lane 0 state is re-seeded from the stored state
            for i in evs:
                self._step(key, i, X, k, items, exclude, exclude_seen, out_i, out_s)
        return out_i, out_s

    def _step(self, key, i, X, k, items, exclude, exclude_seen, out_i, out_s):
        st = self.hist.get(key)
        fresh = st is None
        h = [] if fresh else st[1]
        h = h + [int(X[i])]
        if not fresh:
            for li, s in enumerate(st[0]):
                self.eng.set('He%d' % li, s)
        ex = list(exclude[i]) if exclude is not None and exclude[i] is not None else []
        if exclude_seen:
            ex += h
        filt = items is not None or exclude is not None or exclude_seen
        r = self.eng.predict_topk(X[i:i + 1], k, np.array([1 if fresh else 0], np.uint8), items=items,
                                  exclude=[np.array(ex, np.int64)] if filt else None)
        out_i[i], out_s[i] = r[0][0], r[1][0]
        self.hist[key] = ([self.eng.get('He%d' % li)[:1].copy() for li in range(self.eng.cfg.n_layers)], h)

    def end(self, key):
        self.hist.pop(key, None)


def _assert_same(got, ref, soft, what):
    np.testing.assert_array_equal(got[0], ref[0], err_msg=what)
    live = ref[0] >= 0
    if soft:
        np.testing.assert_allclose(got[1][live], ref[1][live], rtol=1e-5, err_msg=what)
    else:
        np.testing.assert_array_equal(got[1][live].view(np.uint32), ref[1][live].view(np.uint32), err_msg=what)
    assert np.isnan(got[1][~live]).all(), what


MODELS = {
    'none_elu': ('elu-0.5', dict()),
    'none_tanh_2layer': ('tanh', dict(layers=(40, 24))),
    'embed_relu': ('relu', dict(embedding=32)),
    'shared_linear': ('linear', dict(constrained_embedding=True)),
    'none_softmax': ('softmax', dict()),
    'embed_softmax_logit_2layer': ('softmax_logit', dict(layers=(40, 24), embedding=32)),
}


@pytest.mark.parametrize('tc', TC)
@pytest.mark.parametrize('model', list(MODELS))
def test_replay_equality(model, tc):
    """1: an interleaved stream of 400 events over 100 sessions in calls of mixed size equals each session replayed alone"""
    act, kw = MODELS[model]
    mk, m = _model(act, **kw)
    eng = _engine(mk, m, 8, tc, capacity=1000)
    rep = Replay(mk, m, tc)
    rs = np.random.RandomState(1)
    keys, X = _stream(rs, 100, 400)
    soft = act.startswith('softmax')
    for a, b in _calls(rs, keys):
        got = eng.sessions_topk(keys[a:b], X[a:b], 20)
        _assert_same(got, rep.run(keys[a:b], X[a:b], 20), soft, '%s tc=%s events %d..%d' % (model, tc, a, b))
    assert eng.sessions_count() == (len(np.unique(keys)), 400)


@pytest.mark.parametrize('model', ['none_elu', 'none_tanh_2layer', 'embed_relu', 'shared_linear'])
def test_exported_states_match_float64(model):
    """2: every session's exported state against the float64 forward of its events from a zero state"""
    act, kw = MODELS[model]
    mk, m = _model(act, **kw)
    eng = _engine(mk, m, 16, capacity=500)
    rs = np.random.RandomState(2)
    keys, X = _stream(rs, 60, 360)
    eng.sessions_feed(keys, X)
    m64 = _oracle(eng, mk, N_ITEMS)
    ek, states, off, items = eng.sessions_export()
    for j, key in enumerate(ek):
        xs = X[keys == key]
        np.testing.assert_array_equal(items[off[j]:off[j + 1]], xs)
        H = [np.zeros((1, L)) for L in mk['layers']]
        for x in xs:
            _, H = _gru(m64, [x], H)
        a, r = f64_errors(states[j], np.concatenate([h[0] for h in H]))
        assert a <= HID_REL and r <= HID_RTOL, 'session %d (%d events): %.3g / %.3g' % (key, len(xs), a, r)


@pytest.mark.parametrize('tc', TC)
def test_feed_with_repeated_keys_equals_single_events(tc):
    """3: one feed with repeated keys (several rounds, chunked by 8 lanes) equals single-event feeds, bitwise, and so does the next top-k"""
    mk, m = _model('elu-0.5', layers=(40, 24), embedding=32)
    a = _engine(mk, m, 8, tc, capacity=200)
    b = _engine(mk, m, 8, tc, capacity=200)
    rs = np.random.RandomState(3)
    keys, X = _stream(rs, 30, 300)
    a.sessions_feed(keys, X)
    for i in range(len(keys)):
        b.sessions_feed(keys[i:i + 1], X[i:i + 1])
    ea, eb = a.sessions_export(), b.sessions_export()
    for u, v in zip(ea, eb):
        np.testing.assert_array_equal(u.view(np.uint8) if u.dtype == np.float32 else u, v.view(np.uint8) if v.dtype == np.float32 else v)
    ks = np.unique(keys)
    x = rs.randint(0, N_ITEMS, len(ks)).astype(np.int32)
    _assert_same(a.sessions_topk(ks, x, 10), b.sessions_topk(ks, x, 10), False, 'next top-k')


def test_lru_eviction():
    """4: capacity 16, 40 sessions: evictions in least-recent-use order, the count bounded, an evicted session restarts fresh,
    a call naming more distinct keys than the capacity is refused without a change"""
    mk, m = _model('tanh')
    eng = _engine(mk, m, 8, capacity=16)
    fresh = _engine(mk, m, 8, capacity=16)
    rs = np.random.RandomState(4)
    order = []                                     # model of the store: keys, least recently used first
    for c in range(60):
        n = rs.randint(1, 9)
        keys = rs.choice(40, n, replace=False).astype(np.int64)
        X = rs.randint(0, N_ITEMS, n).astype(np.int32)
        for key in keys:
            if key in order:
                order.remove(key)
            elif len(order) == 16:
                victim = next(k for k in order if k not in keys)
                order.remove(victim)
            order.append(key)
        eng.sessions_feed(keys, X)
        assert eng.sessions_count()[0] == len(order) <= 16
        np.testing.assert_array_equal(eng.sessions_export()[0], order)
    # an evicted session's next event equals a fresh session's
    gone = [k for k in range(40) if k not in order][:4]
    X = rs.randint(0, N_ITEMS, len(gone)).astype(np.int32)
    _assert_same(eng.sessions_topk(np.array(gone, np.int64), X, 15), fresh.sessions_topk(np.array(gone, np.int64), X, 15), False, 'evicted')
    before = eng.sessions_export()
    with pytest.raises(NotImplementedError):
        eng.sessions_feed(np.arange(100, 117, dtype=np.int64), np.zeros(17, np.int32))
    with pytest.raises(NotImplementedError):
        eng.sessions_topk(np.arange(100, 117, dtype=np.int64), np.zeros(17, np.int32), 5)
    for u, v in zip(before, eng.sessions_export()):
        np.testing.assert_array_equal(u, v)


@pytest.mark.parametrize('tc', TC)
def test_filters_match_replay(tc):
    """5: items, exclude and exclude_seen against the replay with the matching candidate and exclusion lists; history is
    cleared by end and by eviction"""
    mk, m = _model('elu-0.5')
    eng = _engine(mk, m, 8, tc, capacity=40)
    rep = Replay(mk, m, tc)
    rs = np.random.RandomState(5)
    keys, X = _stream(rs, 60, 300)
    X = (X % 40).astype(np.int32)                  # small item set: histories overlap the top-k
    cand = rs.choice(N_ITEMS, 1500, replace=False)
    for ci, (a, b) in enumerate(_calls(rs, keys)):
        ks = keys[a:b]
        # the replay's view of the store: ended or evicted sessions start over
        for k in list(rep.hist):
            if k not in set(eng.sessions_export()[0]):
                rep.end(k)
        excl = [rs.randint(0, 40, rs.randint(0, 6)) for _ in range(b - a)]
        items = cand if ci % 2 else None
        got = eng.sessions_topk(ks, X[a:b], 12, items=items, exclude=excl, exclude_seen=True)
        ref = rep.run(ks, X[a:b], 12, items=items, exclude=excl, exclude_seen=True)
        _assert_same(got, ref, False, 'call %d' % ci)
        if ci % 7 == 3:
            eng.sessions_end(ks[:1]); rep.end(ks[0])
    n, nh = eng.sessions_count()
    assert n <= 40 and nh == sum(len(v[1]) for k, v in rep.hist.items() if k in set(eng.sessions_export()[0]))


def _trained(tmp_path, mk):
    import gru4rec
    df = make_sessions(n_items=400, n_events=3000, seed=6)
    g = gru4rec.GRU4Rec(**mk)
    with contextlib.redirect_stdout(io.StringIO()):
        g.fit(df.copy(), sample_store=mk['n_sample'] * 8)
    fn = str(tmp_path / 'm.pickle')
    g.savemodel(fn)
    return g, fn, df


def _other_paths(g, df, x, j):
    """one round of the lane-addressed scoring paths: predict_next_batch, recommend_next_batch, evaluate_gpu"""
    from gru4rec_b200.evaluation import evaluate_gpu
    p = g.predict_next_batch(np.arange(50) + j, x, batch=50).values
    r = g.recommend_next_batch(np.arange(50) + j, x, k=5, batch=50)
    e = evaluate_gpu(g, df.head(400), batch_size=64)
    return p, r[0], r[1], np.array(e[0] + e[1])


def test_independence_long_calls_and_round_trips(tmp_path):
    """6, 7: interleaving predict_next_batch / recommend_next_batch / evaluate_gpu with session calls changes neither path;
    a 1,300-event call on 512 lanes equals chunked calls; export -> fresh model -> import carries on bitwise; a
    predict_next_batch wider than the engine keeps every session"""
    import gru4rec
    mk = dict(loss='bpr-max', final_act='elu-0.5', layers=[64], batch_size=32, n_epochs=1, n_sample=64)
    g, fn, df = _trained(tmp_path, mk)
    a, b, c = (gru4rec.GRU4Rec.loadmodel(fn) for _ in range(3))
    ids = a.itemidmap.index.values
    rs = np.random.RandomState(7)
    keys = np.unique(rs.randint(0, 2 ** 62, 1300, dtype=np.int64))
    assert len(keys) == 1300
    inp = ids[rs.randint(0, len(ids), 1300)]
    lane_x = [ids[rs.randint(0, len(ids), 50)] for _ in range(7)]
    r_long = a.recommend_sessions(keys, inp, k=25)
    assert a._engine.cfg.eval_batch_size == 512
    # b: the same events in chunks, the lane-addressed paths interleaved; c: those paths alone
    got_i, got_s = [], []
    for n, j in enumerate(range(0, 1300, 200)):
        ob = _other_paths(b, df, lane_x[n], n)
        r = b.recommend_sessions(keys[j:j + 200], inp[j:j + 200], k=25)
        got_i.append(r[0]); got_s.append(r[1])
        oc = _other_paths(c, df, lane_x[n], n)
        for u, v in zip(ob, oc):
            np.testing.assert_array_equal(u, v)
    np.testing.assert_array_equal(np.concatenate(got_i), r_long[0])
    np.testing.assert_array_equal(np.concatenate(got_s).view(np.uint32), r_long[1].view(np.uint32))
    # export -> fresh model -> import
    sid, st, hist = a.export_sessions()
    assert len(sid) == 1300 and all(len(h) == 1 for h in hist)
    d = gru4rec.GRU4Rec.loadmodel(fn)
    d.import_sessions(sid, st, hist)
    nxt = ids[rs.randint(0, len(ids), 300)]
    ra = a.recommend_sessions(keys[:300], nxt, k=25, exclude_seen=True)
    rd = d.recommend_sessions(keys[:300], nxt, k=25, exclude_seen=True)
    np.testing.assert_array_equal(ra[0], rd[0])
    np.testing.assert_array_equal(ra[1].view(np.uint32), rd[1].view(np.uint32))
    # a wider predict_next_batch rebuilds the engine and keeps every session
    before = a.export_sessions()
    a.predict_next_batch(np.arange(700), ids[rs.randint(0, len(ids), 700)], batch=700)
    assert a._engine.cfg.eval_batch_size == 700
    after = a.export_sessions()
    np.testing.assert_array_equal(before[0], after[0])
    np.testing.assert_array_equal(before[1].view(np.uint32), after[1].view(np.uint32))
    assert all(np.array_equal(u, v) for u, v in zip(before[2], after[2]))


def test_errors_leave_the_store_unchanged_and_runs_repeat():
    """8: every refused argument leaves keys, order, states and histories as they were; two identical runs are bitwise equal"""
    mk, m = _model('elu-0.5', layers=(40, 24), embedding=32)
    runs = []
    for _ in range(2):
        eng = _engine(mk, m, 8, True, capacity=24)
        rs = np.random.RandomState(8)
        keys, X = _stream(rs, 40, 200)
        res = []
        for a, b in _calls(rs, keys):
            res.append(eng.sessions_topk(keys[a:b], X[a:b], 7, exclude_seen=True))
        before = eng.sessions_export()
        k0 = before[0][:3]
        bad = [
            lambda: eng.sessions_topk(k0, np.array([0, 1, N_ITEMS], np.int32), 5),                      # item out of range
            lambda: eng.sessions_topk(np.array([k0[0], k0[0]]), np.array([0, 1], np.int32), 5),         # repeated key
            lambda: eng.sessions_topk(k0, np.zeros(3, np.int32), 0),                                    # k
            lambda: eng.sessions_topk(k0, np.zeros(3, np.int32), 5, items=[1, 2]),                      # k > candidates
            lambda: eng.sessions_topk(k0, np.zeros(3, np.int32), 5, items=[1, N_ITEMS]),                # candidate out of range
            lambda: eng.sessions_topk(k0, np.zeros(3, np.int32), 5, exclude=[[1], [N_ITEMS], []]),      # exclusion out of range
            lambda: eng.sessions_topk(np.arange(1000, 1025), np.zeros(25, np.int32), 5),                # more keys than capacity
            lambda: eng.sessions_feed(np.arange(1000, 1025), np.zeros(25, np.int32)),
            lambda: eng.sessions_feed(k0, np.array([0, -1, 2], np.int32)),
            lambda: eng.sessions_import(np.array([5, 5]), np.zeros((2, 64), np.float32)),
            lambda: eng.sessions_import(np.array([5]), np.zeros((1, 64), np.float32), np.array([0, 1]), np.array([N_ITEMS])),
        ]
        for f in bad:
            with pytest.raises((NotImplementedError, IndexError, ValueError)):
                f()
            after = eng.sessions_export()
            for u, v in zip(before, after):
                np.testing.assert_array_equal(u.view(np.uint8), v.view(np.uint8))
        res.append(before)
        runs.append(res)
        eng.close()
    for u, v in zip(runs[0], runs[1]):
        for p, q in zip(u, v):
            np.testing.assert_array_equal(np.asarray(p).view(np.uint8), np.asarray(q).view(np.uint8))
