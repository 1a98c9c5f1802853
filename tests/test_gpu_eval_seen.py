"""-m gpu: evaluation with exclude_seen (Engine.set_eval_exclude_seen, csrc/g4r_seen.cuh, DESIGN §3g).  The test sessions repeat
items, reload them (target = input) and run long, so seen items often compete with the target and many targets are misses.
- fp32 tiles: every event's counts are exactly the counts without exclusion minus the seen items (from a twin's predict scores,
  bitwise the tile scores) that beat or tie the target, with and without a candidate list that holds duplicates and seen items;
  a miss counts (-1, -1)
- wgmma tiles: within the float64 bar over the eligible items, and equal to the fp32 tiles wherever nothing is ambiguous
- sums: equal to a recomputation from the per-event ranks in all four modes, to eval_schedule, and across per-event windows
- lists: equal to a twin replaying the schedule through predict_topk with each session's history as its exclusions, on both
  tile kinds, through overflowing lanes and with fewer eligible items than k
- isolation after a call and refusal over the lists' memory budget"""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gpu_utils import push_weights

pytestmark = pytest.mark.gpu


def _model(n_items, act, layers, seed, by=None, wy_scale=1.0, **extra):
    loss = {'softmax': 'cross-entropy', 'softmax_logit': 'xe_logit'}.get(act, 'bpr-max')
    mk = dict(layers=layers, batch_size=8, n_sample=0, loss=loss, final_act=act, **extra)
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


def _sessions(n_items, n_sessions, seed, lo=0, long_every=7, long_len=60):
    """sessions with reloads (the input again), repeats of earlier inputs and a long session every long_every; items from lo up"""
    rs = np.random.RandomState(seed)
    items, off = [], [0]
    for s in range(n_sessions):
        n = long_len if s % long_every == 0 else rs.randint(2, 12)
        seq = [rs.randint(lo, n_items)]
        while len(seq) < n:
            u = rs.rand()
            seq.append(seq[-1] if u < 0.15 else seq[rs.randint(len(seq))] if u < 0.4 else rs.randint(lo, n_items))
        items += seq
        off.append(len(items))
    return np.array(items, np.int64), np.array(off, np.int32)


def _schedule(n_items, lanes, n_sessions, seed, **kw):
    items, off = _sessions(n_items, n_sessions, seed, **kw)
    return _lib.Schedule(items, off, None, lanes, 0, mode=1)


def _seen_sets(sched):
    """the seen set (sorted item array) of every event in schedule order: the inputs of its slot since its zero-before flag"""
    e = sched.export()
    cur, out = {}, []
    for s in range(sched.n_steps):
        for b in range(int(e['M'][s])):
            sl = int(e['slots'][s, b])
            if e['F'][s, b] & 2 or sl not in cur:
                cur[sl] = set()
            cur[sl].add(int(e['X'][s, b]))
            out.append(np.array(sorted(cur[sl]), np.int64))
    return out


def _targets(sched):
    e = sched.export()
    return np.concatenate([e['Y'][s, :int(e['M'][s])] for s in range(sched.n_steps)]).astype(np.int64)


def _replay_scores(twin, sched):
    """every event's predict row on the twin (lane = the event's state slot, reset where the schedule zeroes)"""
    e = sched.export()
    B = sched.batch_size
    rows = []
    twin.reset_eval_hidden()
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        sl = e['slots'][s, :M]
        X = np.zeros(B, np.int32); X[sl] = e['X'][s, :M]
        R = np.zeros(B, np.uint8); R[sl] = (e['F'][s, :M] & 2) != 0
        rows.append(twin.predict(X, R)[sl])
    return np.concatenate(rows)


def _replay_topk(twin, sched, k, seen, cand=None):
    e = sched.export()
    B = sched.batch_size
    items, scores = [], []
    twin.reset_eval_hidden()
    ev = 0
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        sl = e['slots'][s, :M]
        X = np.zeros(B, np.int32); X[sl] = e['X'][s, :M]
        R = np.zeros(B, np.uint8); R[sl] = (e['F'][s, :M] & 2) != 0
        ex = [np.zeros(0, np.int64)] * B
        for b in range(M):
            ex[sl[b]] = seen[ev + b]
        i, sc = twin.predict_topk(X, k, R, items=cand, exclude=ex)
        items.append(i[sl]); scores.append(sc[sl])
        ev += M
    return np.concatenate(items), np.concatenate(scores)


def _events(eng, sched, cuts, mode, k=0, seen=True):
    eng.set_eval_exclude_seen(seen)
    try:
        return eng.eval_events(sched, cuts, mode, k)
    finally:
        eng.set_eval_exclude_seen(False)


def _windowed(n_items, mk, m, lanes, tc, window, sched, monkeypatch):
    """an engine whose per-event windows hold at most `window` mini-batches: G4R_EVENTS_WINDOW is read when a handle first runs
    eval_events, so it stays set until that first call has run"""
    monkeypatch.setenv('G4R_EVENTS_WINDOW', str(window))
    try:
        eng = _engine(n_items, mk, m, lanes, tc)
        eng.eval_events(sched, [20], 0)
    finally:
        monkeypatch.delenv('G4R_EVENTS_WINDOW')
    return eng


def _rescoring_launches(eng, sched, k, wy, by, seen=True):
    """launches of eval_events(exclude_seen) with the item table (wy, by) minus those with the scores reversed (nothing
    overflows): 4 per chunk of overflowed lanes rescored at the end of a per-event window"""
    d = []
    for b in (by, -by):
        eng.set('Wy', wy); eng.set('By', b)
        n0 = eng.kernel_launches()
        _events(eng, sched, [20], 0, k=k, seen=seen)
        d.append(eng.kernel_launches() - n0)
    return d[0] - d[1]


@pytest.mark.parametrize('with_items', [False, True])
def test_fp32_counts_exact(with_items):
    n_items, lanes = 700, 24
    mk, m = _model(n_items, 'relu', [32], seed=1, by=-0.05)         # relu below zero: ties among seen items and the target
    sched = _schedule(n_items, lanes, 160, seed=2)
    seen, Y = _seen_sets(sched), _targets(sched)
    twin = _engine(n_items, mk, m, lanes, False)
    sc = _replay_scores(twin, sched)
    twin.close()
    eng = _engine(n_items, mk, m, lanes, False)
    cand = None
    if with_items:
        rs = np.random.RandomState(3)
        cand = np.concatenate([rs.choice(n_items, 300), rs.choice(n_items, 50), np.unique(np.concatenate(seen[:40]))])   # duplicates, seen items
        eng.set_eval_items(cand)
    mult = np.bincount(cand, minlength=n_items) if with_items else np.ones(n_items, np.int64)
    miss = np.array([np.isin(y, s) for y, s in zip(Y, seen)])
    assert 0.1 < miss.mean() < 0.6
    for mode in range(3):
        base = eng.eval_events(sched, [20], mode)[3]
        got = _events(eng, sched, [20], mode)[3]
        t = sc[np.arange(len(Y)), Y]
        want = base.copy()
        for j, s in enumerate(seen):
            if miss[j]:
                want[j] = -1
                continue
            v = sc[j, s]
            want[j, 0] -= int((mult[s] * (v > t[j])).sum()); want[j, 1] -= int((mult[s] * (v == t[j])).sum())
        np.testing.assert_array_equal(got, want, err_msg='mode %d' % mode)
        assert np.all(got[~miss] >= 0)
        assert (want[~miss] != base[~miss]).any()
    eng.close()


def test_wgmma_counts_within_float64_bar_and_equal_fp32():
    n_items, lanes = 2500, 64
    mk, m = _model(n_items, 'linear', [32], seed=4)
    sched = _schedule(n_items, lanes, 260, seed=5, lo=2300)            # sessions from the top items: seen items compete
    seen, Y = _seen_sets(sched), _targets(sched)
    out = {}
    for tc in (False, True):
        eng = _engine(n_items, mk, m, lanes, tc)
        out[tc] = _events(eng, sched, [20], 0)[3]
        eng.close()
    e = sched.export()
    H = [np.zeros((lanes, L), dtype=np.float32) for L in m.layers]
    sure, amb, j = [], [], 0
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        m.predict_step(e['X'][s, :M].astype(np.int64), H, slots=e['slots'][s, :M].astype(np.int64), zero=(e['F'][s, :M] & 2) != 0)
        y = H[-1][e['slots'][s, :M]].astype(np.float64)
        sc = y @ m.Wy.astype(np.float64).T + m.By.reshape(-1).astype(np.float64)
        for b in range(M):
            row = np.delete(sc[b], seen[j + b])                        # the eligible items (the target included unless seen)
            t = sc[b, Y[j + b]]
            tol = 1e-5 * (abs(t) + 1.0)
            sure.append((row > t + tol).sum()); amb.append((np.abs(row - t) <= tol).sum())
        j += M
    sure, amb = np.array(sure), np.array(amb)
    miss = np.array([np.isin(y, s) for y, s in zip(Y, seen)])
    assert miss.mean() > 0.1
    for tc, cnt in out.items():
        assert np.all(cnt[miss] == -1), 'eval_tc=%s' % tc
        g = cnt[~miss, 0]
        assert np.all(g >= sure[~miss]) and np.all(g <= sure[~miss] + amb[~miss]), 'eval_tc=%s' % tc
    clear = ~miss & (amb == 1)
    assert clear.mean() > 0.4
    np.testing.assert_array_equal(out[False][clear], out[True][clear])


@pytest.mark.parametrize('tc', [False, True])
def test_sums_from_ranks_and_windows(tc, monkeypatch):
    """more than 512 mini-batches (two staging windows), per-event windows of 7: sums, counts and lists equal the default window's,
    the sums equal eval_schedule's and a recomputation from the per-event ranks (inf adds nothing) in all four modes.  That the
    short windows apply is shown by the overflow rescoring, which runs once per window: with scores rising with the item index
    (every lane overflows) the 7-step windows rescore in more chunks than the 512-step ones"""
    n_items, lanes = 8000, 8
    mk, m = _model(n_items, 'relu', [16], seed=12, by=-0.2)
    sched = _schedule(n_items, lanes, 700, seed=13, long_every=40, long_len=120)
    assert sched.n_steps > 512
    eng = _engine(n_items, mk, m, lanes, tc)
    short = _windowed(n_items, mk, m, lanes, tc, 7, sched, monkeypatch)
    cuts = [1, 5, 20]
    for mode in range(4):
        a = _events(eng, sched, cuts, mode, k=10)
        b = _events(short, sched, cuts, mode, k=10)
        eng.set_eval_exclude_seen(True)
        rec, mrr, n = eng.eval_schedule(sched, cuts, mode)
        eng.set_eval_exclude_seen(False)
        for x, y in zip(a, b):
            if isinstance(x, np.ndarray):
                np.testing.assert_array_equal(x.view(np.uint8), y.view(np.uint8), err_msg='mode %d' % mode)
            else:
                assert x == y
        np.testing.assert_array_equal(a[0].view(np.uint64), rec.view(np.uint64))
        np.testing.assert_array_equal(a[1].view(np.uint64), mrr.view(np.uint64))
        cnt = a[3]
        gt, eq = cnt[:, 0].astype(np.float64), cnt[:, 1].astype(np.float64)
        rank = gt + eq if mode == 1 else gt + 0.5 * (eq - 1) + 1 if mode == 2 else gt + 1
        rank[cnt[:, 0] < 0] = np.inf
        assert (cnt[:, 0] < 0).mean() > 0.1
        for c, r_dev, q_dev in zip(cuts, a[0], a[1]):
            assert r_dev == (rank <= c).sum()
            np.testing.assert_allclose(q_dev, (1.0 / rank[rank <= c]).sum(), rtol=1e-12)
    rising = np.linspace(0.01, 1, n_items, dtype=np.float32).reshape(-1, 1)     # positive: relu keeps the order
    wy = (m.Wy * np.float32(1e-3)).astype(np.float32)
    d_long, d_short = (_rescoring_launches(x, sched, 10, wy, rising) for x in (eng, short))
    assert d_long >= 4 * 2 and d_short > d_long, (d_long, d_short)      # one window per staging window / many more
    eng.close(); short.close()


CASES = [
    (3000, [48], 40, 'elu-0.5', 20, {}),
    (3000, [64], 96, 'tanh', 20, dict(constrained_embedding=True)),     # shared embedding
    (3000, [64], 100, 'softmax', 20, {}),
]


@pytest.mark.parametrize('n_items,layers,lanes,act,k,extra', CASES, ids=['elu', 'tanh-shared', 'softmax'])
def test_lists_equal_predict_topk_replay(n_items, layers, lanes, act, k, extra):
    mk, m = _model(n_items, act, layers, seed=6, **extra)
    sched = _schedule(n_items, lanes, 3 * lanes, seed=7, lo=2700)
    seen = _seen_sets(sched)
    twin = _engine(n_items, mk, m, lanes)
    e_items, e_scores = _replay_topk(twin, sched, k, seen)
    twin.close()
    for tc in (False, True):
        eng = _engine(n_items, mk, m, lanes, tc)
        items, scores = _events(eng, sched, [20], 0, k=k)[4:]
        eng.close()
        np.testing.assert_array_equal(items, e_items, err_msg='eval_tc=%s' % tc)
        for j, s in enumerate(seen):
            assert not np.isin(items[j], s).any()
        if act.startswith('softmax'):
            np.testing.assert_allclose(scores, e_scores, rtol=1e-5, atol=0, err_msg='eval_tc=%s' % tc)
        else:
            np.testing.assert_array_equal(scores.view(np.uint32), e_scores.view(np.uint32), err_msg='eval_tc=%s' % tc)


def test_fewer_eligible_than_k():
    n_items, lanes, k = 500, 16, 8
    mk, m = _model(n_items, 'elu-0.5', [16], seed=8)
    cand = np.array([3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 3], np.int32)      # 10 distinct, one duplicate
    rs = np.random.RandomState(9)
    items, off = [], [0]
    for s in range(40):                                                 # sessions over the candidates: many seen
        items += list(rs.choice(cand, rs.randint(2, 9)))
        off.append(len(items))
    sched = _lib.Schedule(np.array(items, np.int64), np.array(off, np.int32), None, lanes, 0, mode=1)
    seen = _seen_sets(sched)
    twin = _engine(n_items, mk, m, lanes)
    e_items, e_scores = _replay_topk(twin, sched, k, seen, cand=cand)
    twin.close()
    eng = _engine(n_items, mk, m, lanes)
    eng.set_eval_items(cand)
    got_i, got_s = _events(eng, sched, [5], 0, k=k)[4:]
    eng.close()
    assert (got_i == -1).any()
    np.testing.assert_array_equal(got_i, e_items)
    np.testing.assert_array_equal(got_s.view(np.uint32), e_scores.view(np.uint32))
    assert np.all(np.isnan(got_s[got_i < 0]))


@pytest.mark.parametrize('act,seen_on', [('linear', True), ('softmax', True), ('linear', False)])
def test_overflow_in_every_window(act, seen_on, monkeypatch):
    """scores rising with the item index overflow the survivor lists of nearly every lane, and are rescored at the end of each
    per-event window.  The sessions input the top items, so with exclude_seen that rescoring must use each lane's seen set of its
    own mini-batch, rebuilt from the schedule at a step that depends on the staging window (more than 512 mini-batches) and on
    where the per-event window starts inside it.  Lists equal the predict_topk replay and are bitwise the same for windows of
    512, 1 and 7 mini-batches; windows of one mini-batch rescore at least once per mini-batch (10 lanes: the 512-step windows
    rescore about 10 / 16 chunks per mini-batch).  seen_on=False: the same for the plain lists."""
    n_items, lanes, k = 20000, 10, 20
    rising = np.linspace(-1, 1, n_items, dtype=np.float32).reshape(-1, 1)
    mk, m = _model(n_items, act, [16], seed=6, by=rising, wy_scale=1e-3)
    sched = _schedule(n_items, lanes, 560, seed=10, lo=n_items - 40, long_every=5, long_len=25)
    assert sched.n_steps > 512
    seen = _seen_sets(sched) if seen_on else [np.zeros(0, np.int64)] * sched.n_events
    twin = _engine(n_items, mk, m, lanes)
    e_items, e_scores = _replay_topk(twin, sched, k, seen)
    twin.close()
    for tc in (False, True):
        got, launches = {}, {}
        for window in (None, 1, 7):
            eng = _engine(n_items, mk, m, lanes, tc) if window is None else _windowed(n_items, mk, m, lanes, tc, window, sched, monkeypatch)
            eng.set_eval_exclude_seen(seen_on)
            got[window] = eng.eval_events(sched, [1, 20], 2, k=k)
            eng.set_eval_exclude_seen(False)
            launches[window] = _rescoring_launches(eng, sched, k, m.Wy, rising, seen_on)
            eng.close()
        items, scores = got[None][4:]
        for j, s in enumerate(seen):
            assert not np.isin(items[j], s).any()
        assert launches[1] >= 4 * int(0.9 * sched.n_steps) and launches[1] > launches[None], launches
        np.testing.assert_array_equal(items, e_items, err_msg='eval_tc=%s' % tc)
        if act == 'softmax':
            np.testing.assert_allclose(scores, e_scores, rtol=1e-5, atol=0)
        else:
            np.testing.assert_array_equal(scores.view(np.uint32), e_scores.view(np.uint32))
        for window in (1, 7):
            for a, b in zip(got[None], got[window]):
                if isinstance(a, np.ndarray):
                    np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8), err_msg='eval_tc=%s window=%s' % (tc, window))
                else:
                    assert a == b


def test_isolation_after_a_call():
    n_items, lanes = 3000, 64
    mk, m = _model(n_items, 'elu-0.5', [48], seed=11)
    sched = _schedule(n_items, lanes, 150, seed=12)
    X = np.random.RandomState(13).randint(0, n_items, lanes).astype(np.int32)

    def run(eng):
        r = eng.eval_schedule(sched, [5, 20], 0)
        ev = eng.eval_events(sched, [5, 20], 0, k=10)
        eng.reset_eval_hidden()
        p = eng.predict(X)
        eng.reset_eval_hidden()
        t = eng.predict_topk(X, 10)
        return r[:2] + ev[:2] + ev[3:] + (p,) + t
    fresh = _engine(n_items, mk, m, lanes)
    want = run(fresh)
    fresh.close()
    eng = _engine(n_items, mk, m, lanes)
    _events(eng, sched, [5, 20], 0, k=10)
    eng.set_eval_exclude_seen(True)
    eng.eval_schedule(sched, [5, 20], 1)
    eng.set_eval_exclude_seen(False)
    for a, b in zip(want, run(eng)):
        np.testing.assert_array_equal(a, b)
    eng.close()


def test_refused_over_budget(monkeypatch):
    """a schedule whose seen lists exceed the budget is refused before any device work: the hidden state and the evaluation
    settings are as they were"""
    n_items, lanes = 1000, 32
    mk, m = _model(n_items, 'tanh', [24], seed=14)
    sched = _schedule(n_items, lanes, 100, seed=15)                    # longest session 60: 32 x 59 x 4 bytes
    X1, X2 = (np.random.RandomState(s).randint(0, n_items, lanes).astype(np.int32) for s in (16, 17))
    cand = np.arange(0, n_items, 3)
    ref = _engine(n_items, mk, m, lanes)
    ref.set_eval_items(cand)
    ref.predict(X1)
    want_p = ref.predict(X2)
    want_ev = _events(ref, sched, [20], 0, k=5)
    ref.close()
    eng = _engine(n_items, mk, m, lanes)
    eng.set_eval_items(cand)
    eng.predict(X1)
    eng.set_eval_exclude_seen(True)
    monkeypatch.setenv('G4R_SEEN_BUDGET', str(32 * 59 * 4 - 1))
    for call in (lambda: eng.eval_schedule(sched, [20], 0), lambda: eng.eval_events(sched, [20], 0, 5)):
        with pytest.raises(NotImplementedError, match='exclude_seen'):
            call()
    monkeypatch.setenv('G4R_SEEN_BUDGET', str(32 * 59 * 4))
    np.testing.assert_array_equal(eng.predict(X2), want_p)            # the hidden state was untouched
    got = eng.eval_events(sched, [20], 0, 5)                           # still exclude_seen, still the candidates
    eng.set_eval_exclude_seen(False)
    eng.close()
    for a, b in zip(want_ev, got):
        np.testing.assert_array_equal(a, b)
