"""-m gpu: evaluation from each session's history (Schedule(n_history=...), csrc/g4r_history.cuh, DESIGN §3h).  A history
schedule walks the same mini-batches as the plain schedule of the same data, so the plain evaluation of the concatenated data,
restricted to the counted events, is an exact oracle:
- fp32 tiles, all four modes, with and without exclude_seen and a candidate list with duplicates: per-event counts bitwise, hit
  sums exact, MRR sums within 1e-12 relative (the blocks sum in another order); eval_schedule's sums are eval_events'
- wgmma tiles (shown to run by the launch count): within the float64 bar, and equal to the fp32 counts wherever the bar is
  unambiguous
- overflow rescoring of ranking blocks (per-event windows of 512, 1 and 7 steps, both tile kinds): lists equal to a replay
  through the session store (feed_sessions of the history, recommend_sessions per test event)
- edge shapes: leave-one-out, histories of 0, 1 and more than 600 events (over staging windows), more sessions than lanes,
  sessions that are all history; shared-embedding, separate-embedding and two-layer models
- top-k lists: bitwise the plain lists of the same events (themselves held to a predict_topk replay in test_gpu_eval_seen.py)
- ranking launches grow with the counted events, not with the steps
- determinism, the refusal over the seen-list budget, and evaluate_gpu / evaluate_events(history=) end to end"""
import contextlib
import io

import numpy as np
import pandas as pd
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gpu_utils import push_weights

pytestmark = pytest.mark.gpu

MODELS = {
    'plain': dict(layers=[24]),
    'shared': dict(layers=[24], constrained_embedding=True),
    'embed': dict(layers=[24], embedding=16),
    'two_layer': dict(layers=[24, 16]),
}


def _model(n_items, act, seed, **extra):
    loss = {'softmax': 'cross-entropy', 'softmax_logit': 'xe_logit'}.get(act, 'bpr-max')
    mk = dict(batch_size=8, n_sample=0, loss=loss, final_act=act, **extra)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    return mk, m


def _engine(n_items, mk, m, lanes, tc=None):
    eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=tc))
    push_weights(eng, m)
    return eng


def _data(n_items, n_sessions, seed, long_every=0, long_hist=650):
    """sessions that repeat and reload items; n_history per session: 0, 1, a few, all of the session, and (every long_every-th
    session) more than 600 events"""
    rs = np.random.RandomState(seed)
    items, off, nh = [], [0], []
    for s in range(n_sessions):
        h = long_hist if long_every and s % long_every == 0 else [0, 1, rs.randint(2, 15)][s % 3]
        t = rs.randint(1, 6) if s % 11 or h == 0 else 0
        n = h + t
        seq = [rs.randint(n_items)]
        while len(seq) < n:
            u = rs.rand()
            seq.append(seq[-1] if u < 0.1 else seq[rs.randint(len(seq))] if u < 0.3 else rs.randint(n_items))
        items += seq[:n]
        off.append(len(items))
        nh.append(min(h, n))
    return np.array(items, np.int64), np.array(off, np.int32), np.array(nh, np.int32)


def _pair(items, off, nh, lanes):
    plain = _lib.Schedule(items, off, None, lanes, 0, mode=1)
    hist = _lib.Schedule(items, off, None, lanes, 0, mode=1, n_history=nh)
    used = np.arange(lanes)[None, :] < plain.batch_sizes()[:, None]
    return plain, hist, hist.counted()[used]


def _events(eng, sched, cuts, mode, k=0, seen=False):
    eng.set_eval_exclude_seen(seen)
    try:
        return eng.eval_events(sched, cuts, mode, k)
    finally:
        eng.set_eval_exclude_seen(False)


def _sums(counts, cuts, mode):
    gt, eq = counts[:, 0].astype(np.float64), counts[:, 1].astype(np.float64)
    rk = gt + eq if mode == 1 else gt + 0.5 * (eq - 1.0) + 1.0 if mode == 2 else gt + 1.0
    rk[counts[:, 0] < 0] = np.inf
    with np.errstate(divide='ignore'):                                    # 'conservative' with items= can give rank 0
        return np.array([(rk <= c).sum() for c in cuts], np.float64), np.array([(1.0 / rk[rk <= c]).sum() for c in cuts], np.float64)


def _check_against_plain(eng, plain, hist, keep, cuts, mode, seen, k=0):
    rp, mp, np_, cp, ip, sp = _events(eng, plain, cuts, mode, k, seen)
    rh, mh, nh_, ch, ih, sh = _events(eng, hist, cuts, mode, k, seen)
    assert nh_ == keep.sum() == len(ch) and np_ == len(cp)
    np.testing.assert_array_equal(ch, cp[keep])
    hits, rr = _sums(cp[keep], cuts, mode)
    np.testing.assert_array_equal(rh, hits)
    np.testing.assert_allclose(mh, rr, rtol=1e-12, atol=0)
    eng.set_eval_exclude_seen(seen)
    try:
        rs, ms, ns = eng.eval_schedule(hist, cuts, mode)
    finally:
        eng.set_eval_exclude_seen(False)
    assert ns == nh_
    np.testing.assert_array_equal(rs, rh)
    np.testing.assert_array_equal(ms, mh)
    if k:
        np.testing.assert_array_equal(ih, ip[keep])
        np.testing.assert_array_equal(sh, sp[keep])
    return ch


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
@pytest.mark.parametrize('seen', [False, True])
def test_fp32_counts_equal_the_concatenated_evaluation(mode, seen):
    n_items = 300
    mk, m = _model(n_items, 'softmax', 1, **MODELS['plain'])
    eng = _engine(n_items, mk, m, 16, tc=False)
    items, off, nh = _data(n_items, 90, seed=2 + mode)
    plain, hist, keep = _pair(items, off, nh, 16)
    ch = _check_against_plain(eng, plain, hist, keep, [1, 5, 20], mode, seen)
    if seen:
        assert (ch[:, 0] < 0).any()
    cand = np.concatenate([np.arange(0, n_items, 3), np.arange(0, 40)])    # duplicates
    eng.set_eval_items(cand)
    try:
        _check_against_plain(eng, plain, hist, keep, [1, 5, 20], mode, seen)
    finally:
        eng.set_eval_items(None)


@pytest.mark.parametrize('model', sorted(MODELS))
def test_models_edge_shapes_and_lists(model):
    n_items = 500
    act = 'softmax' if model != 'embed' else 'elu-0.5'
    mk, m = _model(n_items, act, 3, **MODELS[model])
    eng = _engine(n_items, mk, m, 8, tc=False)
    items, off, nh = _data(n_items, 60, seed=5, long_every=17)              # > 600-event histories cross staging windows
    plain, hist, keep = _pair(items, off, nh, 8)
    assert plain.n_steps > 600 and len(off) - 1 > 8
    for seen in (False, True):
        _check_against_plain(eng, plain, hist, keep, [5, 20], 0, seen, k=7)


def test_leave_one_out():
    n_items = 400
    mk, m = _model(n_items, 'tanh', 4, **MODELS['plain'])
    eng = _engine(n_items, mk, m, 12, tc=False)
    rs = np.random.RandomState(6)
    lens = rs.randint(1, 30, size=70)
    off = np.concatenate([[0], np.cumsum(lens + 1)]).astype(np.int32)
    items = rs.randint(0, n_items, size=off[-1]).astype(np.int64)
    plain, hist, keep = _pair(items, off, lens.astype(np.int32), 12)
    assert hist.n_events == 70
    for seen in (False, True):
        _check_against_plain(eng, plain, hist, keep, [10], 3, seen, k=5)


def _seen_sets(sched):
    """the seen set of every event of the schedule in (step, lane) order: its slot's inputs since its zero-before flag"""
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


def _float64_bar(m, sched, lanes, seen):
    """per event of the schedule: items surely above the target's float64 score and items within the tolerance of it (the target
    included unless seen), over the eligible items"""
    e = sched.export()
    H = [np.zeros((lanes, L), dtype=np.float32) for L in m.layers]
    sure, amb, j = [], [], 0
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        m.predict_step(e['X'][s, :M].astype(np.int64), H, slots=e['slots'][s, :M].astype(np.int64), zero=(e['F'][s, :M] & 2) != 0)
        y = H[-1][e['slots'][s, :M]].astype(np.float64)
        sc = y @ m.Wy.astype(np.float64).T + m.By.reshape(-1).astype(np.float64)
        for b in range(M):
            row = np.delete(sc[b], seen[j + b])
            t = sc[b, int(e['Y'][s, b])]
            tol = 1e-5 * (abs(t) + 1.0)
            sure.append((row > t + tol).sum()); amb.append((np.abs(row - t) <= tol).sum())
        j += M
    return np.array(sure), np.array(amb)


@pytest.mark.parametrize('seen_on', [False, True])
def test_wgmma_counts_within_float64_bar_and_equal_fp32(seen_on):
    """the blocks of 128 rows take the wgmma tiles (one more launch per block than the fp32 tiles: k_tc_split + k_eval_tc against
    k_eval_score); their counts lie within the float64 bar and equal the fp32 counts wherever the bar is unambiguous"""
    n_items, lanes = 4096, 128
    mk, m = _model(n_items, 'linear', 7, **MODELS['plain'])
    eng_tc = _engine(n_items, mk, m, lanes, tc=None)
    eng_f = _engine(n_items, mk, m, lanes, tc=False)
    items, off, nh = _data(n_items, 400, seed=8)
    plain, hist, keep = _pair(items, off, nh, lanes)
    _events(eng_tc, hist, [20], 0, 0, seen_on)                               # the item table's split, once
    n0 = eng_tc.kernel_launches(); ch = _events(eng_tc, hist, [20], 0, 0, seen_on)[3]; n_tc = eng_tc.kernel_launches() - n0
    cf = _check_against_plain(eng_f, plain, hist, keep, [20], 0, seen_on)
    n0 = eng_f.kernel_launches(); _events(eng_f, hist, [20], 0, 0, seen_on); n_f = eng_f.kernel_launches() - n0
    full_blocks = hist.n_events // lanes
    assert full_blocks >= 5 and n_tc - n_f >= full_blocks, (n_tc, n_f, full_blocks)
    seen = _seen_sets(plain) if seen_on else [np.zeros(0, np.int64)] * plain.n_events
    sure, amb = _float64_bar(m, plain, lanes, seen)
    sure, amb = sure[keep], amb[keep]
    miss = ch[:, 0] < 0
    np.testing.assert_array_equal(miss, cf[:, 0] < 0)
    if seen_on:
        assert miss.any()
    g = ch[~miss, 0]
    assert np.all(g >= sure[~miss]) and np.all(g <= sure[~miss] + amb[~miss])
    clear = ~miss & (amb == 1)
    assert clear.mean() > 0.5
    np.testing.assert_array_equal(ch[clear], cf[clear])


def test_ranking_launches_follow_counted_events():
    n_items = 300
    mk, m = _model(n_items, 'softmax', 9, **MODELS['plain'])
    lanes = 16
    eng = _engine(n_items, mk, m, lanes, tc=False)
    n_sess = 64
    off = (np.arange(n_sess + 1) * 301).astype(np.int32)                   # 300 history events and one test event each
    items = np.random.RandomState(10).randint(0, n_items, size=off[-1]).astype(np.int64)
    nh = np.full(n_sess, 300, np.int32)
    plain, hist, keep = _pair(items, off, nh, lanes)
    assert hist.n_events == n_sess
    l0 = eng.kernel_launches(); eng.eval_schedule(plain, [20]); l1 = eng.kernel_launches()
    eng.eval_schedule(hist, [20]); l2 = eng.kernel_launches()
    per_step_plain = (l1 - l0) / plain.n_steps                              # forward + 3 ranking launches per step
    fwd = per_step_plain - 3
    assert fwd == int(fwd) and fwd >= 2
    windows = -(-hist.n_steps // 512)
    ranking = (l2 - l1) - hist.n_steps * fwd
    assert ranking <= (windows + n_sess / lanes) * 8, (ranking, windows, n_sess / lanes)
    assert (l1 - l0) - plain.n_steps * fwd >= 3 * plain.n_steps


def test_determinism_and_budget(monkeypatch):
    n_items = 300
    mk, m = _model(n_items, 'softmax', 11, **MODELS['plain'])
    eng = _engine(n_items, mk, m, 16, tc=False)
    items, off, nh = _data(n_items, 80, seed=12)
    plain, hist, keep = _pair(items, off, nh, 16)
    a = _events(eng, hist, [5, 20], 3, 4, True)
    b = _events(eng, hist, [5, 20], 3, 4, True)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
    monkeypatch.setenv('G4R_SEEN_BUDGET', '64')
    eng2 = _engine(n_items, mk, m, 16, tc=False)
    l0 = eng2.kernel_launches()
    with pytest.raises(NotImplementedError):
        _events(eng2, hist, [20], 0, 0, True)
    assert eng2.kernel_launches() == l0


def test_evaluate_functions_end_to_end():
    import gru4rec
    import evaluation
    from gru4rec_b200.synth import make_sessions
    train = make_sessions(n_items=200, n_events=6000, seed=3)
    gru = gru4rec.GRU4Rec(loss='cross-entropy', final_act='softmax', layers=[32], batch_size=32, n_epochs=1, n_sample=0)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
    rs = np.random.RandomState(4)
    ids = gru.itemidmap.index.values
    hist = pd.DataFrame([(s, rs.choice(ids), float(j)) for s in range(150) for j in range(rs.randint(0, 8))], columns=['SessionId', 'ItemId', 'Time'])
    test = pd.DataFrame([(s, rs.choice(ids), float(j)) for s in range(150) for j in range(rs.randint(1, 4))], columns=['SessionId', 'ItemId', 'Time'])
    both = pd.concat([hist.assign(t=0), test.assign(t=1)]).sort_values(['SessionId', 't', 'Time'], kind='stable').reset_index(drop=True)
    both['Time'] = np.arange(len(both), dtype=np.float64)
    with contextlib.redirect_stdout(io.StringIO()):
        for mode in ('standard', 'tiebreaking'):
            res = evaluation.evaluate_events(gru, test.copy(), history=hist.copy(), cut_off=[5, 20], batch_size=20, mode=mode, k=5, exclude_seen=True)
            ref = evaluation.evaluate_events(gru, both.drop(columns='t'), cut_off=[5, 20], batch_size=20, mode=mode, k=5, exclude_seen=True)
            rec, mrr = evaluation.evaluate_gpu(gru, test.copy(), history=hist.copy(), cut_off=[5, 20], batch_size=20, mode=mode, exclude_seen=True)
            keep = both.t.values[1:][both.SessionId.values[1:] == both.SessionId.values[:-1]] == 1
            np.testing.assert_array_equal(res['events']['rank'].values, ref['events']['rank'].values[keep])
            np.testing.assert_array_equal(res['events']['input_item'].values, ref['events']['input_item'].values[keep])
            np.testing.assert_array_equal(res['topk_items'], ref['topk_items'][keep])
            assert rec == res['recall'] and mrr == res['mrr']
        plain = evaluation.evaluate_gpu(gru, test.copy(), cut_off=[5, 20], batch_size=20)
        for h in (None, hist.iloc[:0]):
            assert evaluation.evaluate_gpu(gru, test.copy(), cut_off=[5, 20], batch_size=20, history=h) == plain


def _replay_sessions(eng, items, off, nh, k, seen_on, lanes):
    """every counted event's list from the session store: each session's inputs fed in order, recommend_sessions (sessions_topk)
    at the inputs whose target lies past the history.  Returns {input position: (items, scores)}"""
    lens = np.diff(off).astype(np.int64)
    eng.sessions_open(len(lens))
    out = {}
    for j in range(int(lens.max()) - 1):
        act = np.flatnonzero(lens - 1 > j)
        cnt = j + 1 >= nh[act]
        f = act[~cnt]
        if len(f):
            eng.sessions_feed(f, items[off[f] + j])
        t = act[cnt]
        for c0 in range(0, len(t), lanes):
            c = t[c0:c0 + lanes]
            it, sc = eng.sessions_topk(c, items[off[c] + j], k, exclude_seen=seen_on)
            for r, ss in enumerate(c):
                out[int(off[ss]) + j] = (it[r], sc[r])
    eng.sessions_end()
    return out


@pytest.mark.parametrize('act,seen_on', [('linear', True), ('softmax', True), ('linear', False)])
def test_overflow_rescoring_of_blocks_equals_session_replay(act, seen_on, monkeypatch):
    """scores rising with the item index overflow the survivor lists of nearly every row, which is then rescored at the end of its
    per-event window from its saved y row; with exclude_seen its seen set is rebuilt from the schedule at the row's own step and
    lane.  More than 512 steps, sessions over the top items with histories of 0 to all but one of their events.  The lists equal
    an independent replay through the session store, and are bitwise the same for per-event windows of 512, 1 and 7 blocks.  The
    launch counts show the rescoring of nearly every block (full blocks of `lanes` rows rescore in the same number of chunks
    whatever the window, so they cannot show the window length)"""
    from test_gpu_eval_seen import _windowed
    n_items, lanes, k = 20000, 10, 20
    rising = np.linspace(-1, 1, n_items, dtype=np.float32).reshape(-1, 1)
    mk, m = _model(n_items, act, 6, layers=[16])
    m.By[:] = rising
    m.Wy[:] = (m.Wy * np.float32(1e-3)).astype(np.float32)
    rs = np.random.RandomState(10)
    lens = np.where(np.arange(560) % 5 == 0, 25, rs.randint(2, 12, size=560))
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    items = rs.randint(n_items - 40, n_items, size=int(off[-1])).astype(np.int64)
    nh = np.array([rs.randint(0, n) for n in lens], np.int32)
    hist = _lib.Schedule(items, off, None, lanes, 0, mode=1 | _lib.SCHED_POSITIONS, n_history=nh)
    assert hist.n_steps > 512
    pos = hist.positions()[hist.counted()]
    twin = _engine(n_items, mk, m, lanes)
    rep = _replay_sessions(twin, items, off, nh, k, seen_on, lanes)
    twin.close()
    e_items = np.stack([rep[int(p)][0] for p in pos]); e_scores = np.stack([rep[int(p)][1] for p in pos])
    for tc in (False, True):
        got, resc = {}, {}
        for window in (None, 1, 7):
            eng = _engine(n_items, mk, m, lanes, tc) if window is None else _windowed(n_items, mk, m, lanes, tc, window, hist, monkeypatch)
            got[window] = _events(eng, hist, [1, 20], 2, k, seen_on)
            d = []
            for b in (rising, -rising):                                   # reversed scores: nothing overflows
                eng.set('By', b)
                n0 = eng.kernel_launches()
                _events(eng, hist, [20], 0, k, seen_on)
                d.append(eng.kernel_launches() - n0)
            resc[window] = d[0] - d[1]
            eng.close()
        # nearly every block overflows and is rescored, in chunks of at most `lanes` rows (4 launches each), whatever the window
        assert all(r >= 4 * int(0.9 * hist.n_events / lanes) for r in resc.values()), resc
        items_got, scores_got = got[None][4:]
        np.testing.assert_array_equal(items_got, e_items, err_msg='eval_tc=%s' % tc)
        if act == 'softmax':
            np.testing.assert_allclose(scores_got, e_scores, rtol=1e-5, atol=0)
        else:
            np.testing.assert_array_equal(scores_got.view(np.uint32), e_scores.view(np.uint32))
        for window in (1, 7):
            for a, b in zip(got[None], got[window]):
                if isinstance(a, np.ndarray):
                    np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8), err_msg='eval_tc=%s window=%s' % (tc, window))
                else:
                    assert a == b
