"""-m gpu: Engine.eval_events (g4r_eval_events, csrc/g4r_events.cuh).  The Recall / MRR sums must equal eval_schedule's bit for bit;
the per-event counts must agree with eval_counts and hold to a float64 bar; the top-k lists must equal a twin engine that replays
the same schedule through predict_topk mini-batch by mini-batch (same inputs, resets and lanes from the schedule's exports), on
both tile kinds, through overflowing lanes and under a forced short window."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
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


def _schedule(n_items, lanes, n_events, seed):
    d = orc.prepare_fit_data(make_sessions(n_items=n_items, n_events=n_events, seed=seed))
    return _lib.Schedule(d['data_items'] % n_items, d['offset_sessions'], None, lanes, 0, mode=1)


def _replay_topk(twin, sched, k, cand=None):
    """the lists of every event by predict_topk on the twin: lane = the event's state slot, reset where the schedule zeroes"""
    e = sched.export()
    B = sched.batch_size
    items, scores = [], []
    twin.reset_eval_hidden()
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        sl = e['slots'][s, :M]
        X = np.zeros(B, np.int32); X[sl] = e['X'][s, :M]
        R = np.zeros(B, np.uint8); R[sl] = (e['F'][s, :M] & 2) != 0
        i, sc = twin.predict_topk(X, k, R, items=cand)
        items.append(i[sl]); scores.append(sc[sl])
    return np.concatenate(items), np.concatenate(scores)


@pytest.mark.parametrize('tc', [False, True])
@pytest.mark.parametrize('with_items', [False, True])
def test_sums_equal_eval_schedule_and_counts(tc, with_items):
    n_items, lanes = 3000, 100
    mk, m = _model(n_items, 'elu-0.5', [64], seed=1)
    eng = _engine(n_items, mk, m, lanes, tc)
    sched = _schedule(n_items, lanes, 2500, seed=2)
    if with_items:
        eng.set_eval_items(np.random.RandomState(3).choice(n_items, 900))
    cuts = [1, 5, 20, 100]
    for mode in range(4):
        rec, mrr, n = eng.eval_schedule(sched, cuts, mode)
        last = eng.eval_counts(int(sched.batch_sizes()[-1]))
        r2, q2, n2, cnt, ti, ts = eng.eval_events(sched, cuts, mode)
        assert n2 == n == sched.n_events and ti is None and ts is None
        np.testing.assert_array_equal(r2.view(np.uint64), rec.view(np.uint64))
        np.testing.assert_array_equal(q2.view(np.uint64), mrr.view(np.uint64))
        np.testing.assert_array_equal(cnt[-len(last):], last)
        r3, q3, _, cnt3, ti3, _ = eng.eval_events(sched, cuts, mode, k=20)       # the lists leave the sums and counts alone
        np.testing.assert_array_equal(r3.view(np.uint64), rec.view(np.uint64))
        np.testing.assert_array_equal(q3.view(np.uint64), mrr.view(np.uint64))
        np.testing.assert_array_equal(cnt3, cnt)
        assert ti3.shape == (n, 20)
    eng.close()


def test_counts_hold_to_float64():
    """every event: #greater within [sure, sure + ambiguous] of a float64 restatement (scores of the float32 oracle forward taken in
    float64; within 1e-5 of the target counts as ambiguous); fp32 and wgmma tiles agree exactly where nothing is ambiguous"""
    n_items, lanes = 2500, 64
    mk, m = _model(n_items, 'linear', [32], seed=4)
    sched = _schedule(n_items, lanes, 900, seed=5)
    out = {}
    for tc in (False, True):
        eng = _engine(n_items, mk, m, lanes, tc)
        out[tc] = eng.eval_events(sched, [20], 0)[3]
        eng.close()
    e = sched.export()
    H = [np.zeros((lanes, L), dtype=np.float32) for L in m.layers]
    rows = []
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        X, Y = e['X'][s, :M].astype(np.int64), e['Y'][s, :M]
        m.predict_step(X, H, slots=e['slots'][s, :M].astype(np.int64), zero=(e['F'][s, :M] & 2) != 0)
        y = np.concatenate([H[-1][e['slots'][s, :M]]], 0).astype(np.float64)
        sc = y @ m.Wy.astype(np.float64).T + m.By.reshape(-1).astype(np.float64)
        t = sc[np.arange(M), Y][:, None]
        tol = 1e-5 * (np.abs(t) + 1.0)
        rows.append(np.stack([(sc > t + tol).sum(1), (np.abs(sc - t) <= tol).sum(1)], 1))
    sure, amb = np.concatenate(rows)[:, 0], np.concatenate(rows)[:, 1]
    for tc, cnt in out.items():
        assert np.all(cnt[:, 0] >= sure) and np.all(cnt[:, 0] <= sure + amb), 'eval_tc=%s' % tc
    clear = amb == 1                                          # only the target itself within the tolerance
    assert clear.mean() > 0.5
    np.testing.assert_array_equal(out[False][clear], out[True][clear])


# n_items, layers, lanes, act, k, By, extra model arguments
CASES = [
    (3000, [48], 1, 'elu-0.5', 20, None, {}),
    (2049, [64], 33, 'relu', 20, -0.35, {}),                     # zero ties and a padded last tile
    (4100, [40], 129, 'selu-1.05-1.67', 100, None, {}),
    (3000, [32], 512, 'tanh', 20, None, {}),
    (2500, [48, 24], 64, 'elu-0.5', 20, None, {}),               # two layers
    (3000, [64], 96, 'linear', 20, None, dict(constrained_embedding=True)),
    (3000, [64], 100, 'softmax', 20, None, {}),
    (3000, [64], 100, 'softmax_logit', 20, None, {}),
]


@pytest.mark.parametrize('n_items,layers,lanes,act,k,by,extra',
                         [pytest.param(*c, id='%d-%s-%d-%s-k%d' % (c[0], 'x'.join(map(str, c[1])), c[2], c[3], c[4])) for c in CASES])
def test_lists_equal_predict_topk_replay(n_items, layers, lanes, act, k, by, extra):
    mk, m = _model(n_items, act, layers, seed=6, by=by, **extra)
    sched = _schedule(n_items, lanes, max(6 * lanes, 600), seed=7)
    twin = _engine(n_items, mk, m, lanes)
    e_items, e_scores = _replay_topk(twin, sched, k)
    twin.close()
    for tc in (False, True):
        eng = _engine(n_items, mk, m, lanes, tc)
        _, _, n, _, items, scores = eng.eval_events(sched, [20], 0, k=k)
        assert n == len(e_items)
        np.testing.assert_array_equal(items, e_items, err_msg='eval_tc=%s' % tc)
        if act.startswith('softmax'):
            np.testing.assert_allclose(scores, e_scores, rtol=1e-5, atol=0, err_msg='eval_tc=%s' % tc)
        else:
            np.testing.assert_array_equal(scores.view(np.uint32), e_scores.view(np.uint32), err_msg='eval_tc=%s' % tc)
        eng.close()


@pytest.mark.parametrize('tc', [False, True])
def test_lists_with_candidate_items(tc):
    n_items, lanes, k = 3000, 80, 20
    mk, m = _model(n_items, 'softmax', [48], seed=8)
    sched = _schedule(n_items, lanes, 900, seed=9)
    for cand in (np.random.RandomState(1).choice(n_items, 1500), np.arange(0, n_items, 7)):   # tiles / prefix holds every candidate
        twin = _engine(n_items, mk, m, lanes)
        e_items, e_scores = _replay_topk(twin, sched, k, cand=cand.astype(np.int32))
        twin.close()
        eng = _engine(n_items, mk, m, lanes, tc)
        eng.set_eval_items(cand)
        items = eng.eval_events(sched, [20], 0, k=k)
        np.testing.assert_array_equal(items[4], e_items)
        np.testing.assert_allclose(items[5], e_scores, rtol=1e-5, atol=0)
        eng.close()


def _overflow_windows(sched, window):
    """per-event windows of `window` mini-batches over the schedule (within one staging window of 512)"""
    return -(-sched.n_steps // window)


@pytest.mark.parametrize('act', ['linear', 'softmax'])
def test_overflow_and_short_windows(act, monkeypatch):
    """scores rising with the item index: the lanes of every window overflow their survivor lists (the deferred rescoring
    launches four kernels per chunk of at most 16 overflowed lanes: counted against falling scores, where nothing overflows) and
    are rescored at the end of their window; the lists stay exact, and windows of 3 mini-batches give bitwise the same outputs"""
    n_items, lanes, k = 20000, 16, 20
    rising = np.linspace(-1, 1, n_items, dtype=np.float32).reshape(-1, 1)
    mk, m = _model(n_items, act, [16], seed=6, by=rising, wy_scale=1e-3)
    sched = _schedule(n_items, lanes, 400, seed=10)
    assert sched.n_steps > 6
    twin = _engine(n_items, mk, m, lanes)
    e_items, e_scores = _replay_topk(twin, sched, k)
    twin.close()

    def run(eng, by):
        eng.set('By', by)
        n0 = eng.kernel_launches()
        out = eng.eval_events(sched, [1, 20], 2, k=k)
        return out, eng.kernel_launches() - n0

    for tc in (False, True):
        eng = _engine(n_items, mk, m, lanes, tc)
        full, d_rising = run(eng, rising)
        _, d_falling = run(eng, rising[::-1].copy())
        eng.close()
        assert d_rising - d_falling >= 4 * -(-int(0.9 * sched.n_events) // lanes)     # nearly every lane overflowed
        np.testing.assert_array_equal(full[4], e_items)
        if act == 'softmax':
            np.testing.assert_allclose(full[5], e_scores, rtol=1e-5, atol=0)
        else:
            np.testing.assert_array_equal(full[5].view(np.uint32), e_scores.view(np.uint32))
        monkeypatch.setenv('G4R_EVENTS_WINDOW', '3')
        short = _engine(n_items, mk, m, lanes, tc)
        monkeypatch.delenv('G4R_EVENTS_WINDOW')
        got, d_short = run(short, rising)
        _, d_short_falling = run(short, rising[::-1].copy())
        short.close()
        assert d_short - d_short_falling >= 4 * _overflow_windows(sched, 3)              # in every window
        for a, b in zip(full, got):
            if isinstance(a, np.ndarray):
                np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8))
            else:
                assert a == b


@pytest.mark.parametrize('tc', [False, True])
def test_tied_scores_independent_of_window(tc, monkeypatch):
    """relu below zero: most targets tie with many items, so 'tiebreaking' counts depend on the tie noise, which hashes the
    mini-batch's step.  A schedule of more than 512 mini-batches (two staging windows), per-event windows of 7 mini-batches that do
    not divide them: the sums equal eval_schedule's in every mode, and counts and lists equal those of the default window"""
    n_items, lanes = 600, 16
    mk, m = _model(n_items, 'relu', [16], seed=12, by=-0.35)
    sched = _schedule(n_items, lanes, 16000, seed=13)
    assert sched.n_steps > 512
    eng = _engine(n_items, mk, m, lanes, tc)
    monkeypatch.setenv('G4R_EVENTS_WINDOW', '7')
    short = _engine(n_items, mk, m, lanes, tc)
    monkeypatch.delenv('G4R_EVENTS_WINDOW')
    cuts = [5, 20, 100]
    greater = {}
    for mode in range(4):
        rec, mrr, n = eng.eval_schedule(sched, cuts, mode)
        a = eng.eval_events(sched, cuts, mode, k=10)
        b = short.eval_events(sched, cuts, mode, k=10)
        for got in (a, b):
            np.testing.assert_array_equal(got[0].view(np.uint64), rec.view(np.uint64), err_msg='mode %d' % mode)
            np.testing.assert_array_equal(got[1].view(np.uint64), mrr.view(np.uint64), err_msg='mode %d' % mode)
        for x, y in zip(a[3:], b[3:]):
            np.testing.assert_array_equal(x, y, err_msg='mode %d' % mode)
        greater[mode] = a[3][:, 0]
    assert (greater[3] != greater[0]).mean() > 0.2                # the noise decides many ties
    eng.close(); short.close()


def test_other_scoring_paths_unchanged_by_eval_events():
    n_items, lanes = 3000, 64
    mk, m = _model(n_items, 'elu-0.5', [48], seed=11)
    eng = _engine(n_items, mk, m, lanes)
    sched = _schedule(n_items, lanes, 800, seed=12)
    X = np.random.RandomState(13).randint(0, n_items, lanes).astype(np.int32)

    def run():
        r = eng.eval_schedule(sched, [5, 20], 0)
        eng.reset_eval_hidden()
        p = eng.predict(X)
        eng.reset_eval_hidden()
        t = eng.predict_topk(X, 10)
        return r[:2] + (p,) + t
    before = run()
    eng.eval_events(sched, [5, 20], 0, k=50)
    after = run()
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a, b)
    eng.close()
