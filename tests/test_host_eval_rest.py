"""CPU tests of evaluate_rest on the engine double (tests/oracle_engine.py with the exclude_seen and history ranking of
test_host_eval_history.py), extended here by an eval_rest computed in float64 NumPy from the schedule's positions: the relevant
sets against a plain pandas restatement on messy data, the metric formulas against a direct per-event restatement (median
halves, the |R| = 1 reduction), items= / exclude_seen / history= misses, the budget refusal, the baseline and 2-process
refusals and run.py --rest_of_session.  The device path is tested in test_gpu_eval_rest.py."""
import contextlib
import io
import os

import numpy as np
import pandas as pd
import pytest
import torch.multiprocessing as mp

from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
import oracle_engine
from test_host_eval_history import HistOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rank_of(counts, mode):
    gt, eq = counts[:, 0].astype(np.float64), counts[:, 1].astype(np.float64)
    r = gt + eq if mode == 1 else gt + 0.5 * (eq - 1.0) + 1.0 if mode == 2 else gt + 1.0
    r[counts[:, 0] < 0] = np.inf
    return r


def event_metrics(r, n, N):
    """the six metrics of one event: r the ranks of its relevant items (inf: miss), n = |R|"""
    hit = np.sort(r[r <= N])
    m = min(n, N)
    idcg = sum(1.0 / np.log2(i + 1.0) for i in range(1, m + 1))
    ap = sum((r <= x).sum() / x for x in hit)
    return np.array([float(len(hit) > 0), len(hit) / N, len(hit) / n, 1.0 / hit[0] if len(hit) else 0.0,
                     sum(1.0 / np.log2(x + 1.0) for x in hit) / idcg, ap / m])


class RestOracleEngine(HistOracleEngine):
    """eval_rest of the double: every counted event's relevant items from the schedule's positions, each ranked in float64
    against the eligible columns as if it were the target"""

    def eval_rest(self, sched, cuts, mode=0):
        m, e, P = self.m, sched.export(), sched.positions()
        run, longest = {}, 1
        for s in range(sched.n_steps):
            for b in range(int(e['M'][s])):
                sl = int(e['slots'][s, b])
                run[sl] = 1 if (e['F'][s, b] & 2 or sl not in run) else run[sl] + 1
                longest = max(longest, run[sl])
        budget = min(256 << 20, int(os.environ.get('G4R_SEEN_BUDGET', 256 << 20)))
        if sched.batch_size * longest * 4 > budget:                     # the library's refusal (G4R_ERR_INVALID)
            raise NotImplementedError('eval_rest: relevant lists over the budget')
        rows = int(P.max()) + 2
        item, nx = np.full(rows, -1, np.int64), np.zeros(rows, bool)
        for s in range(sched.n_steps):
            M = int(e['M'][s])
            item[P[s, :M]], item[P[s, :M] + 1], nx[P[s, :M]] = e['X'][s, :M], e['Y'][s, :M], True
        H = [np.zeros((sched.batch_size, L), dtype=np.float32) for L in m.layers]
        cols = np.arange(m.Wy.shape[0]) if self.eval_items is None else np.asarray(self.eval_items)
        seen, counts, offsets = {}, [], [0]
        for s in range(sched.n_steps):
            M = int(e['M'][s])
            X = e['X'][s, :M].astype(np.int64)
            slots, zero = e['slots'][s, :M].astype(np.int64), (e['F'][s, :M] & 2) != 0
            for b in range(M):
                if zero[b] or slots[b] not in seen:
                    seen[slots[b]] = set()
                seen[slots[b]].add(int(X[b]))
            yhat = m.predict_step(X, H, slots=slots, zero=zero).astype(np.float64)
            for b in range(M):
                if sched.history and not e['F'][s, b] & 4:
                    continue
                rel, q = [], int(P[s, b]) + 1
                while True:
                    if item[q] not in rel:
                        rel.append(int(item[q]))
                    if not nx[q]:
                        break
                    q += 1
                sb = seen[slots[b]] if self.seen_on else set()
                comp = yhat[b, cols[~np.isin(cols, list(sb))]]
                for j in rel:
                    if j in sb or j not in set(cols.tolist()):
                        counts.append((-1, -1))
                    else:
                        counts.append(((comp > yhat[b, j]).sum(), (comp == yhat[b, j]).sum()))
                offsets.append(offsets[-1] + len(rel))
        counts, offsets = np.array(counts, np.int32).reshape(-1, 2), np.array(offsets, np.int64)
        sums = np.zeros((6, len(cuts)))
        r = rank_of(counts, mode)
        for i in range(len(offsets) - 1):
            for j, N in enumerate(cuts):
                sums[:, j] += event_metrics(r[offsets[i]:offsets[i + 1]], offsets[i + 1] - offsets[i], N)
        return sums, len(offsets) - 1, len(counts), counts, offsets


def _install(monkeypatch, gru):
    def make(cfg, device=0):
        return RestOracleEngine(cfg, oracle_engine.model_kwargs_of(gru), device)
    monkeypatch.setattr(_lib, 'Engine', make)


@pytest.fixture(scope='module')
def trained():
    import gru4rec
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    train['ItemId'] = train.ItemId.map(lambda i: 'it%d' % i)            # string ids
    gru = gru4rec.GRU4Rec(loss='cross-entropy', final_act='softmax', layers=[12], batch_size=16, n_epochs=1, n_sample=0)
    mp_ = pytest.MonkeyPatch()
    _install(mp_, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
    mp_.undo()
    return gru, train


def _messy(train, seed, n_sessions=40):
    """test sessions with repeated items, unknown items, length-1 sessions and shuffled rows"""
    rs = np.random.RandomState(seed)
    known = train.ItemId.unique()
    rows = []
    for s in range(n_sessions):
        seq = [rs.choice(known)]
        for _ in range(0 if s % 7 == 0 else rs.randint(1, 12)):
            u = rs.rand()
            seq.append(seq[-1] if u < 0.15 else rs.choice(seq) if u < 0.4 else 'unknown' if u < 0.5 else rs.choice(known))
        rows += [(3000 + s, it, float(t)) for t, it in enumerate(seq)]
    te = pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])
    return te.sample(frac=1.0, random_state=seed).reset_index(drop=True)


def _pandas_pairs(gru, test):
    """the relevant sets restated: known rows sorted by session, time and item; for every row but a session's last, the distinct
    later items of its session with the offset of their first occurrence"""
    t = test[test.ItemId.isin(gru.itemidmap.index)].sort_values(['SessionId', 'Time', 'ItemId']).reset_index(drop=True)
    out = []
    for sid, g in t.groupby('SessionId', sort=True):
        its, tm = g.ItemId.tolist(), g.Time.tolist()
        for p in range(len(its) - 1):
            first = {}
            for q in range(p + 1, len(its)):
                first.setdefault(its[q], q - p)
            out += [(sid, tm[p + 1], its[p], it, o) for it, o in first.items()]
    return pd.DataFrame(out, columns=['SessionId', 'Time', 'input_item', 'ItemId', 'offset'])


def _rest(gru, test, **kw):
    import evaluation
    with contextlib.redirect_stdout(io.StringIO()):
        return evaluation.evaluate_rest(gru, test.copy(), **kw)


def test_relevant_sets_on_messy_data(trained, monkeypatch):
    gru, train = trained
    _install(monkeypatch, gru)
    test = _messy(train, seed=5)
    res = _rest(gru, test, batch_size=5)
    want = _pandas_pairs(gru, test)
    got = res['pairs']
    assert list(got.columns) == ['SessionId', 'Time', 'input_item', 'ItemId', 'offset', 'rank']
    pd.testing.assert_frame_equal(got.drop(columns='rank').reset_index(drop=True), want, check_dtype=False)
    assert res['n_pairs'] == len(want) and res['n_events'] == int((want.offset == 1).sum())
    assert got['rank'].dtype == np.float64 and np.isfinite(got['rank']).all()
    assert (got.groupby(['SessionId']).offset.min() == 1).all()


@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_metric_formulas(trained, mode, monkeypatch):
    gru, train = trained
    _install(monkeypatch, gru)
    test = _messy(train, seed=11)
    cuts = [1, 3, 10]
    res = _rest(gru, test, batch_size=4, cut_off=cuts, mode=mode)
    p = res['pairs']
    ev = (p.offset == 1).cumsum().values                               # every event's pairs start with its next item
    n_ev = ev.max()
    assert res['n_events'] == n_ev and res['n_pairs'] == len(p)
    tot = np.zeros((6, len(cuts)))
    for k in range(1, n_ev + 1):
        r = p['rank'].values[ev == k]
        for j, N in enumerate(cuts):
            tot[:, j] += event_metrics(r, len(r), N)
    for i, name in enumerate(['hitrate', 'precision', 'recall', 'mrr', 'ndcg', 'map']):
        np.testing.assert_allclose(res[name], tot[i] / n_ev, rtol=1e-12, atol=0)


def test_reduction_to_next_item(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    rs = np.random.RandomState(2)
    known = train.ItemId.unique()
    rows = [(100 + s, it, float(t)) for s in range(30) for t, it in enumerate(rs.choice(known, 2, replace=False))]
    test = pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])
    cuts = [1, 5, 20]
    for mode in ('standard', 'conservative', 'median'):
        res = _rest(gru, test, batch_size=7, cut_off=cuts, mode=mode)
        with contextlib.redirect_stdout(io.StringIO()):
            rec, mrr = evaluation.evaluate_gpu(gru, test.copy(), batch_size=7, cut_off=cuts, mode=mode)
            evs = evaluation.evaluate_events(gru, test.copy(), batch_size=7, cut_off=cuts, mode=mode)
        np.testing.assert_allclose(res['hitrate'], rec, rtol=1e-12)
        np.testing.assert_allclose(res['recall'], rec, rtol=1e-12)
        np.testing.assert_allclose(res['mrr'], mrr, rtol=1e-12)
        np.testing.assert_allclose(res['map'], mrr, rtol=1e-12)
        np.testing.assert_allclose(res['ndcg'], evs['ndcg'], rtol=1e-12)
        np.testing.assert_allclose(res['precision'], np.array(rec) / np.array(cuts), rtol=1e-12)
        np.testing.assert_array_equal(res['pairs']['rank'].values, evs['events']['rank'].values)


def test_items_and_exclude_seen_misses(trained, monkeypatch):
    gru, train = trained
    _install(monkeypatch, gru)
    known = list(gru.itemidmap.index)
    a, b, c, d = known[:4]
    # one session a b a c d: from input a, relevant b, a, c, d; a is seen (the input itself), d is not listed below
    test = pd.DataFrame({'SessionId': [1] * 5, 'ItemId': [a, b, a, c, d], 'Time': np.arange(5.0)})
    listed = [x for x in known if x != d]
    res = _rest(gru, test, batch_size=1, items=listed, exclude_seen=True, cut_off=[len(known)])
    p = res['pairs']
    first = p[p.Time == 1.0]
    assert first.ItemId.tolist() == [b, a, c, d]
    r = dict(zip(first.ItemId, first['rank']))
    assert np.isinf(r[a]) and np.isinf(r[d]) and np.isfinite(r[b]) and np.isfinite(r[c])
    # the misses still count in |R|: recall of that event is at most 2 / 4
    plain = _rest(gru, test, batch_size=1, cut_off=[len(known)])
    assert np.isfinite(plain['pairs']['rank']).all()
    n_ev = res['n_events']
    rr = res['pairs']['rank'].values
    ev = (res['pairs'].offset == 1).cumsum().values
    want = np.mean([np.isfinite(rr[ev == k]).sum() / (ev == k).sum() for k in range(1, n_ev + 1)])
    assert abs(res['recall'][0] - want) < 1e-12 and res['recall'][0] < 1.0


def test_history_counts_only_test_events(trained, monkeypatch):
    from test_host_eval_history import _split
    gru, train = trained
    _install(monkeypatch, gru)
    tr = train.copy()
    hist, test = _split(tr, seed=4)
    res = _rest(gru, test, history=hist, batch_size=5)
    ref = _rest(gru, test, batch_size=5)
    import evaluation
    with contextlib.redirect_stdout(io.StringIO()):
        evs = evaluation.evaluate_events(gru, test.copy(), history=hist.copy(), batch_size=5)
    assert res['n_events'] == len(evs['events'])
    nxt = res['pairs'][res['pairs'].offset == 1]
    np.testing.assert_array_equal(nxt['rank'].values, evs['events']['rank'].values)
    assert nxt.input_item.tolist() == evs['events'].input_item.tolist()
    assert res['n_events'] >= ref['n_events']


def test_budget_names_the_session(trained, monkeypatch):
    gru, train = trained
    _install(monkeypatch, gru)
    test = _messy(train, seed=5)
    t = test[test.ItemId.isin(gru.itemidmap.index)]
    sizes = t.groupby('SessionId').size()
    longest, n = int(sizes.idxmax()), int(sizes.max())
    monkeypatch.setenv('G4R_SEEN_BUDGET', str(5 * (n - 1) * 4 - 4))
    with pytest.raises(ValueError, match='session %d ' % longest):
        _rest(gru, test, batch_size=5)
    monkeypatch.setenv('G4R_SEEN_BUDGET', str(5 * (n - 1) * 4))
    _rest(gru, test, batch_size=5)


def test_baseline_refused():
    import evaluation
    from gru4rec_b200.baselines import Pop
    with pytest.raises(NotImplementedError, match='baselines'):
        evaluation.evaluate_rest(Pop(), pd.DataFrame({'SessionId': [1, 1], 'ItemId': ['a', 'b'], 'Time': [0.0, 1.0]}))


def _gloo_worker(rank, world, port, model, test, q):
    import sys
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle')); sys.path.insert(0, os.path.join(ROOT, 'tests'))
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    import torch
    import torch.distributed as dist
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.cuda.current_device = lambda: 0
    import gru4rec
    import evaluation
    gru = gru4rec.GRU4Rec.loadmodel(model)
    mpatch = pytest.MonkeyPatch()
    _install(mpatch, gru)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            evaluation.evaluate_rest(gru, pd.read_pickle(test), batch_size=4)
        q.put((rank, 'ran'))
    except NotImplementedError as err:
        q.put((rank, 'refused: %s' % err))
    mpatch.undo()
    dist.destroy_process_group()


def test_two_process_gloo_refused(trained, tmp_path):
    gru, train = trained
    gru.savemodel(str(tmp_path / 'model.pickle'))
    _messy(train, seed=3).to_pickle(str(tmp_path / 'test.pickle'))
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29850 + os.getpid() % 40
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, str(tmp_path / 'model.pickle'), str(tmp_path / 'test.pickle'), q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = dict(q.get(timeout=5) for _ in range(2))
    assert all(v.startswith('refused: evaluate_rest runs in a single process') for v in res.values()), res


def test_run_py_rest_of_session(trained, monkeypatch):
    import evaluation
    import run
    gru, train = trained
    _install(monkeypatch, gru)
    test = _messy(train, seed=9, n_sessions=600)                 # run.py scores with 512 lanes
    monkeypatch.setattr(run, 'load_data', lambda fname, args: test.copy())
    args = run.build_parser().parse_args(['x', '-t', 'test.tsv', '-m', '5', '20', '--rest_of_session', '-e', 'conservative', '--exclude_seen'])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        run._evaluate(gru, evaluation, args)
    lines = buf.getvalue().splitlines()
    rec = [ln for ln in lines if ln.startswith('Recall@')]
    rest = [ln for ln in lines if ln.startswith('Rest@')]
    assert len(rec) == 2 and lines.index(rest[0]) > lines.index(rec[-1])
    want = _rest(gru, test, batch_size=512, cut_off=[5, 20], mode='conservative', exclude_seen=True)
    assert rest == ['Rest@{}: HitRate {:.6f} Precision {:.6f} Recall {:.6f} MAP {:.6f} NDCG {:.6f} MRR {:.6f}'.format(
        c, *(want[m][i] for m in ('hitrate', 'precision', 'recall', 'map', 'ndcg', 'mrr'))) for i, c in enumerate([5, 20])]


def test_run_py_refuses_baseline():
    import run
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf), pytest.raises(SystemExit):
        run.main(['train.tsv', '--baseline', 'pop', '-t', 'test.tsv', '--rest_of_session'])
    assert 'rest_of_session' in buf.getvalue()
