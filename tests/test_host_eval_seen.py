"""CPU tests of evaluate_gpu / evaluate_events(exclude_seen=True) on the engine double (tests/oracle_engine.py, extended here by
set_eval_exclude_seen and an exclude_seen ranking made of the double's own forward): misses exactly where the target is in the
session's history after unknown items are dropped, inf ranks and NDCG, items= with duplicates, None padding and coverage, the
library's refusal as a ValueError, a 2-process gloo evaluate_gpu and run.py --exclude_seen.  The device path is tested in
test_gpu_eval_seen.py; the C ABI symbol from a C99 caller at the end."""
import contextlib
import io
import os
import shutil
import subprocess

import numpy as np
import pandas as pd
import pytest
import torch.multiprocessing as mp

from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
import oracle_engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class SeenOracleEngine(oracle_engine.OracleEngine):
    """the engine double plus exclude_seen: per-event counts over the eligible columns (the catalogue or the candidate list
    without the session's inputs so far), (-1, -1) for a target among them, and top-k lists over the eligible items"""
    seen_on = False

    def set_eval_exclude_seen(self, on):
        self.seen_on = bool(on)

    def _pass(self, sched, k=0):
        m, e = self.m, sched.export()
        if self.seen_on:
            longest, run = 1, {}
            for s in range(sched.n_steps):
                for b in range(int(e['M'][s])):
                    sl = int(e['slots'][s, b])
                    run[sl] = 1 if (e['F'][s, b] & 2 or sl not in run) else run[sl] + 1
                    longest = max(longest, run[sl])
            budget = min(256 << 20, int(os.environ.get('G4R_SEEN_BUDGET', 256 << 20)))
            if sched.batch_size * longest * 4 > budget:                 # the library's refusal (G4R_ERR_INVALID)
                raise NotImplementedError('exclude_seen: seen lists over the budget')
        H = [np.zeros((sched.batch_size, L), dtype=np.float32) for L in m.layers]
        cols = np.arange(m.Wy.shape[0]) if self.eval_items is None else self.eval_items
        cand = None if self.eval_items is None else np.unique(self.eval_items)
        seen, counts, items, scores = {}, [], [], []
        for s in range(sched.n_steps):
            M = int(e['M'][s])
            X, Y = e['X'][s, :M].astype(np.int64), e['Y'][s, :M].astype(np.int64)
            slots, zero = e['slots'][s, :M].astype(np.int64), (e['F'][s, :M] & 2) != 0
            for b in range(M):
                if zero[b] or slots[b] not in seen:
                    seen[slots[b]] = set()
                seen[slots[b]].add(int(X[b]))
            H0 = [h.copy() for h in H]
            ycols = None if self.eval_items is None else np.concatenate([Y, self.eval_items])
            yhat = m.predict_step(X, H, slots=slots, zero=zero, Y=ycols)
            tg = yhat[np.arange(M), Y if ycols is None else np.arange(M)]
            others = yhat if ycols is None else yhat[:, M:]
            for b in range(M):
                sb = np.array(sorted(seen[slots[b]])) if self.seen_on else np.zeros(0, np.int64)
                if np.isin(Y[b], sb):
                    counts.append((-1, -1))
                    continue
                keep = ~np.isin(cols, sb)
                counts.append(((others[b, keep] > tg[b]).sum(), (others[b, keep] == tg[b]).sum()))
            if k:
                sc = m.predict_step(X, H0, slots=slots, zero=zero, Y=cand)
                ids = np.arange(sc.shape[1]) if cand is None else cand
                for b in range(M):
                    sb = np.array(sorted(seen[slots[b]])) if self.seen_on else np.zeros(0, np.int64)
                    ok = np.flatnonzero(~np.isin(ids, sb))
                    best = ok[np.argsort(-sc[b, ok], kind='stable')[:k]]
                    it = np.full(k, -1, np.int32); sv = np.full(k, np.nan, np.float32)
                    it[:len(best)] = ids[best]; sv[:len(best)] = sc[b, best]
                    items.append(it); scores.append(sv)
        counts = np.array(counts, np.int32).reshape(-1, 2)
        return counts, (np.array(items) if k else None), (np.array(scores) if k else None)

    def eval_schedule(self, sched, cuts, mode=0):
        if not self.seen_on:
            return oracle_engine.OracleEngine.eval_schedule(self, sched, cuts, mode)
        counts = self._pass(sched)[0]
        gt, eq = counts[:, 0].astype(np.float64), counts[:, 1].astype(np.float64)
        rk = gt + eq if mode == 1 else gt + 0.5 * (eq - 1.0) + 1.0 if mode == 2 else gt + 1.0
        rk[counts[:, 0] < 0] = np.inf
        with np.errstate(divide='ignore'):
            rec = np.array([(rk <= c).sum() for c in cuts], np.float64)
            mrr = np.array([(1.0 / rk[rk <= c]).sum() for c in cuts], np.float64)
        return rec, mrr, len(counts)

    def eval_events(self, sched, cuts, mode=0, k=0):
        rec, mrr, n = self.eval_schedule(sched, cuts, mode)
        counts, items, scores = self._pass(sched, k)
        return rec, mrr, n, counts, items, scores


def _install(monkeypatch, gru):
    def make(cfg, device=0):
        return SeenOracleEngine(cfg, oracle_engine.model_kwargs_of(gru), device)
    monkeypatch.setattr(_lib, 'Engine', make)


def _test_frame(train, seed, n_sessions=60):
    """test sessions with repeated and reloaded items, item ids the model does not know and unsorted rows"""
    rs = np.random.RandomState(seed)
    known = train.ItemId.unique()
    rows = []
    for s in range(n_sessions):
        seq = [rs.choice(known)]
        for _ in range(rs.randint(1, 14)):
            u = rs.rand()
            seq.append(seq[-1] if u < 0.15 else rs.choice(seq) if u < 0.4 else 999999 if u < 0.5 else rs.choice(known))
        rows += [(5000 + s, it, float(t)) for t, it in enumerate(seq)]
    te = pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])
    return te.sample(frac=1.0, random_state=seed).reset_index(drop=True)


@pytest.fixture(scope='module')
def trained():
    import gru4rec
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    gru = gru4rec.GRU4Rec(loss='cross-entropy', final_act='softmax', layers=[12], batch_size=16, n_epochs=1, n_sample=0)
    mp_ = pytest.MonkeyPatch()
    _install(mp_, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
    mp_.undo()
    return gru, train


def _history_misses(gru, te):
    """per scored row of the sorted, merged frame: is the target among the session's inputs so far (unknown items dropped)"""
    df = pd.merge(te, pd.DataFrame({'ItemId': gru.itemidmap.index}), on='ItemId', how='inner')
    df = df.sort_values(['SessionId', 'Time', 'ItemId']).reset_index(drop=True)
    out = []
    for _, g in df.groupby('SessionId', sort=True):
        it = list(g.ItemId.values)
        out += [it[j] in it[:j] for j in range(1, len(it))]
    return np.array(out)


@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_misses_ranks_ndcg_and_sums(trained, mode, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    te = _test_frame(train, seed=11)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(gru, te.copy(), cut_off=[1, 5, 20], batch_size=7, mode=mode, exclude_seen=True)
        plain = evaluation.evaluate_events(gru, te.copy(), cut_off=[1, 5, 20], batch_size=7, mode=mode)
        rec, mrr = evaluation.evaluate_gpu(gru, te.copy(), cut_off=[1, 5, 20], batch_size=7, mode=mode, exclude_seen=True)
        rec0, mrr0 = evaluation.evaluate_gpu(gru, te.copy(), cut_off=[1, 5, 20], batch_size=7, mode=mode)
    r, r0 = res['events']['rank'].values, plain['events']['rank'].values
    miss = _history_misses(gru, te)
    assert len(r) == len(miss) and 0.1 < miss.mean() < 0.7
    np.testing.assert_array_equal(np.isinf(r), miss)                   # inf exactly for a target already input
    assert np.all(r[~miss] <= r0[~miss]) and np.any(r[~miss] < r0[~miss])
    assert (rec, mrr) != (rec0, mrr0) and (plain['recall'], plain['mrr']) == (rec0, mrr0)
    assert res['recall'] == rec and res['mrr'] == mrr
    for j, c in enumerate([1, 5, 20]):
        with np.errstate(divide='ignore'):
            assert abs(res['ndcg'][j] - np.where(r <= c, 1.0 / np.log2(r + 1.0), 0.0).mean()) <= 1e-12
        assert abs(rec[j] - np.mean(r <= c)) <= 1e-12
        assert abs(mrr[j] - np.sum(1.0 / r[r <= c]) / len(r)) <= 1e-12
    assert gru._engine.seen_on is False                                 # reset after the call


def test_items_padding_and_coverage(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    ids = gru.itemidmap.index.values
    cand = list(ids[:6]) + [ids[0]]                                     # 6 distinct candidates and a duplicate
    rs = np.random.RandomState(4)
    rows = [(s, rs.choice(ids[:6]), float(t)) for s in range(30) for t in range(rs.randint(2, 9))]
    te = pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(gru, te.copy(), items=cand, cut_off=[3], batch_size=5, mode='conservative', k=4, exclude_seen=True)
    ti, ts = res['topk_items'], res['topk_scores']
    pad = np.array([[x is None for x in row] for row in ti])
    assert ti.dtype == object and pad.any() and np.all(np.isnan(ts[pad])) and not np.isnan(ts[~pad]).any()
    assert res['coverage'] == len(set(ti[~pad])) / gru.n_items
    hist = {}
    df = te.sort_values(['SessionId', 'Time', 'ItemId'])
    for sid, g in df.groupby('SessionId'):
        hist[sid] = list(g.ItemId.values)
    ev = res['events']
    pos = ev.groupby('SessionId').cumcount().values                     # the event's index inside its session
    for j in range(len(ev)):
        seen = set(hist[ev.SessionId.values[j]][:pos[j] + 1])
        assert not (set(ti[j][~pad[j]]) & seen)
        assert set(ti[j][~pad[j]]) == set(cand) - seen or (~pad[j]).sum() == 4
        assert np.isinf(ev['rank'].values[j]) == (ev.ItemId.values[j] in seen)
    assert gru._engine.eval_items is None and gru._engine.seen_on is False


def test_refusal_names_the_longest_session(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    te = _test_frame(train, seed=5)
    longest = te[te.ItemId.isin(gru.itemidmap.index)].groupby('SessionId').size().idxmax()     # after unknown items are dropped
    monkeypatch.setenv('G4R_SEEN_BUDGET', '64')
    for call in (evaluation.evaluate_gpu, evaluation.evaluate_events):
        with contextlib.redirect_stdout(io.StringIO()), pytest.raises(ValueError, match='session %d ' % longest):
            call(gru, te.copy(), batch_size=7, exclude_seen=True)
        assert gru._engine.seen_on is False
    with contextlib.redirect_stdout(io.StringIO()):
        evaluation.evaluate_gpu(gru, te.copy(), batch_size=7)           # without exclude_seen nothing is refused


def _gloo_worker(rank, world, port, model, test, q):
    import sys
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle')); sys.path.insert(0, os.path.join(ROOT, 'tests'))
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    import torch
    import torch.distributed as dist
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.cuda.current_device = lambda: 0                         # no device needed: the engine double ignores it
    import gru4rec
    import evaluation
    gru = gru4rec.GRU4Rec.loadmodel(model)
    mpatch = pytest.MonkeyPatch()
    _install(mpatch, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        out = evaluation.evaluate_gpu(gru, pd.read_pickle(test), cut_off=[1, 5, 20], batch_size=7, exclude_seen=True)
        os.environ['G4R_SEEN_BUDGET'] = '64'                     # over the budget: every rank refuses, none waits for the others
        try:
            evaluation.evaluate_gpu(gru, pd.read_pickle(test), cut_off=[1, 5, 20], batch_size=7, exclude_seen=True)
            refused = False
        except ValueError:
            refused = True
        del os.environ['G4R_SEEN_BUDGET']
    mpatch.undo()
    q.put((rank, (out, refused)))
    dist.destroy_process_group()


def test_two_process_gloo_equals_single(trained, tmp_path, monkeypatch):
    import evaluation
    gru, train = trained
    te = _test_frame(train, seed=8)
    gru.savemodel(str(tmp_path / 'model.pickle'))
    te.to_pickle(str(tmp_path / 'test.pickle'))
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29910 + os.getpid() % 40
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, str(tmp_path / 'model.pickle'), str(tmp_path / 'test.pickle'), q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = dict(q.get(timeout=5) for _ in range(2))
    assert res[0][1] and res[1][1]
    res = {r: v[0] for r, v in res.items()}
    _install(monkeypatch, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        rec, mrr = evaluation.evaluate_gpu(gru, te.copy(), cut_off=[1, 5, 20], batch_size=7, exclude_seen=True)
    for r in (0, 1):
        np.testing.assert_allclose(res[r][0], rec, rtol=1e-12, atol=0)
        np.testing.assert_allclose(res[r][1], mrr, rtol=1e-12, atol=0)


def test_run_py_exclude_seen(trained, monkeypatch):
    import evaluation
    import run
    gru, train = trained
    _install(monkeypatch, gru)
    te = _test_frame(train, seed=9, n_sessions=600)                    # run.py scores with 512 lanes
    monkeypatch.setattr(run, 'load_data', lambda fname, args: te.copy())
    out = {}
    for flag in ([], ['--exclude_seen']):
        args = run.build_parser().parse_args(['x', '-t', 'test.tsv', '-m', '5', '20'] + flag)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            run._evaluate(gru, evaluation, args)
        out[bool(flag)] = [ln for ln in buf.getvalue().splitlines() if ln.startswith('Recall@') or ln.startswith('Starting')]
    with contextlib.redirect_stdout(io.StringIO()):
        want = {on: evaluation.evaluate_gpu(gru, te.copy(), batch_size=512, cut_off=[5, 20], exclude_seen=on) for on in (False, True)}
    for on in (False, True):
        assert out[on][1:] == ['Recall@{}: {:.6f} MRR@{}: {:.6f}'.format(c, want[on][0][i], c, want[on][1][i]) for i, c in enumerate([5, 20])]
    assert out[False][0] == 'Starting evaluation (cut-off=[5, 20], using standard mode for tiebreaking)'
    assert out[True][0].endswith(', seen items excluded)') and out[True][1:] != out[False][1:]


C_SRC = r'''
#include "g4r.h"

int main(void) {
  if (g4r_set_eval_exclude_seen(NULL, 1) != G4R_ERR_INVALID) return 1;
  if (g4r_set_eval_exclude_seen(NULL, 0) != G4R_ERR_INVALID) return 2;
  return 0;
}
'''


def test_c99_caller_of_exclude_seen(tmp_path):
    gcc = shutil.which('gcc') or shutil.which('cc')
    if gcc is None:
        pytest.skip('no C compiler')
    inc, libdir = os.path.join(ROOT, 'include'), os.path.join(ROOT, 'gru4rec_b200')
    src = tmp_path / 'caller.c'
    src.write_text(C_SRC)
    exe = str(tmp_path / 'caller')
    cuda_lib = '/usr/local/cuda/lib64'
    r = subprocess.run([gcc, '-std=c99', '-Wall', '-Wextra', '-pedantic', '-Werror', '-I' + inc, str(src), '-L' + libdir, '-lg4r',
                        '-Wl,-rpath,' + libdir, '-L' + cuda_lib, '-Wl,-rpath,' + cuda_lib, '-o', exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
