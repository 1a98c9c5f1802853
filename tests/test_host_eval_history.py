"""CPU tests of evaluate_gpu / evaluate_events(history=...) on the engine double (tests/oracle_engine.py with the exclude_seen
ranking of test_host_eval_seen.py, extended here to count only the events a history schedule flags): the schedule's counted
lanes, the frame semantics (history first whatever the times, the first row's input item), equality with the concatenated
workaround, NDCG and inf ranks, a 2-process gloo evaluate_gpu, run.py --history and the C ABI symbol from a C99 caller.  The
device path is tested in test_gpu_eval_history.py."""
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
from test_host_eval_seen import SeenOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class HistOracleEngine(SeenOracleEngine):
    """the double's per-event counts over the whole schedule, kept only for the counted lanes of a history schedule"""

    def _counted(self, sched, k=0):
        counts, items, scores = self._pass(sched, k)
        used = np.arange(sched.batch_size)[None, :] < sched.batch_sizes()[:, None]
        keep = sched.counted()[used]
        return counts[keep], (items[keep] if k else None), (scores[keep] if k else None)

    def eval_schedule(self, sched, cuts, mode=0):
        if not getattr(sched, 'history', False):
            return SeenOracleEngine.eval_schedule(self, sched, cuts, mode)
        counts = self._counted(sched)[0]
        gt, eq = counts[:, 0].astype(np.float64), counts[:, 1].astype(np.float64)
        rk = gt + eq if mode == 1 else gt + 0.5 * (eq - 1.0) + 1.0 if mode == 2 else gt + 1.0
        rk[counts[:, 0] < 0] = np.inf
        with np.errstate(divide='ignore'):
            rec = np.array([(rk <= c).sum() for c in cuts], np.float64)
            mrr = np.array([(1.0 / rk[rk <= c]).sum() for c in cuts], np.float64)
        return rec, mrr, len(counts)

    def eval_events(self, sched, cuts, mode=0, k=0):
        if not getattr(sched, 'history', False):
            return SeenOracleEngine.eval_events(self, sched, cuts, mode, k)
        rec, mrr, n = self.eval_schedule(sched, cuts, mode)
        counts, items, scores = self._counted(sched, k)
        return rec, mrr, n, counts, items, scores


def _install(monkeypatch, gru):
    def make(cfg, device=0):
        return HistOracleEngine(cfg, oracle_engine.model_kwargs_of(gru), device)
    monkeypatch.setattr(_lib, 'Engine', make)


def _split(train, seed, n_sessions=50, max_hist=9, max_test=5):
    """history and test frames: every history row is later than its session's test rows (the split, not the time, decides the
    order), some sessions without history, some history-only sessions, unknown items in both"""
    rs = np.random.RandomState(seed)
    known = train.ItemId.unique()
    hist, test = [], []
    for s in range(n_sessions):
        h = rs.randint(0, max_hist + 1) if s % 5 else 0
        t = rs.randint(1, max_test + 1)
        seq = [999999 if rs.rand() < 0.08 else rs.choice(known) for _ in range(h + t)]
        hist += [(7000 + s, it, 100.0 + j) for j, it in enumerate(seq[:h])]
        test += [(7000 + s, it, float(j)) for j, it in enumerate(seq[h:])]
    for s in range(5):                                                  # history-only sessions: ignored
        hist += [(9000 + s, rs.choice(known), float(j)) for j in range(4)]
    hist = pd.DataFrame(hist, columns=['SessionId', 'ItemId', 'Time']).sample(frac=1.0, random_state=seed).reset_index(drop=True)
    test = pd.DataFrame(test, columns=['SessionId', 'ItemId', 'Time']).sample(frac=1.0, random_state=seed + 1).reset_index(drop=True)
    return hist, test


def _concat(gru, hist, test):
    """the workaround's frame: each test session's known history rows, then its known test rows, with times that keep that order,
    and per row whether it is a test row"""
    known = set(gru.itemidmap.index)
    h = hist[hist.ItemId.isin(known) & hist.SessionId.isin(test.SessionId)].sort_values(['SessionId', 'Time', 'ItemId'])
    t = test[test.ItemId.isin(known)].sort_values(['SessionId', 'Time', 'ItemId'])
    both = pd.concat([h.assign(is_test=False), t.assign(is_test=True)]).sort_values('SessionId', kind='stable').reset_index(drop=True)
    both['Time'] = np.arange(len(both), dtype=np.float64)
    return both


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


def test_schedule_flags_counted_lanes():
    # 4 sessions (lengths 3, 5, 2, 4) with 1, 0, 2, 3 history events, 2 lanes
    offs = np.array([0, 3, 8, 10, 14], np.int32)
    items = np.arange(14, dtype=np.int64) % 7
    nh = np.array([1, 0, 2, 3], np.int32)
    plain = _lib.Schedule(items, offs, None, 2, 0, mode=1 | _lib.SCHED_POSITIONS)
    hs = _lib.Schedule(items, offs, None, 2, 0, mode=1 | _lib.SCHED_POSITIONS, n_history=nh)
    ep, eh = plain.export(), hs.export()
    for key in ('X', 'Y', 'M', 'slots'):
        np.testing.assert_array_equal(ep[key], eh[key])                 # the schedule of the concatenated data, unchanged
    np.testing.assert_array_equal(ep['F'] & 3, eh['F'] & 3)
    pos = hs.positions()
    sess = np.searchsorted(offs, pos + 1, side='right') - 1
    used = np.arange(2)[None, :] < ep['M'][:, None]
    want = used & (pos + 1 >= offs[np.clip(sess, 0, 3)] + nh[np.clip(sess, 0, 3)])
    np.testing.assert_array_equal(hs.counted(), want)
    assert hs.n_events == want.sum() == (3 - 1) + (5 - 1) + (2 - 2) + (4 - 3) and plain.n_events == used.sum()
    np.testing.assert_array_equal(plain.counted(), used)
    with pytest.raises(RuntimeError, match='longer than the session'):
        _lib.Schedule(items, offs, None, 2, 0, mode=1, n_history=np.array([1, 0, 3, 3], np.int32))
    with pytest.raises(RuntimeError, match='evaluation schedule'):
        _lib.Schedule(items, offs, None, 2, 0, mode=0, n_history=nh)


@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
@pytest.mark.parametrize('exclude_seen', [False, True])
def test_frame_equals_concatenated_workaround(trained, mode, exclude_seen, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    hist, test = _split(train, seed=21)
    both = _concat(gru, hist, test)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(gru, test.copy(), history=hist.copy(), cut_off=[1, 5, 20], batch_size=6, mode=mode, k=3, exclude_seen=exclude_seen)
        ref = evaluation.evaluate_events(gru, both.drop(columns='is_test'), cut_off=[1, 5, 20], batch_size=6, mode=mode, k=3, exclude_seen=exclude_seen)
        rec, mrr = evaluation.evaluate_gpu(gru, test.copy(), history=hist.copy(), cut_off=[1, 5, 20], batch_size=6, mode=mode, exclude_seen=exclude_seen)
    ev, rv = res['events'], ref['events']
    keep = both.is_test.values[1:][both.SessionId.values[1:] == both.SessionId.values[:-1]]   # the workaround's rows with a test target
    np.testing.assert_array_equal(ev['rank'].values, rv['rank'].values[keep])
    np.testing.assert_array_equal(ev['input_item'].values, rv['input_item'].values[keep])
    np.testing.assert_array_equal(ev['ItemId'].values, rv['ItemId'].values[keep])
    np.testing.assert_array_equal(res['topk_items'], ref['topk_items'][keep])
    r = ev['rank'].values
    for j, c in enumerate([1, 5, 20]):
        with np.errstate(divide='ignore'):
            assert abs(res['ndcg'][j] - np.where(r <= c, 1.0 / np.log2(r + 1.0), 0.0).mean()) <= 1e-12
        assert abs(rec[j] - np.mean(r <= c)) <= 1e-12 and rec[j] == res['recall'][j] and mrr[j] == res['mrr'][j]
    # counted events per session: t with history, t - 1 without; history-only sessions contribute nothing
    known = set(gru.itemidmap.index)
    tk, hk = test[test.ItemId.isin(known)], hist[hist.ItemId.isin(known)]
    for sid, g in tk.groupby('SessionId'):
        h = (hk.SessionId == sid).sum()
        assert (ev.SessionId == sid).sum() == (len(g) if h else len(g) - 1)
        if h:                                                           # the first row's input is the last history item
            last = hk[hk.SessionId == sid].sort_values(['Time', 'ItemId']).ItemId.values[-1]
            assert ev[ev.SessionId == sid].input_item.values[0] == last
    assert not ev.SessionId.isin(range(9000, 9005)).any()
    if exclude_seen:
        assert np.isinf(r).any()
    assert gru._engine.seen_on is False


def test_leave_one_out_and_seen_only_in_history(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    ids = gru.itemidmap.index.values
    hist = pd.DataFrame([(s, ids[(s + j) % 10], float(j)) for s in range(20) for j in range(3)], columns=['SessionId', 'ItemId', 'Time'])
    test = pd.DataFrame([(s, ids[s % 10] if s % 2 else ids[30 + s], 50.0) for s in range(20)], columns=['SessionId', 'ItemId', 'Time'])
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(gru, test.copy(), history=hist, batch_size=4, cut_off=[5], exclude_seen=True)
        rec, mrr = evaluation.evaluate_gpu(gru, test.copy(), history=hist, batch_size=4, cut_off=[5], exclude_seen=True)
    assert _lib.Schedule(np.zeros(20, np.int64), np.arange(21, dtype=np.int32), None, 4, 0, mode=1).n_events == 0   # none without history
    ev = res['events']
    assert len(ev) == 20 and list(ev.SessionId) == list(range(20))
    np.testing.assert_array_equal(np.isinf(ev['rank'].values), np.arange(20) % 2 == 1)   # odd sessions: target seen in the history
    assert res['ndcg'][0] == pytest.approx(np.where(ev['rank'] <= 5, 1.0 / np.log2(ev['rank'] + 1.0), 0.0).mean(), abs=1e-12)
    assert (rec, mrr) == (res['recall'], res['mrr'])


def test_no_or_empty_history_is_the_plain_evaluation(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    hist, test = _split(train, seed=4)
    with contextlib.redirect_stdout(io.StringIO()):
        a = evaluation.evaluate_events(gru, test.copy(), batch_size=6, k=2)
        for h in (None, hist.iloc[:0], hist[hist.SessionId >= 9000]):    # none, empty, nothing on a test session
            b = evaluation.evaluate_events(gru, test.copy(), batch_size=6, k=2, history=h)
            pd.testing.assert_frame_equal(a['events'], b['events'])
            assert (a['recall'], a['mrr'], a['ndcg']) == (b['recall'], b['mrr'], b['ndcg'])
            assert evaluation.evaluate_gpu(gru, test.copy(), batch_size=6, history=h) == evaluation.evaluate_gpu(gru, test.copy(), batch_size=6)


def test_budget_uses_the_concatenated_session(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    hist, test = _split(train, seed=6)
    both = _concat(gru, hist, test)
    longest = both.groupby('SessionId').size().idxmax()
    lanes, n = 6, both.groupby('SessionId').size().max()
    monkeypatch.setenv('G4R_SEEN_BUDGET', str(lanes * (n - 1) * 4 - 4))
    for call in (evaluation.evaluate_gpu, evaluation.evaluate_events):
        with contextlib.redirect_stdout(io.StringIO()), pytest.raises(ValueError, match='session %d ' % longest):
            call(gru, test.copy(), history=hist.copy(), batch_size=lanes, exclude_seen=True)


def _gloo_worker(rank, world, port, model, test, hist, q):
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
        out = evaluation.evaluate_gpu(gru, pd.read_pickle(test), history=pd.read_pickle(hist), cut_off=[1, 5, 20], batch_size=6, exclude_seen=True)
    mpatch.undo()
    q.put((rank, out))
    dist.destroy_process_group()


def test_two_process_gloo_equals_single(trained, tmp_path, monkeypatch):
    import evaluation
    gru, train = trained
    hist, test = _split(train, seed=8)
    gru.savemodel(str(tmp_path / 'model.pickle'))
    test.to_pickle(str(tmp_path / 'test.pickle')); hist.to_pickle(str(tmp_path / 'hist.pickle'))
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29950 + os.getpid() % 40
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, str(tmp_path / 'model.pickle'), str(tmp_path / 'test.pickle'),
                                                    str(tmp_path / 'hist.pickle'), q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = dict(q.get(timeout=5) for _ in range(2))
    _install(monkeypatch, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        rec, mrr = evaluation.evaluate_gpu(gru, test.copy(), history=hist.copy(), cut_off=[1, 5, 20], batch_size=6, exclude_seen=True)
        rec0, _ = evaluation.evaluate_gpu(gru, test.copy(), cut_off=[1, 5, 20], batch_size=6, exclude_seen=True)
    assert rec != rec0
    for r in (0, 1):
        np.testing.assert_allclose(res[r][0], rec, rtol=1e-12, atol=0)
        np.testing.assert_allclose(res[r][1], mrr, rtol=1e-12, atol=0)


def test_run_py_history(trained, monkeypatch):
    import evaluation
    import run
    gru, train = trained
    _install(monkeypatch, gru)
    hist, test = _split(train, seed=9, n_sessions=600)                 # run.py scores with 512 lanes
    monkeypatch.setattr(run, 'load_data', lambda fname, args: (hist if fname == 'hist.tsv' else test).copy())
    out = {}
    for flag in ([], ['--history', 'hist.tsv']):
        args = run.build_parser().parse_args(['x', '-t', 'test.tsv', '-m', '5', '20'] + flag)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            run._evaluate(gru, evaluation, args)
        out[bool(flag)] = [ln for ln in buf.getvalue().splitlines() if ln.startswith('Recall@')]
    with contextlib.redirect_stdout(io.StringIO()):
        want = {on: evaluation.evaluate_gpu(gru, test.copy(), batch_size=512, cut_off=[5, 20], history=hist if on else None) for on in (False, True)}
    for on in (False, True):
        assert out[on] == ['Recall@{}: {:.6f} MRR@{}: {:.6f}'.format(c, want[on][0][i], c, want[on][1][i]) for i, c in enumerate([5, 20])]
    assert out[True] != out[False]


C_SRC = r'''
#include <stdint.h>
#include "g4r.h"

int main(void) {
  /* sessions of 3 and 4 events, the first 2 of the second session history: counted targets 1, 2 and 5, 6 */
  const int64_t items[7] = {0, 1, 2, 3, 4, 5, 6};
  const int32_t offs[3] = {0, 3, 7};
  const int32_t hist[2] = {0, 2};
  const int32_t bad[2] = {0, 5};
  g4r_schedule* s = 0;
  if (g4r_schedule_build_history(items, 7, offs, 2, 0, bad, 2, 1, &s) != G4R_ERR_INVALID) return 1;
  if (g4r_schedule_build_history(items, 7, offs, 2, 0, hist, 2, 0, &s) != G4R_ERR_INVALID) return 2;
  if (g4r_schedule_build_history(items, 7, offs, 2, 0, hist, 2, 1, &s) != G4R_OK) return 3;
  if (g4r_schedule_events(s) != 4) return 4;
  g4r_schedule_free(s);
  return 0;
}
'''


def test_c99_caller_of_build_history(tmp_path):
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
