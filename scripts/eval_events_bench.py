"""Time of per-event evaluation (Engine.eval_events, g4r_eval_events, DESIGN §3f) against evaluate_gpu's device call
(Engine.eval_schedule) and against the only way to get per-event top-k lists without it, a Python loop of predict_topk
(recommend_next_batch's device call) over the same schedule.  Shapes: RSC15 (37,483 items, GRU(100)) and Rees46 (172,000 items,
GRU(512)), 100 and 512 lanes.  Before timing, the loop's lists must equal eval_events' lists.  The engine calls are timed, not
the public functions: the pandas preparation of evaluate_gpu / evaluate_events, the events frame and recommend_next_batch's item
id mapping are left out.

  python scripts/eval_events_bench.py [--rounds R] [--exclude_seen] [--parent-lib PATH]

--exclude_seen: instead, the cost of exclude_seen (DESIGN §3g): eval_schedule against the same call with the seen lists, and
eval_events with them at k = 0 and 20, timed in alternating rounds; the lists are checked to hold no seen item.
--parent-lib: instead, a libg4r.so built from the parent commit runs eval_schedule and eval_events at k = 0 and 20 (with
--exclude_seen: all with the seen lists) on the same schedule and weights; every output must equal this build's bit for bit, and
the two builds are timed in alternating rounds (median and min-max of --rounds).

Env: EE_EVENTS (test events per shape, default 100,000, at least twice the items), EE_SHAPES (e.g. 'rsc15,rees46'), EE_LANES (e.g. '100,512')."""
import argparse, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
import numpy as np
import torch
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays
import gru4rec as g4
from serve_bench import card
from serve_filter_bench import make_engine, parent_lib

SHAPES = {'rsc15': (37483, 100), 'rees46': (172000, 512)}

ap = argparse.ArgumentParser()
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--exclude_seen', action='store_true')
ap.add_argument('--parent-lib', default=None)
a = ap.parse_args()
plib = parent_lib(a.parent_lib) if a.parent_lib else None
print('card: %s | nvidia-smi name, power.limit, clocks.max.sm: %s' % card(), flush=True)
n_ev = int(os.environ.get('EE_EVENTS', 100000))
CUTS = [1, 5, 20]


def timed(f):
    ts = []
    for _ in range(a.rounds):
        torch.cuda.synchronize(); t0 = time.time()
        f()
        torch.cuda.synchronize(); ts.append(time.time() - t0)
    return float(np.median(ts))


def seen_calls(eng, on, f):
    eng.set_eval_exclude_seen(on)
    try:
        return f()
    finally:
        eng.set_eval_exclude_seen(False)


def seen_leg(eng, sched, e, shape, I, L, lanes):
    """eval_schedule with and without exclude_seen, and eval_events with it, in alternating rounds (median of --rounds)"""
    got = seen_calls(eng, True, lambda: eng.eval_events(sched, CUTS, 0, k=20))
    cur, j = {}, 0                                             # no list holds an item its session has input so far
    for s in range(sched.n_steps):
        for b in range(int(e['M'][s])):
            sl = int(e['slots'][s, b])
            if e['F'][s, b] & 2 or sl not in cur:
                cur[sl] = set()
            cur[sl].add(int(e['X'][s, b]))
            if cur[sl] & set(got[4][j].tolist()):
                raise SystemExit('MISMATCH: a seen item in an exclude_seen list (%s, %d lanes)' % (shape, lanes))
            j += 1
    calls = {'eval_schedule': lambda: eng.eval_schedule(sched, CUTS, 0),
             'eval_schedule exclude_seen': lambda: seen_calls(eng, True, lambda: eng.eval_schedule(sched, CUTS, 0)),
             'eval_events k=0 exclude_seen': lambda: seen_calls(eng, True, lambda: eng.eval_events(sched, CUTS, 0, k=0)),
             'eval_events k=20 exclude_seen': lambda: seen_calls(eng, True, lambda: eng.eval_events(sched, CUTS, 0, k=20))}
    for f in calls.values():
        f()
    ts = {n: [] for n in calls}
    for _ in range(a.rounds):
        for n, f in calls.items():
            torch.cuda.synchronize(); t0 = time.time()
            f()
            torch.cuda.synchronize(); ts[n].append(time.time() - t0)
    base = float(np.median(ts['eval_schedule']))
    for n, v in ts.items():
        dt = float(np.median(v))
        print('%-7s I=%d GRU(%d) lanes=%3d %-30s %8.3f s (min-max %.3f-%.3f)  %8.1f us / mini-batch  %+6.1f %%  (%d mini-batches, %d events)'
              % (shape, I, L, lanes, n, dt, min(v), max(v), dt / sched.n_steps * 1e6, 100.0 * (dt / base - 1.0), sched.n_steps, sched.n_events), flush=True)


def bitwise_equal(x, y):
    """two results (tuples of arrays, numbers or None) hold the same bytes"""
    if isinstance(x, tuple):
        return len(x) == len(y) and all(bitwise_equal(p, q) for p, q in zip(x, y))
    if x is None or y is None:
        return x is y
    x, y = np.asarray(x), np.asarray(y)
    return x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()


def parent_leg(eng, par, sched, shape, I, L, lanes):
    """eval_schedule and eval_events of this build and the parent build: bitwise-equal outputs, then alternating rounds"""
    calls = {'eval_schedule': lambda g: g.eval_schedule(sched, CUTS, 0)}
    for k in (0, 20):
        calls['eval_events k=%d' % k] = lambda g, k=k: g.eval_events(sched, CUTS, 0, k=k)
    tag = ' exclude_seen' if a.exclude_seen else ''
    for g in (eng, par):
        g.set_eval_exclude_seen(a.exclude_seen)
    for n, f in calls.items():
        if not bitwise_equal(f(eng), f(par)):
            raise SystemExit('MISMATCH: %s%s differs from the parent build (%s, %d lanes)' % (n, tag, shape, lanes))
    ts = {(n, b): [] for n in calls for b in ('parent', 'pr')}
    for r in range(a.rounds):
        for n, f in calls.items():
            for b, g in (('parent', par), ('pr', eng))[::1 if r % 2 == 0 else -1]:    # either build first in turn
                torch.cuda.synchronize(); t0 = time.time()
                f(g)
                torch.cuda.synchronize(); ts[(n, b)].append(time.time() - t0)
    for n in calls:
        p, q = ts[(n, 'parent')], ts[(n, 'pr')]
        print('%-7s I=%d GRU(%d) lanes=%3d %-30s parent median %.4f s (min-max %.4f-%.4f)  this build median %.4f s (min-max %.4f-%.4f)  '
              'same result: True' % (shape, I, L, lanes, n + tag, np.median(p), min(p), max(p), np.median(q), min(q), max(q)), flush=True)


def loop_topk(eng, sched, e, k):
    """the per-event lists by predict_topk, one call per mini-batch of the schedule (lanes = state slots)"""
    B = sched.batch_size
    out = []
    eng.reset_eval_hidden()
    for s in range(sched.n_steps):
        M = int(e['M'][s]); sl = e['slots'][s, :M]
        X = np.zeros(B, np.int32); X[sl] = e['X'][s, :M]
        R = np.zeros(B, np.uint8); R[sl] = (e['F'][s, :M] & 2) != 0
        out.append(eng.predict_topk(X, k, R)[0][sl])
    return np.concatenate(out)


for shape in os.environ.get('EE_SHAPES', 'rsc15,rees46').split(','):
    I, L = SHAPES[shape]
    mk = dict(layers=[L], loss='bpr-max', final_act='elu-0.5', batch_size=32, n_sample=2048)
    gru = g4.GRU4Rec(**mk); gru.n_items = I
    w = gru._init_host_weights()
    items, offset, _, _ = make_session_arrays(I, max(n_ev, 2 * I), seed=1)
    for lanes in [int(x) for x in os.environ.get('EE_LANES', '100,512').split(',')]:
        eng = make_engine(I, mk, lanes, w)
        sched = _lib.Schedule(items, offset, None, lanes, 0, mode=1)
        e = sched.export()
        if plib is not None:
            par = make_engine(I, mk, lanes, w, plib)
            parent_leg(eng, par, sched, shape, I, L, lanes)
            eng.close(); par.close()
            continue
        if a.exclude_seen:
            seen_leg(eng, sched, e, shape, I, L, lanes)
            eng.close()
            continue
        ref = loop_topk(eng, sched, e, 20)
        got = eng.eval_events(sched, CUTS, 0, k=20)
        if not np.array_equal(ref, got[4]):
            raise SystemExit('MISMATCH: predict_topk loop and eval_events lists differ (%s, %d lanes)' % (shape, lanes))
        rec = eng.eval_schedule(sched, CUTS, 0)
        if not (np.array_equal(rec[0], got[0]) and np.array_equal(rec[1], got[1])):
            raise SystemExit('MISMATCH: eval_events sums differ from eval_schedule (%s, %d lanes)' % (shape, lanes))
        t = {'evaluate_gpu (eval_schedule)': timed(lambda: eng.eval_schedule(sched, CUTS, 0))}
        for k in (0, 20, 100):
            t['eval_events k=%d' % k] = timed(lambda: eng.eval_events(sched, CUTS, 0, k=k))
        t['predict_topk loop k=20'] = timed(lambda: loop_topk(eng, sched, e, 20))
        for name, dt in t.items():
            print('%-7s I=%d GRU(%d) lanes=%3d %-30s %8.3f s  %8.1f us / mini-batch  (%d mini-batches, %d events)'
                  % (shape, I, L, lanes, name, dt, dt / sched.n_steps * 1e6, sched.n_steps, sched.n_events), flush=True)
        eng.close()
