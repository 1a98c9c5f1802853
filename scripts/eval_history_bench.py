"""Time of evaluation from each session's history (Schedule(n_history=...), DESIGN §3h) against the workaround it replaces: the
per-event evaluation of the concatenated data (history then test events), whose rows with a test target are kept afterwards.
Leave-one-out synthetic data: every user is one session of history events and one test event, history lengths from
make_session_arrays' session lengths times EH_SCALE, or geometric with mean EH_MEAN_HIST.  Shapes: RSC15 (37,483 items,
GRU(100)), Rees46 (172,000 items, GRU(512)) and ml20m (27,000 items, GRU(100): with EH_USERS=138000 EH_MEAN_HIST=144, a
20M-event leave-one-out set of MovieLens-20M's size).  Before timing, the history mode's per-event counts must equal the workaround's counts of the test events wherever
both rank a block / mini-batch with the same tile kind (all of them with EH_TC=fp32).  The engine calls are timed, not the
public functions (their pandas preparation is the same for both).

  python scripts/eval_history_bench.py [--rounds R] [--parent-lib PATH]

--parent-lib: instead of the workaround, a libg4r.so built from the parent commit runs the history schedule (eval_schedule, and
eval_events at k = 0 and 20, with and without exclude_seen) with the same weights; every output must equal this build's bit for
bit, and the two builds are timed in alternating rounds (median and min-max of --rounds).

Env: EH_USERS (users per shape, default 20,000), EH_SCALE (history length multiplier, default 4), EH_SHAPES (e.g. 'rsc15,rees46'),
EH_LANES (default 512), EH_TC ('auto' or 'fp32')."""
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

SHAPES = {'rsc15': (37483, 100), 'rees46': (172000, 512), 'ml20m': (27000, 100)}

ap = argparse.ArgumentParser()
ap.add_argument('--rounds', type=int, default=3)
ap.add_argument('--parent-lib', default=None)
a = ap.parse_args()
plib = parent_lib(a.parent_lib) if a.parent_lib else None
print('card: %s | nvidia-smi name, power.limit, clocks.max.sm: %s' % card(), flush=True)
n_users = int(os.environ.get('EH_USERS', 20000))
scale = int(os.environ.get('EH_SCALE', 4))
mean_hist = float(os.environ.get('EH_MEAN_HIST', 0))
lanes = int(os.environ.get('EH_LANES', 512))
tc = {'auto': None, 'fp32': False}[os.environ.get('EH_TC', 'auto')]
CUTS = [1, 5, 20]


def leave_one_out(I, seed):
    """n_users sessions: history lengths from synthetic session lengths x scale, one test event each"""
    rs = np.random.RandomState(seed)
    if mean_hist > 0:
        lens = rs.geometric(1.0 / mean_hist, size=n_users)
    else:
        items, offset, _, _ = make_session_arrays(I, max(4 * n_users, 2 * I), seed=seed)
        lens = np.diff(offset)[:n_users] * scale
    off = np.zeros(len(lens) + 1, np.int64)
    off[1:] = np.cumsum(lens + 1)
    data = rs.randint(0, I, size=int(off[-1])).astype(np.int64)
    return data, off.astype(np.int32), lens.astype(np.int32)


def timed(calls):
    ts = {n: [] for n in calls}
    for f in calls.values():
        f()
    for _ in range(a.rounds):
        for n, f in calls.items():
            torch.cuda.synchronize(); t0 = time.time()
            f()
            torch.cuda.synchronize(); ts[n].append(time.time() - t0)
    return ts


def bitwise_equal(x, y):
    """two results (tuples of arrays, numbers or None) hold the same bytes"""
    if isinstance(x, tuple):
        return len(x) == len(y) and all(bitwise_equal(p, q) for p, q in zip(x, y))
    if x is None or y is None:
        return x is y
    x, y = np.asarray(x), np.asarray(y)
    return x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()


def seen(g, on, f):
    g.set_eval_exclude_seen(on)
    try:
        return f()
    finally:
        g.set_eval_exclude_seen(False)


def parent_leg(eng, par, hist, shape, I, L):
    """the history schedule on this build and the parent build: bitwise-equal outputs, then alternating rounds"""
    calls = {}
    for on in (False, True):
        tag = ' exclude_seen' if on else ''
        calls['eval_schedule' + tag] = lambda g, on=on: seen(g, on, lambda: g.eval_schedule(hist, CUTS, 0))
        for k in (0, 20):
            calls['eval_events k=%d%s' % (k, tag)] = lambda g, on=on, k=k: seen(g, on, lambda: g.eval_events(hist, CUTS, 0, k=k))
    for n, f in calls.items():
        if not bitwise_equal(f(eng), f(par)):
            raise SystemExit('MISMATCH: history %s differs from the parent build (%s)' % (n, shape))
    ts = {(n, b): [] for n in calls for b in ('parent', 'pr')}
    for r in range(a.rounds):
        for n, f in calls.items():
            for b, g in (('parent', par), ('pr', eng))[::1 if r % 2 == 0 else -1]:    # either build first in turn
                torch.cuda.synchronize(); t0 = time.time()
                f(g)
                torch.cuda.synchronize(); ts[(n, b)].append(time.time() - t0)
    for n in calls:
        p, q = ts[(n, 'parent')], ts[(n, 'pr')]
        print('%-7s I=%d GRU(%d) lanes=%d history %-28s parent median %.4f s (min-max %.4f-%.4f)  this build median %.4f s (min-max %.4f-%.4f)  '
              'same result: True' % (shape, I, L, lanes, n, np.median(p), min(p), max(p), np.median(q), min(q), max(q)), flush=True)


for shape in os.environ.get('EH_SHAPES', 'rsc15,rees46').split(','):
    I, L = SHAPES[shape]
    mk = dict(layers=[L], loss='bpr-max', final_act='elu-0.5', batch_size=32, n_sample=0)
    gru = g4.GRU4Rec(**mk); gru.n_items = I
    w = gru._init_host_weights()
    eng = make_engine(I, mk, lanes, w, eval_tc=tc)
    data, off, nh = leave_one_out(I, seed=1)
    plain = _lib.Schedule(data, off, None, lanes, 0, mode=1)
    hist = _lib.Schedule(data, off, None, lanes, 0, mode=1, n_history=nh)
    if plib is not None:
        par = make_engine(I, mk, lanes, w, plib, eval_tc=tc)
        print('%-7s I=%d GRU(%d) lanes=%d: %d users, %d events, %d mini-batches, %d counted events'
              % (shape, I, L, lanes, len(nh), int(off[-1]), hist.n_steps, hist.n_events), flush=True)
        parent_leg(eng, par, hist, shape, I, L)
        eng.close(); par.close()
        continue
    used = np.arange(lanes)[None, :] < plain.batch_sizes()[:, None]
    keep = hist.counted()[used]
    got, ref = eng.eval_events(hist, CUTS, 0), eng.eval_events(plain, CUTS, 0)
    same = np.all(got[3] == ref[3][keep], axis=1)
    if tc is False and not same.all():
        raise SystemExit('MISMATCH: history counts differ from the workaround (%s)' % shape)
    print('%-7s I=%d GRU(%d) lanes=%d: %d users, %d events, %d mini-batches, %d counted events; counts equal to the workaround on %.5f of them'
          % (shape, I, L, lanes, len(nh), int(off[-1]), hist.n_steps, hist.n_events, same.mean()), flush=True)
    ts = timed({'workaround: eval_events on the concatenated data': lambda: eng.eval_events(plain, CUTS, 0),
                'history: eval_events': lambda: eng.eval_events(hist, CUTS, 0),
                'history: eval_schedule': lambda: eng.eval_schedule(hist, CUTS, 0)})
    base = float(np.median(ts['workaround: eval_events on the concatenated data']))
    for n, v in ts.items():
        dt = float(np.median(v))
        print('%-7s %-52s %8.3f s (min-max %.3f-%.3f)  %6.1fx faster than the workaround' % (shape, n, dt, min(v), max(v), base / dt), flush=True)
    eng.close()
