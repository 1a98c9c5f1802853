"""Device time per mini-batch of rest-of-session evaluation (Engine.eval_rest) next to next-item evaluation (Engine.eval_schedule)
and the pair-replication workaround (Engine.eval_events on one session per (event, later item): the event's prefix, then the
item), at the DESIGN §3f shapes.  Before timing, eval_rest's pair counts are checked against the workaround's (fp32 tiles) and
its next-item pairs against eval_events'.  Host time around each call (it ends in a device synchronise) and device time (the
call's kernels and copies, torch.profiler), the latter also for eval_rest searching every score (G4R_REST_SEARCH_ALL=1) instead of
skipping those below a row's lowest threshold.  Prints the card and its power limit, then one JSON line per shape.

    python scripts/eval_rest_bench.py [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests')]
from gru4rec_b200 import _lib  # noqa: E402

SHAPES = [('rsc15', 37483, 100), ('rees46', 172000, 512)]


def sessions(n_items, n_sessions, seed):
    """session lengths 2 .. 30 (geometric, mean ~ 6), items Zipf-like with repeats inside sessions"""
    rs = np.random.RandomState(seed)
    items, off = [], [0]
    for _ in range(n_sessions):
        n = min(30, 1 + rs.geometric(0.2))
        seq = [int(rs.zipf(1.3)) % n_items]
        while len(seq) < n:
            seq.append(rs.choice(seq) if rs.rand() < 0.2 else int(rs.zipf(1.3)) % n_items)
        items += seq
        off.append(len(items))
    return np.array(items, np.int64), np.array(off, np.int32)


def workaround_data(items, off, inp):
    data, woff = [], [0]
    for p in inp:
        s = np.searchsorted(off, p, side='right') - 1
        seen = []
        for q in range(p + 1, off[s + 1]):
            if items[q] not in seen:
                seen.append(items[q])
                data += list(items[off[s]:p + 1]) + [items[q]]
                woff.append(len(data))
    return np.array(data, np.int64), np.array(woff, np.int32)


def engine(n_items, L, lanes, tc):
    mk = dict(layers=[L], batch_size=lanes, n_sample=0, loss='cross-entropy', final_act='softmax')
    cfg = _lib.make_config(n_items, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=tc)
    eng = _lib.Engine(cfg)
    rs = np.random.RandomState(0)
    for name in ('Wx0', 'Wh0', 'Wrz0', 'Wy'):
        shp = eng.shape(name)
        eng.set(name, (rs.randn(*shp) * 0.1).astype(np.float32))
    eng.set('By', (rs.randn(*eng.shape('By')) * 0.1).astype(np.float32))
    return eng


def device_ms(fn):
    """kernel and copy time of one call on the device (CUPTI through torch.profiler: every CUDA activity of the process)"""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    return sum(e.self_device_time_total for e in prof.key_averages()) / 1e3


def timed(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()                          # every Engine call ends in a device synchronise
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    for name, n_items, L in SHAPES:
        for lanes in (100, 512):
            items, off = sessions(n_items, lanes * 8, seed=lanes)
            mode = 1 | _lib.SCHED_POSITIONS
            sched = _lib.Schedule(items, off, None, lanes, 0, mode=mode)
            inp = sched.positions()[sched.counted()]
            wdata, woff = workaround_data(items, off, inp)
            wsched = _lib.Schedule(wdata, woff, None, lanes, 0, mode=mode)
            # outputs first: fp32 tiles, eval_rest's pairs = the workaround's, its next-item pairs = eval_events'
            eng = engine(n_items, L, lanes, False)
            sums, n, n_pairs, counts, offsets = eng.eval_rest(sched, [20], 0)
            wc = eng.eval_events(wsched, [20], 0)[3]
            wt = wsched.positions()[wsched.counted()] + 1
            last = dict(zip(wt.tolist(), range(len(wt))))
            assert np.array_equal(counts, wc[[last[e - 1] for e in woff[1:]]]), 'eval_rest != workaround'
            assert np.array_equal(counts[offsets[:-1]], eng.eval_events(sched, [20], 0)[3]), 'next-item pairs != eval_events'
            del eng
            eng = engine(n_items, L, lanes, None)      # the default tile choice
            calls = dict(schedule=lambda: eng.eval_schedule(sched, [20], 0), rest=lambda: eng.eval_rest(sched, [20], 0),
                         workaround=lambda: eng.eval_events(wsched, [20], 0))
            t_sched, t_rest, t_work = (timed(calls[k], args.reps) for k in ('schedule', 'rest', 'workaround'))
            dev = {k: device_ms(f) for k, f in calls.items()}
            os.environ['G4R_REST_SEARCH_ALL'] = '1'     # read when a handle first ranks the rest of sessions
            eng_all = engine(n_items, L, lanes, None)
            dev['rest_search_all'] = device_ms(lambda: eng_all.eval_rest(sched, [20], 0))
            del os.environ['G4R_REST_SEARCH_ALL'], eng_all
            steps = sched.n_steps
            print(json.dumps(dict(shape=name, n_items=n_items, L=L, lanes=lanes, events=int(n), pairs=int(n_pairs),
                                  mean_R=round(n_pairs / n, 3), steps=int(steps), workaround_steps=int(wsched.n_steps),
                                  ms_per_batch_eval_schedule=round(1e3 * t_sched / steps, 3), ms_per_batch_eval_rest=round(1e3 * t_rest / steps, 3),
                                  ms_per_batch_workaround=round(1e3 * t_work / steps, 3), rest_over_schedule=round(t_rest / t_sched, 2),
                                  workaround_over_rest=round(t_work / t_rest, 2),
                                  device_ms_per_batch={k: round(v / steps, 3) for k, v in dev.items()})), flush=True)
            del eng


if __name__ == '__main__':
    main()
