"""Times the rule-based baselines (DESIGN §3q, §5): the device fit (g4r_bl_rules_fit: device ms from the first kernel to the last,
the host call's wall time including its checks and the upload, the pair work and the accumulators' scratch bytes) and the device
call behind evaluate_gpu (g4r_bl_evaluate, sums only, after a warm-up; the host preparation of the frame is not timed), for
SR(steps=10, weighting='div') and AR at pruning 20, on two sets:
- rsc15: RSC15-shaped synthetic sessions (37,483 items, about 31M training events, sessions of 2 + Geometric(0.5) - 1 events);
- long: 2,000 sessions of 500 .. 3,000 events over 20,000 items (AR's pair work grows with the square of the length).
Then tests/rules_oracle.py on the first sessions of each set, for its CPU rate in pairs per second.  Prints one JSON line per
measurement, then the card's name and power limit.

    python scripts/rules_bench.py [--events 31000000] [--test_events 130000] [--oracle_events 60000] [--oracle_long_events 5000]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from gru4rec_b200 import _lib  # noqa: E402
from gru4rec_b200.synth import make_session_arrays  # noqa: E402

MODELS = (('sr', 10, 'div'), ('ar', None, None))


def emit(**kw):
    print(json.dumps(kw), flush=True)


def long_set(n_items, n_sessions, seed):
    rs = np.random.RandomState(seed)
    lens = rs.randint(500, 3001, n_sessions)
    p = 1.0 / np.arange(1, n_items + 1)
    items = rs.choice(n_items, int(lens.sum()), p=p / p.sum()).astype(np.int32)
    return items, np.r_[0, np.cumsum(lens)].astype(np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--items', type=int, default=37483)
    ap.add_argument('--events', type=int, default=31000000)
    ap.add_argument('--test_events', type=int, default=130000)
    ap.add_argument('--oracle_events', type=int, default=60000)
    ap.add_argument('--oracle_long_events', type=int, default=5000)
    ap.add_argument('--pruning', type=int, default=20)
    args = ap.parse_args()
    items, off, _, _ = make_session_arrays(args.items, args.events, seed=0)
    sets = {'rsc15': (args.items, items.astype(np.int32), off.astype(np.int64))}
    li, lo = long_set(20000, 2000, seed=1)
    sets['long'] = (20000, li, lo)
    import rules_oracle as ro
    for name, (n, it, of) in sets.items():
        te_items, te_off, _, _ = make_session_arrays(n, args.test_events, seed=9)
        te_items, te_off = te_items.astype(np.int32), te_off.astype(np.int64)
        head = int(te_off[min(200, len(te_off) - 1)])
        for kind, steps, weighting in MODELS:
            dev = _lib.Baselines(kind, n, args.pruning)
            dev.rules_fit(of, it, steps, weighting)                                     # warm-up: module load, first launches
            t0 = time.time()
            pw, sb, ms = dev.rules_fit(of, it, steps, weighting)
            wall = time.time() - t0
            emit(what='fit', set=name, model=kind, steps=steps, weighting=weighting, pruning=args.pruning, n_items=n,
                 sessions=len(of) - 1, events=len(it), longest=int(np.diff(of).max()), pair_work=pw, scratch_mib=round(sb / 2 ** 20, 1),
                 device_ms=round(ms, 2), call_s=round(wall, 3), pairs_per_s=round(pw / (ms * 1e-3), 1))
            dev.evaluate(te_items[:head], te_off[:201], None, [20], 0, counts=False)      # warm-up
            t0 = time.time()
            rec, mrr, nc, _, _, _ = dev.evaluate(te_items, te_off, None, [20], 0, counts=False)
            dt = time.time() - t0
            emit(what='evaluate', set=name, model=kind, events=int(nc), seconds=round(dt, 4), events_per_s=round(nc / dt, 1),
                 recall20=round(float(rec[0] / nc), 6), mrr20=round(float(mrr[0] / nc), 6))
            del dev
        cut = max(1, int(np.searchsorted(of, args.oracle_events if name == 'rsc15' else args.oracle_long_events)))
        sub_off, sub_items = of[:cut + 1], it[:of[cut]]
        lens = np.diff(sub_off)
        for kind, steps, weighting in MODELS:
            pairs = int(np.minimum(steps, np.maximum(lens[:, None] - 1 - np.arange(lens.max())[None, :], 0)).sum()) if steps \
                else int((lens * (lens - 1)).sum())
            t0 = time.time()
            ro.rows(sub_off, sub_items, n, args.pruning, steps, weighting)
            dt = time.time() - t0
            emit(what='numpy_oracle', set=name, model=kind, sessions=cut, events=int(sub_off[-1]), pair_work=pairs, seconds=round(dt, 2),
                 pairs_per_s=round(pairs / dt, 1))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    emit(what='card', nvidia_smi=q.stdout.strip())


if __name__ == '__main__':
    main()
