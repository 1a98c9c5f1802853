"""Times BPR-MF on the device (DESIGN §3k, §5) on synthetic RSC15-shaped data (37,483 items, about 31M training events, F = 100):
per iteration the host draw, the call (argument checks, upload, device work) and the device time, with the largest level (the
longest chain of dependent updates); then the device call behind evaluate_gpu / evaluate_events (g4r_bl_evaluate; the host
preparation of the frame is not timed) on about 0.9M test events, sums only and with k = 20 lists; then the float64 NumPy
restatement's sequential loop on a sample of events, for a CPU figure per iteration.  Prints one JSON line per measurement, then
the card's name and power limit.

    python scripts/bpr_bench.py [--events 31000000] [--iterations 10] [--test_events 1000000]"""
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
from gru4rec_b200 import _lib  # noqa: E402
from gru4rec_b200.synth import make_session_arrays  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--items', type=int, default=37483)
    ap.add_argument('--events', type=int, default=31000000)
    ap.add_argument('--factors', type=int, default=100)
    ap.add_argument('--iterations', type=int, default=10)
    ap.add_argument('--test_events', type=int, default=1000000)
    ap.add_argument('--oracle_sample', type=int, default=20000)
    ap.add_argument('--warps', default='', help='comma-separated max_warps, one per iteration in turn (default and above 4 per SM: the library\'s cap of 4 per SM)')
    args = ap.parse_args()
    NI, F = args.items, args.factors
    items, off, _, _ = make_session_arrays(NI, args.events, seed=0)
    S, N = len(off) - 1, len(items)
    rows_s = np.repeat(np.arange(S, dtype=np.int32), np.diff(off))
    rows_i = items.astype(np.int32)
    rs = np.random.RandomState(0)
    U0 = rs.rand(S, F) * 0.1 - 0.05
    I0 = rs.rand(NI, F) * 0.1 - 0.05
    bI = np.zeros(NI)
    dev = _lib.Baselines('bpr', NI, F)
    t0 = time.time()
    dev.bpr_begin(rows_s, rows_i, S, U0, I0, bI)
    emit(what='bpr_begin', sessions=S, events=N, n_items=NI, factors=F, u_bytes=S * F * 8, seconds=round(time.time() - t0, 3))
    draws0 = None
    for it in range(args.iterations):
        t0 = time.time()
        perm, neg = rs.permutation(N), rs.randint(NI, size=N)
        t1 = time.time()
        warps = [int(w) for w in args.warps.split(',')] if args.warps else [1 << 30]
        mean, level, ms = dev.bpr_iterate(perm, neg, 0.01, 0.0, 0.0, max_warps=warps[it % len(warps)])
        t2 = time.time()
        if draws0 is None:
            draws0 = (perm, neg)
        emit(what='bpr_iteration', it=it, max_warps=warps[it % len(warps)], draw_s=round(t1 - t0, 3), call_s=round(t2 - t1, 3), device_ms=round(ms, 2), max_level=int(level),
             mean_log_sigm=mean, ns_per_level=round(ms * 1e6 / max(level, 1), 1))
    # evaluation of about 0.9M test events with the fitted item factors
    te_items, te_off, _, _ = make_session_arrays(NI, args.test_events + args.test_events // 3, seed=9)
    te_items = te_items.astype(np.int32); te_off = te_off.astype(np.int64)
    for k in (0, 20):
        head = int(te_off[min(2000, len(te_off) - 1)])
        dev.evaluate(te_items[:head], te_off[:2001] if len(te_off) > 2001 else te_off, None, [20], 0, counts=False, k=k)   # warm-up
        t0 = time.time()
        rec, mrr, n, _, _, _ = dev.evaluate(te_items, te_off, None, [20], 0, counts=False, k=k)
        emit(what='evaluate', k=k, events=int(n), seconds=round(time.time() - t0, 3), recall20=round(float(rec[0] / n), 6),
             pairs_per_s=float('%.3g' % (n * NI * F / (time.time() - t0))))
    # the float64 restatement's sequential loop on the first events of iteration 0 (the reference's own loop has the same shape)
    import bpr_oracle
    M = min(args.oracle_sample, N)
    perm, neg = draws0[0][:M], draws0[1][:M]
    uniq, inv = np.unique(rows_s[perm], return_inverse=True)          # only the sample's sessions: U0 is not copied whole
    small_s = np.r_[inv, np.zeros(M, np.int64)]
    small_i = np.r_[rows_i[perm], rows_i[neg]]
    t0 = time.time()
    bpr_oracle.fit(small_s, small_i, U0[uniq], I0, bI, [(np.arange(M), M + np.arange(M))], 0.01, 0.0, 0.0)
    per = (time.time() - t0) / M
    emit(what='numpy_oracle_loop', events=M, us_per_event=round(per * 1e6, 2), seconds_per_iteration=round(per * N, 1))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    emit(what='card', nvidia_smi=q.stdout.strip())


if __name__ == '__main__':
    main()
