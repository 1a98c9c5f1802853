"""Times truncated BPTT (DESIGN §3l, §5): device time per window and events/s of g4r_upload_steps / g4r_run_uploaded for
bptt = T in {1, 2, 4, 8, 16, 32} at three shapes -- the headline shape (no embedding, L = 100, B = 32, bpr-max, 2048 samples), the
rsc15 shared shape (L = 100, B = 32, cross-entropy + logQ, hidden dropout, Adagrad + momentum) and the Rees46 shape (shared,
L = 512, B = 240).  T = 1 runs on the shape's usual path (step_mode 2, the library's choice) as the reference line; T > 1 runs the
window path.  Every timed range is uploaded once, warmed up once, then run `--reps` times.  Prints one JSON line per measurement,
then the card's name and power limit.

    python scripts/bptt_bench.py [--steps 64] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gru4rec_b200 import _lib  # noqa: E402

SHAPES = {
    'headline': (dict(layers=[100], batch_size=32, n_sample=2048, loss='bpr-max', final_act='elu-0.5', bpreg=1.95, adapt='adagrad',
                      learning_rate=0.05), 37483),
    'rsc15_shared': (dict(layers=[100], batch_size=32, n_sample=2048, loss='cross-entropy', final_act='softmax', constrained_embedding=True,
                          logq=1.0, dropout_p_hidden=0.2, adapt='adagrad', momentum=0.3, learning_rate=0.05), 37483),
    'rees46_shared': (dict(layers=[512], batch_size=240, n_sample=2048, loss='bpr-max', final_act='elu-0.5', constrained_embedding=True,
                           adapt='adagrad', learning_rate=0.05), 172000),
}


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=64, help='mini-batches per timed range (a multiple of every T)')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--T', default='1,2,4,8,16,32')
    args = ap.parse_args()
    for name in args.shapes.split(','):
        mk, n_items = SHAPES[name]
        B, S = mk['batch_size'], mk['n_sample']
        rs = np.random.RandomState(0)
        lens = rs.randint(2, 20, 40 * B)
        items = rs.randint(0, n_items, int(lens.sum())).astype(np.int64)
        offset = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        sched = _lib.Schedule(items, offset, np.arange(len(lens), dtype=np.int64), B, S, mode=0)
        for T in [int(t) for t in args.T.split(',')]:
            rows = args.steps * (args.reps + 2)
            eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=rows * S, step_mode=2, bptt=T))
            eng.set_sample_store(rs.randint(0, n_items, size=(rows, S)).astype(np.int64))
            if mk.get('logq'):
                eng.set_logq_support(rs.randint(1, 50, n_items).astype(np.float32))
            events = int(sched.batch_sizes()[:args.steps].sum())
            ms = []
            for r in range(args.reps + 1):
                eng.upload_steps(sched, 0, args.steps)
                _, t = eng.run_uploaded(args.steps, want_cost=False)
                if r > 0:
                    ms.append(t)
            med = float(np.median(ms))
            emit(shape=name, bptt=T, steps=args.steps, windows=args.steps // T, events=events, device_ms_median=round(med, 3),
                 ms_per_window=round(med / (args.steps // T), 4), events_per_s=round(events / med * 1e3), window_path=eng.bptt_windows() > 0)
            eng.close()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    emit(gpu=q.stdout.strip())


if __name__ == '__main__':
    main()
