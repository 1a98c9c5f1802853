"""Times STAN- and VSTAN-style session kNN (DESIGN §3p, §3r, §5) on synthetic RSC15-shaped data (37,483 items, about 31M training events) with
per-event times in seconds: the fit (baselines.STAN.fit on the frame: the host index, positions and decay tables, the library's
checks and the upload; VSTAN's adds F and W4), then the device call behind evaluate_gpu / evaluate_events (g4r_bl_evaluate, sums only; the host
preparation of the frame is not timed) on about 100,000 test events at sample_size 500 and 5000 (k = 100; VSTAN with the
default lambdas for both similarities), the same for SessionKNN cosine on the same data for scale, then the float64 NumPy oracle on a sample of events.  Prints one JSON line per
measurement, then the card's name and power limit.

    python scripts/stan_bench.py [--events 31000000] [--test_events 130000] [--oracle_sample 40]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from gru4rec_b200 import baselines  # noqa: E402
from gru4rec_b200.synth import make_session_arrays  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--items', type=int, default=37483)
    ap.add_argument('--events', type=int, default=31000000)
    ap.add_argument('--test_events', type=int, default=130000)
    ap.add_argument('--k', type=int, default=100)
    ap.add_argument('--oracle_sample', type=int, default=40)
    args = ap.parse_args()
    NI = args.items
    items, off, _, _ = make_session_arrays(NI, args.events, seed=0)
    S = len(off) - 1
    lens = np.diff(off)
    sess = np.repeat(np.arange(S, dtype=np.int64), lens)
    step = np.arange(len(items)) - np.repeat(off[:-1], lens)
    frame = pd.DataFrame({'SessionId': sess, 'ItemId': items, 'Time': (sess // 16) * 60 + step * 30})   # seconds; 16 sessions per minute
    te_items, te_off, _, _ = make_session_arrays(NI, args.test_events, seed=9)
    te_off = te_off.astype(np.int64)
    head = int(te_off[min(200, len(te_off) - 1)])
    for name, model in (('stan', baselines.STAN(k=args.k, sample_size=500)),
                        ('vstan_cosine', baselines.VSTAN(k=args.k, sample_size=500, similarity='cosine')),
                        ('vstan_vector', baselines.VSTAN(k=args.k, sample_size=500, similarity='vector')),
                        ('sknn_cosine', baselines.SessionKNN(k=args.k, sample_size=500, similarity='cosine'))):
        t0 = time.time()
        model.fit(frame)
        emit(what='fit', model=name, sessions=S, events=len(items), n_items=model.n_items, distinct_pairs=int(len(model.session_items)),
             seconds=round(time.time() - t0, 3))
        dev = model._device()
        ti = model.itemidmap.reindex(te_items).values.astype(np.int32)              # ids to item indices (every id is in training)
        if name != 'sknn_cosine':
            model._cover(int(np.diff(te_off).max()))
        for sample in (500, 5000):
            t0 = time.time()
            if name != 'sknn_cosine':
                dev.stan_fit(model.session_offsets, model.session_items, model.positions, model.recency, model.w2, model.w3, sample)
                if name != 'stan':                                                   # the fit clears VSTAN's settings
                    dev.vstan_set(model.similarity, model.f, model._w4(dev.n_w4))
            else:
                dev.sknn_fit(model.session_offsets, model.session_items, model.recency, sample, 'cosine')
            up = time.time() - t0
            dev.evaluate(ti[:head], te_off[:201], None, [20], 0, counts=False)            # warm-up
            t0 = time.time()
            rec, mrr, n, _, _, _ = dev.evaluate(ti, te_off, None, [20], 0, counts=False)
            dt = time.time() - t0
            emit(what='evaluate', model=name, sample_size=sample, k=args.k, events=int(n), seconds=round(dt, 3),
                 events_per_s=round(n / dt, 1), recall20=round(float(rec[0] / n), 6), mrr20=round(float(mrr[0] / n), 6),
                 index_call_s=round(up, 3))
        if name == 'stan':
            stan = model
        else:
            del model, dev
    import stan_oracle
    t0 = time.time()
    ix = stan_oracle.Index.from_arrays(stan.session_offsets, stan.session_items, stan.positions, stan.recency, stan.w2, stan.w3,
                                       stan._w1(int(np.diff(te_off).max())), stan.n_items)
    build = time.time() - t0
    ti = stan.itemidmap.reindex(te_items).values.astype(np.int32)
    n_ev = int((np.diff(te_off) - 1).clip(min=0).sum())
    only = np.sort(np.random.RandomState(0).choice(n_ev, min(args.oracle_sample, n_ev), replace=False))
    for sample in (500, 5000):
        t0 = time.time()
        stan_oracle.rank_events(ix, args.k, sample, ti, te_off, only=only)
        dt = time.time() - t0
        emit(what='numpy_oracle', model='stan', sample_size=sample, events=len(only), events_per_s=round(len(only) / dt, 2),
             index_build_s=round(build, 1))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    emit(what='card', nvidia_smi=q.stdout.strip())


if __name__ == '__main__':
    main()
