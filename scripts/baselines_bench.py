"""Times the session baselines on the device (DESIGN §3j, §5): the ItemKNN fit on synthetic RSC15-shaped (37,483 items, about
30M events) and Rees46-shaped (172,000 items) data, and the evaluation of about 1M test events in 'standard' and 'tiebreaking'
modes for ItemKNN, Pop and SessionPop, with evaluate_gpu of a GRU(100) on the same test events for scale.  Prints one JSON line
per measurement, then the card's name and power limit.

    python scripts/baselines_bench.py [--events 30000000] [--test_events 1000000]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gru4rec_b200 import _lib  # noqa: E402
from gru4rec_b200.synth import make_session_arrays  # noqa: E402


def norm_factors(supp, lmbd=20, alpha=0.5):
    return (np.array([np.power((s + lmbd), alpha) for s in supp], dtype=np.float64),
            np.power((supp + lmbd), (1.0 - alpha)).astype(np.float64))


def knn_fit(n_items, n_events, seed):
    items, off, _, supp = make_session_arrays(n_items, n_events, seed=seed)
    items = items.astype(np.int32)
    a, b = norm_factors(supp)
    dev = _lib.Baselines('itemknn', n_items, 100)
    dev.knn_fit(off, items, a, b)                                      # warm-up
    t0 = time.time()
    pairs, scratch, ms = dev.knn_fit(off, items, a, b)
    wall = time.time() - t0
    print(json.dumps(dict(what='itemknn_fit', n_items=n_items, events=int(len(items)), pair_work=int(pairs), scratch_bytes=int(scratch),
                          fit_device_ms=round(ms, 3), fit_call_s=round(wall, 3))), flush=True)
    return dev, supp


def timed_eval(dev, items, off, mode):
    dev.evaluate(items, off, None, [20], mode, counts=False)           # warm-up
    import torch
    torch.cuda.synchronize()
    t0 = time.time()
    rec, mrr, n, _, _, _ = dev.evaluate(items, off, None, [20], mode, counts=False)
    return time.time() - t0, n, rec[0] / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--events', type=int, default=30000000)
    ap.add_argument('--test_events', type=int, default=1000000)
    args = ap.parse_args()
    knn, supp = knn_fit(37483, args.events, 0)
    knn_fit(172000, args.events, 1)
    te_items, te_off, _, _ = make_session_arrays(37483, args.test_events + args.test_events // 3, seed=9)
    te_items = te_items.astype(np.int32); te_off = te_off.astype(np.int64)
    pop_sc = np.zeros(37483)
    top = np.lexsort((np.arange(37483), -(supp / (supp + 1))))[:100]
    pop_sc[top] = (supp / (supp + 1))[top]
    models = {'itemknn': knn}
    for kind in ('pop', 'sessionpop'):
        models[kind] = _lib.Baselines(kind, 37483, 100)
        models[kind].set_pop(pop_sc)
    for kind, dev in models.items():
        for mode, code in (('standard', 0), ('tiebreaking', 3)):
            s, n, r = timed_eval(dev, te_items, te_off, code)
            print(json.dumps(dict(what='evaluate', model=kind, mode=mode, events=int(n), seconds=round(s, 3), recall20=round(float(r), 6))), flush=True)
    # a GRU(100), trained one epoch on 200k events of the same catalogue, on the same test events through evaluate_gpu
    import contextlib
    import io
    import pandas as pd
    import gru4rec
    import evaluation

    def frame(it, off):
        return pd.DataFrame({'SessionId': np.repeat(np.arange(len(off) - 1), np.diff(off)), 'ItemId': it, 'Time': np.arange(len(it), dtype=np.float64)})
    tr_items, tr_off, _, _ = make_session_arrays(37483, 200000, seed=3)
    gru = gru4rec.GRU4Rec(layers=[100], batch_size=512, n_epochs=1, loss='cross-entropy', final_act='softmax', n_sample=2048)
    test = frame(te_items, te_off)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(frame(tr_items, tr_off))
        evaluation.evaluate_gpu(gru, test.head(20000), batch_size=512)
        t0 = time.time()
        evaluation.evaluate_gpu(gru, test, batch_size=512)
    print(json.dumps(dict(what='evaluate_gru100', events=int(len(te_items) - (len(te_off) - 1)), seconds=round(time.time() - t0, 3))), flush=True)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(json.dumps(dict(what='card', nvidia_smi=q.stdout.strip())), flush=True)


if __name__ == '__main__':
    main()
