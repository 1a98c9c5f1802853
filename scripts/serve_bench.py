"""Serving leg: per-call time of a ranked next-item list for a batch of sessions.

  predict+host   Engine.predict (the [batch x n_items] score matrix copied to the host) + np.argpartition and a sort there
  topk-ffma      Engine.predict_topk on the fp32 FFMA tiles (eval_tc=False)
  topk-wgmma     Engine.predict_topk on the wgmma 3xTF32 tiles (eval_tc=True)

at the RSC15 shape (37,483 items, GRU(100)) and the Rees46 shape (172,000 items, GRU(512)), batch 1 / 32 / 512, k = 20 / 100.
The automatic tile choice (eval_tc=0) takes the wgmma tiles from 64 lanes and 2048 items on, so batch 1 and 32 fall on the
fp32 side and 512 on the wgmma side.  Every timed configuration first checks that both top-k legs return exactly the stable
descending order of predict() (items) and its values (scores).  Each call resets all lanes, so every call does the same work.
Timing: one warm-up call, then three windows of n calls (host clock around calls that end in a device synchronise); the
median window is reported.  Prints the card name and power limit first.  Writes nothing.

  python scripts/serve_bench.py [--shapes rsc15,rees46] [--batches 1,32,512] [--k 20,100]
"""
import argparse
import json
import os
import subprocess
import sys
import time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from gru4rec_b200 import _lib
import gru4rec as g4

SHAPES = {'rsc15': (37483, 100), 'rees46': (172000, 512)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # the card name from torch is still printed
        q = 'nvidia-smi unavailable (%s)' % e
    return name, q


def host_topk(p, k):
    """top k of every row, descending, ties to the smaller index (what predict_topk returns)"""
    part = np.argpartition(-p, k - 1, axis=1)[:, :k]
    vals = np.take_along_axis(p, part, axis=1)
    o = np.lexsort((part, -vals), axis=1)
    items = np.take_along_axis(part, o, axis=1)
    return items, np.take_along_axis(p, items, axis=1)


def timed(fn, target_s=0.4):
    t0 = time.perf_counter(); fn(); first = time.perf_counter() - t0        # warm-up (also sizes the window)
    n = max(1, min(50, int(target_s / max(first, 1e-6))))
    wins = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        wins.append((time.perf_counter() - t0) / n)
    return float(np.median(wins)), float(min(wins)), float(max(wins)), n


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='rsc15,rees46')
    ap.add_argument('--batches', default='1,32,512')
    ap.add_argument('--k', default='20,100')
    a = ap.parse_args(argv)
    batches = [int(x) for x in a.batches.split(',')]
    ks = [int(x) for x in a.k.split(',')]
    name, q = card()
    print('card: %s | nvidia-smi name, power.limit, clocks.max.sm: %s' % (name, q), flush=True)
    rows = []
    for sh in a.shapes.split(','):
        I, L = SHAPES[sh]
        mk = dict(layers=[L], loss='bpr-max', final_act='elu-0.5', batch_size=32, n_sample=2048)
        gru = g4.GRU4Rec(**mk); gru.n_items = I
        w = gru._init_host_weights()
        Be = max(batches)
        engs = {}
        for leg, tc in (('ffma', False), ('wgmma', True)):
            engs[leg] = _lib.Engine(_lib.make_config(I, mk, sample_store=0, eval_lanes=Be, step_mode=1, eval_tc=tc))
            for n, v in w.items():
                engs[leg].set(n, v)
        rs = np.random.RandomState(0)
        for B in batches:
            X = rs.randint(0, I, B).astype(np.int32)
            ones = np.ones(B, np.uint8)
            for k in ks:
                p = engs['ffma'].predict(X, ones)
                e_items = np.argsort(-p, axis=1, kind='stable')[:, :k]
                e_scores = np.take_along_axis(p, e_items, axis=1)
                h_items, h_scores = host_topk(p, k)
                ok = bool(np.array_equal(h_items, e_items))
                for leg in ('ffma', 'wgmma'):
                    it, sc = engs[leg].predict_topk(X, k, ones)
                    ok = ok and bool(np.array_equal(it, e_items)) and bool(np.array_equal(sc.view(np.uint32), e_scores.view(np.uint32)))
                if not ok:
                    raise SystemExit('MISMATCH: top-k differs from the sorted predict() output at %s batch %d k %d' % (sh, B, k))
                r = dict(shape=sh, n_items=I, L=L, batch=B, k=k, auto='wgmma' if (B >= 64 and I >= 2048) else 'ffma', checked=ok)
                r['predict_host_ms'] = timed(lambda: host_topk(engs['ffma'].predict(X, ones), k))[0] * 1e3
                for leg in ('ffma', 'wgmma'):
                    med, lo, hi, n = timed(lambda: engs[leg].predict_topk(X, k, ones))
                    r['topk_%s_ms' % leg] = med * 1e3
                    r['topk_%s_spread_ms' % leg] = [lo * 1e3, hi * 1e3]
                rows.append(r)
                print(json.dumps(r), flush=True)
        for e in engs.values():
            e.close()
    print('\n| shape | batch | k | predict + host sort (ms) | top-k fp32 tiles (ms) | top-k wgmma tiles (ms) | auto picks |')
    print('|---|---|---|---|---|---|---|')
    for r in rows:
        print('| %s | %d | %d | %.3f | %.3f | %.3f | %s |' % (r['shape'], r['batch'], r['k'], r['predict_host_ms'], r['topk_ffma_ms'], r['topk_wgmma_ms'], r['auto']))


if __name__ == '__main__':
    main()
