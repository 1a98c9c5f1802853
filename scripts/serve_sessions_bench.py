"""Serving by session key: per-call time of the session store's top-k and feed throughput (g4r_sessions_*, DESIGN §3e).

  lanes        Engine.predict_topk: the lane-addressed device call behind recommend_next_batch (every lane reset per call)
  sessions     Engine.sessions_topk: the same ranking for B distinct sessions drawn at random from a store of S live sessions
  feed         Engine.sessions_feed: warming 100k sessions x 20 events (randomly interleaved) in calls of 512 / 100,000 events

at the RSC15 shape (37,483 items, GRU(100)) and the Rees46 shape (172,000 items, GRU(512)), B = 1 / 32 / 512 events per call,
k = 20 / 100, S = 10k / 1M, on a 512-lane engine with the automatic tile choice.  Before any timing, each shape checks the
session path against the lane path: two consecutive events of 512 fresh sessions must give bitwise the items and scores of
predict_topk on a twin engine (reset, then carried).  Timing: one warm-up call, then three windows of n calls (host clock around
calls that end in a device synchronise); the median window is reported.  Prints the card name and power limit first.  Writes
nothing.

  python scripts/serve_sessions_bench.py [--shapes rsc15,rees46] [--batches 1,32,512] [--k 20,100] [--stores 10000,1000000]
"""
import argparse
import json
import os
import sys
import time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
import numpy as np
import torch
from gru4rec_b200 import _lib
import gru4rec as g4
from serve_bench import SHAPES, card, timed


def check(engs, I, k, rs):
    """two events of 512 fresh sessions through the store equal predict_topk on the twin engine, bitwise"""
    keys = np.arange(10 ** 12, 10 ** 12 + 512, dtype=np.int64)
    for step in range(2):
        X = rs.randint(0, I, 512).astype(np.int32)
        a = engs['sess'].sessions_topk(keys, X, k)
        b = engs['lane'].predict_topk(X, k, np.full(512, 1 - step, np.uint8))
        if not (np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))):
            raise SystemExit('MISMATCH: session top-k differs from the lane top-k (k %d, event %d)' % (k, step))
    engs['sess'].sessions_end(keys)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='rsc15,rees46')
    ap.add_argument('--batches', default='1,32,512')
    ap.add_argument('--k', default='20,100')
    ap.add_argument('--stores', default='10000,1000000')
    a = ap.parse_args(argv)
    batches = [int(x) for x in a.batches.split(',')]
    ks = [int(x) for x in a.k.split(',')]
    stores = [int(x) for x in a.stores.split(',')]
    name, q = card()
    print('card: %s | nvidia-smi name, power.limit, clocks.max.sm: %s' % (name, q), flush=True)
    rows, feeds = [], []
    for sh in a.shapes.split(','):
        I, L = SHAPES[sh]
        mk = dict(layers=[L], loss='bpr-max', final_act='elu-0.5', batch_size=32, n_sample=2048)
        gru = g4.GRU4Rec(**mk); gru.n_items = I
        w = gru._init_host_weights()
        engs = {}
        for leg in ('lane', 'sess'):
            engs[leg] = _lib.Engine(_lib.make_config(I, mk, sample_store=0, eval_lanes=512, step_mode=1))
            for n, v in w.items():
                engs[leg].set(n, v)
        rs = np.random.RandomState(0)
        sess = engs['sess']
        # feed throughput: 100k sessions x 20 events, randomly interleaved (events of a session stay in order)
        keys = np.repeat(np.arange(100000, dtype=np.int64), 20)
        rs.shuffle(keys)
        X = rs.randint(0, I, keys.size).astype(np.int32)
        for per_call in (512, 100000):
            sess.sessions_open(100000)
            sess.sessions_feed(keys[:per_call], X[:per_call])        # warm-up
            sess.sessions_open(100000)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(0, keys.size, per_call):
                sess.sessions_feed(keys[j:j + per_call], X[j:j + per_call])
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            f = dict(shape=sh, events_per_call=per_call, events=int(keys.size), seconds=dt, events_per_s=keys.size / dt)
            feeds.append(f)
            print(json.dumps(f), flush=True)
        for S in stores:
            sess.sessions_open(S + 1024)
            live = np.arange(S, dtype=np.int64)
            for j in range(0, S, 100000):
                sess.sessions_feed(live[j:j + 100000], rs.randint(0, I, min(100000, S - j)).astype(np.int32))
            for k in ks:
                check(engs, I, k, rs)
                for B in batches:
                    X = rs.randint(0, I, B).astype(np.int32)
                    ones = np.ones(B, np.uint8)
                    r = dict(shape=sh, n_items=I, L=L, store=S, batch=B, k=k)
                    r['lanes_ms'] = timed(lambda: engs['lane'].predict_topk(X, k, ones))[0] * 1e3

                    picks = [rs.permutation(S)[:B] for _ in range(16)]   # random distinct live sessions, drawn before timing
                    it = iter(range(10 ** 9))

                    def call():
                        sess.sessions_topk(picks[next(it) % 16], X, k)
                    med, lo, hi, n = timed(call)
                    r['sessions_ms'] = med * 1e3
                    r['sessions_spread_ms'] = [lo * 1e3, hi * 1e3]
                    rows.append(r)
                    print(json.dumps(r), flush=True)
        for e in engs.values():
            e.close()
    print('\n| shape | live sessions | events / call | k | recommend_next_batch device call (ms) | recommend_sessions device call (ms) |')
    print('|---|---|---|---|---|---|')
    for r in rows:
        print('| %s | %d | %d | %d | %.3f | %.3f |' % (r['shape'], r['store'], r['batch'], r['k'], r['lanes_ms'], r['sessions_ms']))
    print('\n| shape | events / call | feed (events/s) |')
    print('|---|---|---|')
    for f in feeds:
        print('| %s | %d | %.3g |' % (f['shape'], f['events_per_call'], f['events_per_s']))


if __name__ == '__main__':
    main()
