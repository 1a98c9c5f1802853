"""Serving leg with filters: per-call time of Engine.predict_topk with a candidate set and per-lane exclusions
(g4r_predict_topk_filtered), each against a parent build.

  filtered       Engine.predict_topk(X, k, items=..., exclude=...) on the tile choice of --tiles (auto: eval_tc=0), candidates
                 100 % / 50 % / 1 % of the catalogue (random, fixed per shape), 0 / 20 / 1000 random exclusions per lane
  unfiltered     Engine.predict_topk(X, k)
  --parent-lib   a libg4r.so built from the parent commit runs every row too: its predict() and its top-k (unfiltered and
                 filtered) must equal this build's bit for bit, and the two builds are timed in alternating windows in the
                 same process

at the RSC15 shape (37,483 items, GRU(100)) and the Rees46 shape (172,000 items, GRU(512)), batch 1 / 32 / 512, k = 20 / 100.
Every filtered configuration first checks each row against predict() plus the mask and a sort (items exactly, scores bitwise,
-1 / NaN past a lane's eligible items); the unfiltered legs are checked against each other.  Each call resets all lanes, so
every call does the same work.  Timing: one warm-up call, then windows of n calls (host clock around calls that end in a device
synchronise); the median window is reported with the min / max.  Prints the card name and power limit first.  Writes nothing.

  python scripts/serve_filter_bench.py [--shapes rsc15,rees46] [--batches 1,32,512] [--k 20,100] [--tiles auto|fp32|wgmma]
                                       [--parent-lib PATH]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from gru4rec_b200 import _lib
import gru4rec as g4
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
from serve_bench import SHAPES, card

FRACS = (1.0, 0.5, 0.01)
N_EXCL = (0, 20, 1000)


def timed(fn, target_s=0.25, windows=3):
    t0 = time.perf_counter(); fn(); first = time.perf_counter() - t0        # warm-up (also sizes the window)
    n = max(1, min(50, int(target_s / max(first, 1e-6))))
    wins = []
    for _ in range(windows):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        wins.append((time.perf_counter() - t0) / n)
    return wins


def parent_lib(path):
    """the parent build with the ctypes signatures of this build for every symbol it exports"""
    lib, cur = C.CDLL(path), _lib.load()
    for name in _lib.EXPORTS:
        if hasattr(lib, name):
            f, g = getattr(lib, name), getattr(cur, name)
            f.argtypes, f.restype = g.argtypes, g.restype
    return lib


def make_engine(I, mk, Be, w, lib=None, eval_tc=None):
    saved = _lib._lib
    if lib is not None:
        _lib._lib = lib
    try:
        eng = _lib.Engine(_lib.make_config(I, mk, sample_store=0, eval_lanes=Be, step_mode=1, eval_tc=eval_tc))
    finally:
        _lib._lib = saved
    for n, v in w.items():
        eng.set(n, v)
    return eng


def check(p, items, scores, k, cand, excl):
    """rows of predict() restricted to the eligible items, sorted by score then index, against the device result"""
    ok = np.ones(p.shape, bool)
    if cand is not None:
        ok[:] = False; ok[:, cand] = True
    for b, e in enumerate(excl or []):
        if len(e):
            ok[b, e] = False
    q = np.where(ok, p, -np.inf)
    part = np.argpartition(-q, k - 1, axis=1)[:, :k]
    vals = np.take_along_axis(q, part, axis=1)
    o = np.lexsort((part, -vals), axis=1)
    e_items = np.take_along_axis(part, o, axis=1)
    live = np.take_along_axis(ok, e_items, axis=1)
    e_items = np.where(live, e_items, -1)
    e_scores = np.take_along_axis(p, np.maximum(e_items, 0), axis=1)
    return bool(np.array_equal(items, e_items) and np.array_equal(scores[live].view(np.uint32), e_scores[live].view(np.uint32))
                and np.isnan(scores[~live]).all())


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='rsc15,rees46')
    ap.add_argument('--batches', default='1,32,512')
    ap.add_argument('--k', default='20,100')
    ap.add_argument('--tiles', default='auto', choices=['auto', 'fp32', 'wgmma'])
    ap.add_argument('--parent-lib', default=None)
    a = ap.parse_args(argv)
    eval_tc = {'auto': None, 'fp32': False, 'wgmma': True}[a.tiles]
    batches = [int(x) for x in a.batches.split(',')]
    ks = [int(x) for x in a.k.split(',')]
    name, q = card()
    print('card: %s | nvidia-smi name, power.limit, clocks.max.sm: %s' % (name, q), flush=True)
    plib = parent_lib(a.parent_lib) if a.parent_lib else None
    rows, cmp_rows = [], []
    for sh in a.shapes.split(','):
        I, L = SHAPES[sh]
        mk = dict(layers=[L], loss='bpr-max', final_act='elu-0.5', batch_size=32, n_sample=2048)
        gru = g4.GRU4Rec(**mk); gru.n_items = I
        w = gru._init_host_weights()
        Be = max(batches)
        eng = make_engine(I, mk, Be, w, eval_tc=eval_tc)
        par = make_engine(I, mk, Be, w, plib, eval_tc=eval_tc) if plib is not None else None
        rs = np.random.RandomState(0)
        cands = {f: (None if f == 1.0 else np.sort(rs.choice(I, int(f * I), replace=False)).astype(np.int32)) for f in FRACS}
        for B in batches:
            X = rs.randint(0, I, B).astype(np.int32)
            ones = np.ones(B, np.uint8)
            excls = {n: [rs.randint(0, I, n).astype(np.int32) for _ in range(B)] for n in N_EXCL}
            p = eng.predict(X, ones)
            if par is not None and not np.array_equal(p.view(np.uint32), par.predict(X, ones).view(np.uint32)):
                raise SystemExit('MISMATCH: predict differs from the parent build at %s batch %d' % (sh, B))
            for k in ks:
                if par is not None:         # unfiltered: parent and this build, alternating windows
                    i0, s0 = par.predict_topk(X, k, ones)
                    i1, s1 = eng.predict_topk(X, k, ones)
                    same = bool(np.array_equal(i0, i1) and np.array_equal(s0.view(np.uint32), s1.view(np.uint32)))
                    if not same:
                        raise SystemExit('MISMATCH: unfiltered top-k differs from the parent build at %s batch %d k %d' % (sh, B, k))
                    wp, wn = [], []
                    for _ in range(4):
                        wp += timed(lambda: par.predict_topk(X, k, ones), 0.15, 2)
                        wn += timed(lambda: eng.predict_topk(X, k, ones), 0.15, 2)
                    r = dict(shape=sh, batch=B, k=k, cand_frac=1.0, excl_per_lane=0, filtered=False, parent_ms=float(np.median(wp)) * 1e3,
                             parent_spread_ms=[min(wp) * 1e3, max(wp) * 1e3], pr_ms=float(np.median(wn)) * 1e3,
                             pr_spread_ms=[min(wn) * 1e3, max(wn) * 1e3], same_result=same)
                    cmp_rows.append(r)
                    print(json.dumps(r), flush=True)
                for f in FRACS:
                    cand = cands[f]
                    for ne in N_EXCL:
                        excl = excls[ne] if ne else None
                        if cand is not None and k > len(cand):
                            continue
                        items = cand if cand is not None else np.arange(I, dtype=np.int32)
                        call = lambda e=eng: e.predict_topk(X, k, ones, items=items, exclude=excl)
                        it, sc = call()
                        if not check(p, it, sc, k, cand, excl):
                            raise SystemExit('MISMATCH: filtered top-k differs from the masked sort of predict() at %s batch %d k %d '
                                             'candidates %g exclusions %d' % (sh, B, k, f, ne))
                        if par is not None:     # parent and this build, alternating windows
                            i0, s0 = call(par)
                            same = bool(np.array_equal(i0, it) and np.array_equal(s0.view(np.uint32), sc.view(np.uint32)))
                            if not same:
                                raise SystemExit('MISMATCH: filtered top-k differs from the parent build at %s batch %d k %d '
                                                 'candidates %g exclusions %d' % (sh, B, k, f, ne))
                            wp, wn = [], []
                            for _ in range(4):
                                wp += timed(lambda: call(par), 0.15, 2)
                                wn += timed(call, 0.15, 2)
                            r = dict(shape=sh, batch=B, k=k, cand_frac=f, excl_per_lane=ne, filtered=True, parent_ms=float(np.median(wp)) * 1e3,
                                     parent_spread_ms=[min(wp) * 1e3, max(wp) * 1e3], pr_ms=float(np.median(wn)) * 1e3,
                                     pr_spread_ms=[min(wn) * 1e3, max(wn) * 1e3], same_result=same)
                            cmp_rows.append(r)
                            print(json.dumps(r), flush=True)
                        wins = timed(call)
                        r = dict(shape=sh, batch=B, k=k, cand_frac=f, excl_per_lane=ne, checked=True,
                                 ms=float(np.median(wins)) * 1e3, spread_ms=[min(wins) * 1e3, max(wins) * 1e3])
                        rows.append(r)
                        print(json.dumps(r), flush=True)
        eng.close()
        if par is not None:
            par.close()
    if cmp_rows:
        print('\n| shape | batch | k | candidates | exclusions / lane | parent (ms) | parent min-max | this build (ms) | this build min-max |')
        print('|---|---|---|---|---|---|---|---|---|')
        for r in cmp_rows:
            print('| %s | %d | %d | %g %% | %d | %.3f | %.3f-%.3f | %.3f | %.3f-%.3f |' % (
                r['shape'], r['batch'], r['k'], 100 * r['cand_frac'], r['excl_per_lane'], r['parent_ms'], *r['parent_spread_ms'],
                r['pr_ms'], *r['pr_spread_ms']))
    print('\n| shape | batch | k | candidates | exclusions / lane | filtered top-k (ms) | min-max |')
    print('|---|---|---|---|---|---|---|')
    for r in rows:
        print('| %s | %d | %d | %g %% | %d | %.3f | %.3f-%.3f |' % (r['shape'], r['batch'], r['k'], 100 * r['cand_frac'], r['excl_per_lane'], r['ms'],
                                                              *r['spread_ms']))


if __name__ == '__main__':
    main()
