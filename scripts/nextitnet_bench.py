"""NextItNet on the device (DESIGN §3w, §5): training steps at the RSC15 shape (37,483 items, d 100, dilations 1, 2, 1, 2, 1, 2,
kernel_size 3, batch 128 pieces of RSC15-like lengths, max_len 50) and at 172,000 items, and the evaluation of about 0.9M test
events.  Prints the card's name and power limit, the device ms per step (CUDA events over one epoch call after warm-up), the split
of a step's kernel time between the encoder forward, its backward, the catalogue (the three products of role NM_CATALOGUE = 1, the
softmax and the mean; the output bias and its gradient count with the forward and the backward) and Adam, read from torch.profiler
in a separate run of the next steps, and the catalogue's FLOP rate (6 P d I FLOP per step for P positions) over the catalogue
kernels' time (products, softmax and mean) and over the whole step.  Data is synthetic (seeded); nothing is written."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gru4rec_b200 import _lib, baselines  # noqa: E402

PROFILED = 20
CATALOGUE = re.compile(r'k_nm_g(emm|sum)<\(?\w*\)?1>|k_nm_softmax|k_nm_mean')
FORWARD = re.compile(r'k_nm_g(emm|sum)<\(?\w*\)?0>|k_ni_embed|k_sa_ln\b|k_sa_bias|k_ni_relu')
DIL = (1, 2, 1, 2, 1, 2)


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def session_lengths(rs, n_events):
    """RSC15-like lengths: 1 + geometric (mean about 3.5 events), a tail to 200"""
    lens = np.minimum(1 + rs.geometric(0.4, size=n_events // 2), 200)
    return lens[np.cumsum(lens) <= n_events]


def split_us(dev, order):
    """device us per part over one epoch call of `order`, from torch.profiler: catalogue, forward, backward, adam"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev.nextitnet_epoch(order, 0.001)
        torch.cuda.synchronize()
    parts = dict(catalogue=0.0, forward=0.0, backward=0.0, adam=0.0)
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None)
        t = e.cuda_time_total if t is None else t
        if 'Memcpy' in e.key or 'Memset' in e.key:
            continue
        if CATALOGUE.search(e.key):
            parts['catalogue'] += t
        elif FORWARD.search(e.key):
            parts['forward'] += t
        elif 'k_nm_adam' in e.key or 'k_nm_to_double' in e.key:
            parts['adam'] += t
        else:
            parts['backward'] += t       # with the gathers, which the forward and the backward both run
    if parts['catalogue'] <= 0.0:
        raise RuntimeError('the profile holds no catalogue kernel: ' + ', '.join(sorted(e.key for e in prof.key_averages()))[:2000])
    return parts, sorted((e.key, getattr(e, 'device_time_total', 0.0)) for e in prof.key_averages())


def train_rate(NI, steps, warmup, d=100, dil=DIL, K=3, bs=128, max_len=50, seed=0):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, (steps + warmup + PROFILED) * bs * 5)
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = rs.zipf(1.2, size=int(off[-1])) % NI
    poff, pit = baselines.narm_pieces(off, items, max_len + 1)
    th = baselines.nextitnet_init(NI, d, dil, K, rs)
    dev = _lib.Baselines('nextitnet', NI, d)
    dev.nextitnet_begin(dil, K, max_len, bs, poff, pit, th)
    plen = np.diff(poff) - 1
    order = rs.permutation(len(poff) - 1)
    dev.nextitnet_epoch(order[:warmup * bs], 0.001)
    timed = order[warmup * bs:(warmup + steps) * bs]
    t0 = time.time()
    losses, ms = dev.nextitnet_epoch(timed, 0.001)
    wall = time.time() - t0
    pos = int(plen[timed].sum())
    step_ms = ms / steps
    prof_order = order[(warmup + steps) * bs:(warmup + steps + PROFILED) * bs]
    parts, _ = split_us(dev, prof_order)
    prof_flop = 6.0 * int(plen[prof_order].sum()) * d * NI
    cat_gemm_us = parts['catalogue']
    return dict(n_items=NI, d=d, dilations=list(dil), kernel_size=K, batch=bs, max_len=max_len, steps=steps, positions_per_step=pos / steps,
                device_ms_per_step=step_ms, wall_s=wall, profiled_steps=PROFILED,
                ms_per_step_by_part={k: v / 1000.0 / PROFILED for k, v in parts.items()},
                catalogue_tflops_over_catalogue_kernels=prof_flop / (cat_gemm_us * 1e-6) / 1e12,
                catalogue_tflops_over_step=6.0 * pos * d * NI / (ms * 1e-3) / 1e12, last_loss=float(losses[-1]))


def eval_rate(NI, n_events, d=100, dil=DIL, K=3, max_len=50, seed=1):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, int(n_events * 1.45))
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = (rs.zipf(1.2, size=int(off[-1])) % NI).astype(np.int32)
    dev = _lib.Baselines('nextitnet', NI, d)
    dev.nextitnet_import(dil, K, max_len, baselines.nextitnet_init(NI, d, dil, K, rs))
    dev.evaluate(items[:off[10]], off[:11], None, [20], 0)                  # warm-up
    t0 = time.time()
    rec, mrr, n, _, _, _ = dev.evaluate(items, off, None, [20], 0, counts=False)
    dt = time.time() - t0
    return dict(n_items=NI, counted_events=n, eval_s=dt, events_per_s=n / dt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--eval-events', type=int, default=900000)
    a = ap.parse_args()
    out = dict(card=card())
    out['train'] = [train_rate(37483, a.steps, a.warmup), train_rate(172000, max(a.steps // 4, 5), a.warmup)]
    out['eval'] = eval_rate(37483, a.eval_events)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
