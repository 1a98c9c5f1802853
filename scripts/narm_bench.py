"""NARM on the device (DESIGN §3s, §5): training steps at the RSC15 shape (37,483 items, d_e 50, H 100, batch 512 pieces of
RSC15-like lengths) and at a larger catalogue, and the evaluation of about 0.9M test events.  Prints the card's name and power
limit, mini-batches/s, the device time of a full RSC15-sized epoch (31M pairs) extrapolated from the measured steps, and the
achieved FLOP/s of the three catalogue products (6 P d_e I FLOP per step for P pairs): over their own kernel time (the
k_nm_gemm / k_nm_gsum instances of role NM_CATALOGUE = 1, read from torch.profiler in a separate run of the next steps) and over
the whole step's device time.  Data is synthetic (seeded); nothing is written."""
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


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def session_lengths(rs, n_events):
    """RSC15-like lengths: 1 + geometric (mean about 3.5 events), a tail to 200"""
    lens = np.minimum(1 + rs.geometric(0.4, size=n_events // 2), 200)
    return lens[np.cumsum(lens) <= n_events]


def train_rate(NI, steps, warmup, d=50, H=100, bs=512, max_len=50, seed=0):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, (steps + warmup + PROFILED) * bs * 5)
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = rs.zipf(1.2, size=int(off[-1])) % NI
    poff, pit = baselines.narm_pieces(off, items, max_len)
    n_pieces = len(poff) - 1
    th = baselines.narm_init(NI, d, H, rs)
    dev = _lib.Baselines('narm', NI, d)
    dev.narm_begin(H, max_len, bs, poff, pit, th)
    plen = np.diff(poff) - 1
    order = rs.permutation(n_pieces)
    dev.narm_epoch(order[:warmup * bs], seed, 0.001, 0.25, 0.5)
    timed = order[warmup * bs:(warmup + steps) * bs]
    t0 = time.time()
    losses, ms = dev.narm_epoch(timed, seed, 0.001, 0.25, 0.5)
    wall = time.time() - t0
    pairs = int(plen[timed].sum())
    flop = 6.0 * pairs * d * NI
    step_ms = ms / steps
    prof_order = order[(warmup + steps) * bs:(warmup + steps + PROFILED) * bs]
    cat_us, softmax_us = catalogue_kernel_us(dev, prof_order, seed)
    prof_flop = 6.0 * int(plen[prof_order].sum()) * d * NI
    return dict(n_items=NI, d_e=d, hidden=H, batch=bs, steps=steps, pairs_per_step=pairs / steps, device_ms_per_step=step_ms,
                minibatches_per_s=1000.0 / step_ms, wall_s=wall, catalogue_tflops_over_step=flop / (ms * 1e-3) / 1e12,
                catalogue_ms_per_step=cat_us / 1000.0 / PROFILED, softmax_ms_per_step=softmax_us / 1000.0 / PROFILED,
                catalogue_tflops_over_kernels=prof_flop / (cat_us * 1e-6) / 1e12, profiled_steps=PROFILED,
                rsc15_epoch_s_extrapolated=31e6 / (pairs / steps) * step_ms / 1000.0, last_loss=float(losses[-1]))


PROFILED = 20
CATALOGUE = re.compile(r'k_nm_g(emm|sum)<\(?\w*\)?1>')


def catalogue_kernel_us(dev, order, seed):
    """(device us of the catalogue products' kernels, of k_nm_softmax) over one epoch call of `order`, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev.narm_epoch(order, seed, 0.001, 0.25, 0.5)
        torch.cuda.synchronize()
    cat = soft = 0.0
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None)
        t = e.cuda_time_total if t is None else t
        if CATALOGUE.search(e.key):
            cat += t
        elif 'k_nm_softmax' in e.key:
            soft += t
    if cat <= 0.0:
        raise RuntimeError('the profile holds no catalogue product kernel: ' + ', '.join(sorted(e.key for e in prof.key_averages()))[:2000])
    return cat, soft


def eval_rate(NI, n_events, d=50, H=100, max_len=50, seed=1):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, int(n_events * 1.45))
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = (rs.zipf(1.2, size=int(off[-1])) % NI).astype(np.int32)
    dev = _lib.Baselines('narm', NI, d)
    dev.narm_import(H, max_len, baselines.narm_init(NI, d, H, rs))
    dev.evaluate(items[:off[10]], off[:11], None, [20], 0)                  # warm-up
    t0 = time.time()
    rec, mrr, n, _, _, _ = dev.evaluate(items, off, None, [20], 0, counts=False)
    return dict(n_items=NI, counted_events=n, eval_s=time.time() - t0, events_per_s=n / (time.time() - t0))


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
