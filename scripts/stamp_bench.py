"""STAMP on the device (DESIGN §3v, §5): training steps at the RSC15 shape (37,483 items, d 100, batch 512 samples of RSC15-like
sessions, max_len 50) and at 172,000 items, and the evaluation of about 0.9M test events.  Prints the card's name and power
limit, the device ms per step (CUDA events over one epoch call after warm-up), an epoch of 31M RSC15-like events extrapolated
from it, and, from torch.profiler in a process of its own (--profile), the kernel launches per step and the split of a step's
kernel time between the encoder's forward (gather, means, attention, cells and the encoder's products), the catalogue (the three
products of role NM_CATALOGUE = 1, the softmax and the mean), the backward and Adam, and the catalogue's FLOP rate (6 B d I per
step for B samples) over the catalogue kernels' time.  Data is synthetic (seeded); nothing is written."""
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
RSC15_EVENTS = 31_000_000
PARTS = [('catalogue', re.compile(r'k_nm_g(emm|sum)<\(?\w*\)?1>|k_nm_softmax|k_nm_mean')),
         ('encoder_forward', re.compile(r'k_st_gather|k_st_means|k_st_att\b|k_st_att\(|k_st_cells\b|k_st_cells\(|k_nm_g(emm|sum)<\(?\w*\)?0>')),
         ('adam', re.compile(r'k_nm_adam|k_nm_to_double'))]


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def session_lengths(rs, n_events):
    """RSC15-like lengths: 1 + geometric (mean about 3.5 events), a tail to 200"""
    lens = np.minimum(1 + rs.geometric(0.4, size=n_events // 2), 200)
    return lens[np.cumsum(lens) <= n_events]


def setup(NI, n_samples, d=100, bs=512, max_len=50, seed=0):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, int(n_samples * 1.5))
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = (rs.zipf(1.2, size=int(off[-1])) % NI).astype(np.int32)
    th = baselines.stamp_init(NI, d, 0.05, rs)
    dev = _lib.Baselines('stamp', NI, d)
    dev.stamp_begin(max_len, bs, off, items, th)
    slen = np.concatenate([np.minimum(np.arange(1, n), max_len) for n in lens if n > 1])
    return dev, rs.permutation(len(slen)), slen, float(np.sum(lens - 1)) / float(off[-1])


def train_rate(NI, steps, warmup, bs=512, d=100):
    dev, order, slen, per_event = setup(NI, (steps + warmup) * bs * 2, d=d, bs=bs)
    dev.stamp_epoch(order[:warmup * bs], 0.005)
    timed = order[warmup * bs:(warmup + steps) * bs]
    t0 = time.time()
    losses, ms = dev.stamp_epoch(timed, 0.005)
    wall = time.time() - t0
    step_ms = ms / steps
    epoch_steps = RSC15_EVENTS * per_event / bs
    return dict(n_items=NI, d=d, batch=bs, max_len=50, steps=steps, positions_per_step=float(slen[timed].sum()) / steps,
                device_ms_per_step=step_ms, wall_s=wall, samples_per_event=per_event,
                epoch_31M_events_extrapolated_s=epoch_steps * step_ms / 1000.0, last_loss=float(losses[-1]))


def profile_split(NI, bs=512, d=100):
    """device us per part over PROFILED steps, and kernel launches per step, from torch.profiler (run in its own process)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    dev, order, _, _ = setup(NI, (PROFILED + 5) * bs * 2, d=d, bs=bs)
    dev.stamp_epoch(order[:5 * bs], 0.005)
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev.stamp_epoch(order[5 * bs:(5 + PROFILED) * bs], 0.005)
        torch.cuda.synchronize()
    parts = {name: 0.0 for name, _ in PARTS}
    parts['backward'] = 0.0
    launches = 0
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None)
        t = e.cuda_time_total if t is None else t
        if 'Memcpy' in e.key or 'Memset' in e.key or t <= 0:
            continue
        launches += e.count
        for name, rx in PARTS:
            if rx.search(e.key):
                parts[name] += t
                break
        else:
            parts['backward'] += t
    if parts['catalogue'] <= 0.0 or parts['encoder_forward'] <= 0.0:
        raise RuntimeError('the profile misses a part: ' + ', '.join(sorted(e.key for e in prof.key_averages()))[:2000])
    flop = 6.0 * bs * d * NI * PROFILED
    return dict(n_items=NI, profiled_steps=PROFILED, launches_per_step=launches / PROFILED,
                ms_per_step_by_part={k: v / 1000.0 / PROFILED for k, v in parts.items()},
                catalogue_tflops_over_catalogue_kernels=flop / (parts['catalogue'] * 1e-6) / 1e12)


def eval_rate(NI, n_events, d=100, max_len=50, seed=1):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, int(n_events * 1.45))
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = (rs.zipf(1.2, size=int(off[-1])) % NI).astype(np.int32)
    dev = _lib.Baselines('stamp', NI, d)
    dev.stamp_import(max_len, baselines.stamp_init(NI, d, 0.05, rs))
    dev.evaluate(items[:off[10]], off[:11], None, [20], 0)                  # warm-up
    t0 = time.time()
    rec, mrr, n, _, _, _ = dev.evaluate(items, off, None, [20], 0, counts=False)
    dt = time.time() - t0
    return dict(n_items=NI, counted_events=n, eval_s=dt, events_per_s=n / dt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--eval-events', type=int, default=900000)
    ap.add_argument('--profile', type=int, default=0, help='profile one catalogue size in this process and print its split (JSON)')
    a = ap.parse_args()
    if a.profile:
        print(json.dumps(profile_split(a.profile)))
        return
    out = dict(card=card())
    out['train'] = [train_rate(37483, a.steps, a.warmup), train_rate(172000, max(a.steps // 4, 5), a.warmup)]
    out['split'] = [json.loads(subprocess.check_output([sys.executable, os.path.abspath(__file__), '--profile', str(NI)], text=True).strip().split('\n')[-1])
                    for NI in (37483, 172000)]
    out['eval'] = eval_rate(37483, a.eval_events)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
