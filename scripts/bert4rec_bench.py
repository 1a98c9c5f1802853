"""BERT4Rec on the device (DESIGN §3x, §5): training steps at the shipped shape (d 64, 2 blocks of 2 heads, batch 256 pieces of
RSC15-like lengths, max_len 50, mask_prob 0.2, dropout 0.1) at 37,483 items and at 172,000 items, and the evaluation of test
events at 37,483 items.  Prints the card's name and power limit, the device ms per step (CUDA events over one epoch call after
warm-up), the split of a step's kernel time between the encoder forward, its backward, the catalogue (the three products of role
NM_CATALOGUE = 1, the softmax and the mean over the masked positions; the output bias and its gradient count with the forward and
the backward) and Adam, read from torch.profiler in a separate run of the next steps, and the catalogue's FLOP rate (6 Pm d I FLOP
per step for Pm masked positions) over the catalogue kernels' time and over the whole step.  Evaluation encodes up to max_len
positions per event (its own window), so its events/s sit well below SASRec's.  Data is synthetic (seeded); nothing is written."""
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
FORWARD = re.compile(r'k_nm_g(emm|sum)<\(?\w*\)?0>|k_b4_embed|k_sa_ln\b|k_sa_bias|k_b4_gelu\b|k_b4_att_fwd|k_sa_resid|k_b4_gather')
MASK_PROB, DROPOUT = 0.2, 0.1


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def session_lengths(rs, n_events):
    """RSC15-like lengths: 1 + geometric (mean about 3.5 events), a tail to 200"""
    lens = np.minimum(1 + rs.geometric(0.4, size=n_events // 2), 200)
    return lens[np.cumsum(lens) <= n_events]


def split_us(dev, order, masks):
    """device us per part over one epoch call of `order`, from torch.profiler: catalogue, forward, backward, adam"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev.bert4rec_epoch(order, masks, 0, 0.001, DROPOUT)
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


def train_rate(NI, steps, warmup, d=64, blocks=2, heads=2, bs=256, max_len=50, seed=0):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, (steps + warmup + PROFILED) * bs * 5)
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = rs.zipf(1.2, size=int(off[-1])) % NI
    poff, pit = baselines.narm_pieces(off, items, max_len)
    th = baselines.bert4rec_init(NI, d, blocks, max_len, rs)
    dev = _lib.Baselines('bert4rec', NI, d)
    dev.bert4rec_begin(blocks, heads, max_len, bs, poff, pit, th)
    plen = np.diff(poff)
    order = rs.permutation(len(poff) - 1)
    masks = baselines.bert4rec_masks(poff, MASK_PROB, rs)
    n_masked = np.add.reduceat(masks.astype(np.int64), poff[:-1])
    dev.bert4rec_epoch(order[:warmup * bs], masks, 0, 0.001, DROPOUT)
    timed = order[warmup * bs:(warmup + steps) * bs]
    t0 = time.time()
    losses, ms = dev.bert4rec_epoch(timed, masks, 0, 0.001, DROPOUT)
    wall = time.time() - t0
    pos, pm = int(plen[timed].sum()), int(n_masked[timed].sum())
    step_ms = ms / steps
    prof_order = order[(warmup + steps) * bs:(warmup + steps + PROFILED) * bs]
    parts, _ = split_us(dev, prof_order, masks)
    prof_flop = 6.0 * int(n_masked[prof_order].sum()) * d * NI
    return dict(n_items=NI, d=d, n_blocks=blocks, n_heads=heads, batch=bs, max_len=max_len, mask_prob=MASK_PROB, dropout=DROPOUT, steps=steps,
                positions_per_step=pos / steps, masked_positions_per_step=pm / steps, device_ms_per_step=step_ms, wall_s=wall,
                profiled_steps=PROFILED, ms_per_step_by_part={k: v / 1000.0 / PROFILED for k, v in parts.items()},
                catalogue_tflops_over_catalogue_kernels=prof_flop / (parts['catalogue'] * 1e-6) / 1e12,
                catalogue_tflops_over_step=6.0 * pm * d * NI / (ms * 1e-3) / 1e12, last_loss=float(losses[-1]))


def eval_rate(NI, n_events, d=64, blocks=2, heads=2, max_len=50, seed=1):
    rs = np.random.RandomState(seed)
    lens = session_lengths(rs, int(n_events * 1.45))
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    items = (rs.zipf(1.2, size=int(off[-1])) % NI).astype(np.int32)
    dev = _lib.Baselines('bert4rec', NI, d)
    dev.bert4rec_import(blocks, heads, max_len, baselines.bert4rec_init(NI, d, blocks, max_len, rs))
    dev.evaluate(items[:off[10]], off[:11], None, [20], 0)                  # warm-up
    t0 = time.time()
    rec, mrr, n, _, _, _ = dev.evaluate(items, off, None, [20], 0, counts=False)
    dt = time.time() - t0
    return dict(n_items=NI, counted_events=n, eval_s=dt, events_per_s=n / dt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--eval-events', type=int, default=300000)
    a = ap.parse_args()
    out = dict(card=card())
    out['train'] = [train_rate(37483, a.steps, a.warmup), train_rate(172000, max(a.steps // 4, 5), a.warmup)]
    out['eval'] = eval_rate(37483, a.eval_events)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
