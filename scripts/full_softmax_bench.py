"""Full-softmax training against sampled training (DESIGN §3n, §5).

Part 1 times device time per mini-batch of g4r_upload_steps / g4r_run_uploaded at two shapes -- the RSC15 XE-shared parameter file
(L = 100, B = 32, 37,483 items, hidden dropout 0.4, Adagrad + momentum 0.2) and the Rees46 shape (shared, L = 512, B = 240,
172,000 items, embedding dropout 0.45, Adagrad) -- sampled (2048 samples, logQ, step_mode 2: the library's usual path), and
with full_softmax (every item a score column) on the score tiles the shape picks and on the other kind forced (`eval_tc`).
Each range is uploaded once, warmed up once and run `--reps` times; the median, min and max are reported.  A separate pass of
Engine.profile_uploaded over the same range then gives the device time of each phase of the full step (CUDA events around every
launch, so the sum exceeds the un-profiled step by the event overhead).  For the full step it also gives the work the catalogue part needs, computed from the shape: FLOPs (scores
twice, dL/dy and dWy: 8 M I L) and the bytes the kernels move (Wy read four times and written once, the optimizer state read
and written, dL/do written once and read twice), and the fraction of the H100 SXM data-sheet bound (67 TFLOP/s FP32,
3.35 TB/s) the measured step reaches.

Part 2 trains both objectives for the same number of epochs on a synthetic set (gru4rec_b200/synth.py) and reports Recall@20 /
MRR@20 of evaluate_gpu on its held-out sessions.

Prints one JSON line per measurement, then the card's name, power limit and maximum SM clock.

    python scripts/full_softmax_bench.py [--reps 5] [--epochs 3]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gru4rec_b200 import _lib, evaluation  # noqa: E402
from gru4rec_b200.gru4rec import GRU4Rec  # noqa: E402
from gru4rec_b200.synth import make_sessions, train_test_split  # noqa: E402

SHAPES = {
    'rsc15_xe_shared': (dict(layers=[100], batch_size=32, n_sample=2048, loss='cross-entropy', final_act='softmax', constrained_embedding=True,
                             dropout_p_hidden=0.4, learning_rate=0.2, momentum=0.2, sample_alpha=0.5, bpreg=0.0, logq=1.0), 37483, 1000),
    'rees46_xe_shared': (dict(layers=[512], batch_size=240, n_sample=2048, loss='cross-entropy', final_act='softmax', constrained_embedding=True,
                              dropout_p_embed=0.45, learning_rate=0.065, momentum=0.0, sample_alpha=0.5, bpreg=0.0, logq=1.0), 172000, 60),
}
PEAK_FP32, PEAK_BW = 67e12, 3.35e12


def emit(**kw):
    print(json.dumps(kw), flush=True)


def work(mk, n_items, M):
    """FLOPs and bytes of the catalogue part of one full step (the GRU part is the one-step path's and not counted)"""
    L = mk['layers'][-1]
    ldL = (L + 3) // 4 * 4
    flops = 8.0 * M * n_items * L
    state = 1 + (1 if mk.get('momentum', 0) else 0)             # Adagrad accumulator (+ velocity)
    row = n_items * ldL * 4.0
    byts = 5 * row + 2 * state * row + 3 * n_items * M * 4.0
    return flops, byts


def time_shape(name, reps):
    mk, n_items, steps = SHAPES[name]
    B, S = mk['batch_size'], mk['n_sample']
    rs = np.random.RandomState(0)
    lens = rs.randint(2, 20, 4 * B * max(1, steps // 8))
    items = rs.randint(0, n_items, int(lens.sum())).astype(np.int64)
    offset = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    sched = _lib.Schedule(items, offset, np.arange(len(lens), dtype=np.int64), B, S, mode=0)
    events = int(sched.batch_sizes()[:steps].sum())
    out = {}
    auto_tc = B >= 64 and n_items >= 2048          # wgmma_tiles' automatic choice
    for full, tc in ((False, None), (True, auto_tc), (True, not auto_tc)):
        rows = steps * (reps + 2)
        eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0 if full else rows * S, step_mode=2, full_softmax=full,
                                           eval_tc=tc))
        if not full:
            eng.set_sample_store(rs.randint(0, n_items, size=(rows, S)).astype(np.int64))
            eng.set_logq_support(rs.randint(1, 50, n_items).astype(np.float32))
        ms = []
        for r in range(reps + 1):
            eng.upload_steps(sched, 0, steps)
            _, t = eng.run_uploaded(steps, want_cost=False)
            if r > 0:
                ms.append(t)
        med = float(np.median(ms))
        us = med / steps * 1e3
        kind = None if not full else ('wgmma' if tc else 'fp32') + (' (auto)' if tc == auto_tc else ' (forced)')
        rec = dict(shape=name, objective='full' if full else 'sampled', score_tiles=kind, steps=steps, events=events,
                   device_ms_median=round(med, 3), device_ms_min=round(min(ms), 3), device_ms_max=round(max(ms), 3),
                   us_per_minibatch=round(us, 1), us_per_minibatch_min_max=[round(min(ms) / steps * 1e3, 1), round(max(ms) / steps * 1e3, 1)],
                   events_per_s=round(events / med * 1e3))
        if full:
            flops, byts = work(mk, n_items, events / steps)
            t = us * 1e-6
            rec.update(full_steps=eng.full_steps(), catalogue_gflop_per_step=round(flops / 1e9, 3), catalogue_mb_per_step=round(byts / 1e6, 1),
                       achieved_tflops=round(flops / t / 1e12, 2), achieved_tb_per_s=round(byts / t / 1e12, 3),
                       fraction_of_bound=round(max(flops / PEAK_FP32, byts / PEAK_BW) / t, 3),
                       bound='fp32' if flops / PEAK_FP32 > byts / PEAK_BW else 'bandwidth')
        emit(**rec)
        if full:
            eng.upload_steps(sched, 0, steps)
            prof = eng.profile_uploaded()
            emit(shape=name, score_tiles=kind, profile_us_per_step={k: round(v[0] / steps * 1e3, 1) for k, v in prof.items() if v[1]})
        out[kind] = us
        eng.close()
    emit(shape=name, full_over_sampled={k: round(v / out[None], 2) for k, v in out.items() if k})


def quality(epochs):
    data = make_sessions(n_items=3000, n_events=120000, seed=7)
    train, test = train_test_split(data)
    test = test[test.ItemId.isin(train.ItemId.unique())]
    for full in (False, True):
        gru = GRU4Rec(loss='cross-entropy', final_act='softmax', layers=[64], batch_size=32, n_epochs=epochs, n_sample=256, sample_alpha=0.5,
                      logq=1.0, constrained_embedding=True, dropout_p_hidden=0.2, learning_rate=0.1, momentum=0.2)
        gru.full_softmax = full
        with contextlib.redirect_stdout(io.StringIO()):
            gru.fit(train.copy(), sample_store=256 * 2000)
            rec, mrr = evaluation.evaluate_gpu(gru, test.copy(), cut_off=[20], batch_size=100)
        emit(quality='synthetic 3000 items', objective='full' if full else 'sampled (256, logQ)', epochs=epochs,
             recall20=round(float(rec[0]), 4), mrr20=round(float(mrr[0]), 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    for name in args.shapes.split(','):
        time_shape(name, args.reps)
    quality(args.epochs)
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    emit(gpu=q.stdout.strip())


if __name__ == '__main__':
    main()
