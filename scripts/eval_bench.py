"""Time of one evaluation mini-batch (evaluate_gpu's compiled function, evaluation.py:57-76) at the RSC15 shape: 37,483 items x
512 lanes x GRU(100) -- fp32 FFMA tiles vs wgmma 3xTF32 tiles.  The reference reports 4.34 s for a whole evaluation on an A30
(README.md:169, RetailRocket).

  python scripts/eval_bench.py [--parent-lib PATH]

--parent-lib: a libg4r.so built from the parent commit evaluates the same schedule with the same weights; its Recall / MRR sums
and the per-lane counts of the last mini-batch must equal this build's bit for bit, and the two builds are timed in alternating
evaluations (median and min-max of --rounds).  Shape: EV_ITEMS, EV_LANES, EV_L, EV_EVENTS."""
import argparse, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
import numpy as np
import torch
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays
import gru4rec as g4
from serve_bench import card
from serve_filter_bench import make_engine, parent_lib

ap = argparse.ArgumentParser()
ap.add_argument('--parent-lib', default=None)
ap.add_argument('--rounds', type=int, default=3)
a = ap.parse_args()
plib = parent_lib(a.parent_lib) if a.parent_lib else None
print('card: %s | nvidia-smi name, power.limit, clocks.max.sm: %s' % card(), flush=True)
I, LANES = int(os.environ.get('EV_ITEMS', 37483)), int(os.environ.get('EV_LANES', 512))
CUTS = [1, 5, 20]
for L in [int(x) for x in os.environ.get('EV_L', '100,512').split(',')]:
    mk = dict(layers=[L], loss='bpr-max', final_act='elu-0.5', batch_size=32, n_sample=2048)
    items, offset, order, supports = make_session_arrays(I, int(os.environ.get('EV_EVENTS', 400000)), seed=1)
    out = {}
    for name, tc in (('ffma', False), ('tc', True)):
        gru = g4.GRU4Rec(**mk); gru.n_items = I
        w = gru._init_host_weights()
        builds = {'pr': make_engine(I, mk, LANES, w, eval_tc=tc)}
        if plib is not None:
            builds['parent'] = make_engine(I, mk, LANES, w, plib, eval_tc=tc)
        sched = _lib.Schedule(items, offset, None, LANES, 0, mode=1)
        m_last = int(sched.export()['M'][-1])
        res = {}
        for b, eng in builds.items():
            eng.eval_schedule(sched, [20], 0)
            res[b] = eng.eval_schedule(sched, CUTS, 0) + (eng.eval_counts(m_last),)
        if plib is not None:
            same = all(np.array_equal(x, y) for x, y in zip(res['pr'], res['parent']))
            if not same:
                raise SystemExit('MISMATCH: evaluation differs from the parent build at L=%d %s lanes %d' % (L, name, LANES))
        times = {b: [] for b in builds}
        for _ in range(a.rounds if plib is not None else 1):
            for b, eng in builds.items():
                torch.cuda.synchronize(); t0 = time.time()
                eng.eval_schedule(sched, CUTS, 0)
                torch.cuda.synchronize(); times[b].append(time.time() - t0)
        rec, mrr, n, _ = res['pr']
        dt = float(np.median(times['pr']))
        out[name] = (dt, sched.n_steps, rec / n, mrr / n)
        flop = 2.0 * I * LANES * L * sched.n_steps
        print('L=%d %-8s %7.3f s for %d evaluation mini-batches of %d lanes x %d items (%d events): %.1f us / mini-batch, %.1f TFLOP/s (score GEMM incl. GRU forward + ranking)'
              % (L, name, dt, sched.n_steps, LANES, I, n, dt / sched.n_steps * 1e6, flop / dt / 1e12), flush=True)
        if plib is not None:
            print('L=%d %-8s lanes %d  parent median %.4f s (min-max %.4f-%.4f)  this build median %.4f s (min-max %.4f-%.4f)  same result: %s'
                  % (L, name, LANES, np.median(times['parent']), min(times['parent']), max(times['parent']), dt, min(times['pr']),
                     max(times['pr']), same), flush=True)
        for eng in builds.values():
            eng.close()
    print('L=%d recall@1,5,20 ffma %s tc %s ; mrr ffma %s tc %s' % (L, out['ffma'][2], out['tc'][2], out['ffma'][3], out['tc'][3]), flush=True)
