"""Time of one evaluation mini-batch (evaluate_gpu's compiled function, evaluation.py:57-76) at the RSC15 shape: 37,483 items x
512 lanes x GRU(100) -- fp32 FFMA tiles vs wgmma 3xTF32 tiles.  The reference reports 4.34 s for a whole evaluation on an A30
(README.md:169, RetailRocket)."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays
import gru4rec as g4

I, LANES = int(os.environ.get('EV_ITEMS', 37483)), int(os.environ.get('EV_LANES', 512))
for L in [int(x) for x in os.environ.get('EV_L', '100,512').split(',')]:
    mk = dict(layers=[L], loss='bpr-max', final_act='elu-0.5', batch_size=32, n_sample=2048)
    items, offset, order, supports = make_session_arrays(I, int(os.environ.get('EV_EVENTS', 400000)), seed=1)
    out = {}
    for name, tc in (('ffma', False), ('tc', True)):
        eng = _lib.Engine(_lib.make_config(I, mk, sample_store=0, eval_lanes=LANES, step_mode=1, eval_tc=tc))
        gru = g4.GRU4Rec(**mk); gru.n_items = I
        for n, w in gru._init_host_weights().items():
            eng.set(n, w)
        sched = _lib.Schedule(items, offset, None, LANES, 0, mode=1)
        eng.eval_schedule(sched, [20], 0)
        torch.cuda.synchronize(); t0 = time.time()
        rec, mrr, n = eng.eval_schedule(sched, [1, 5, 20], 0)
        torch.cuda.synchronize(); dt = time.time() - t0
        out[name] = (dt, sched.n_steps, rec / n, mrr / n)
        flop = 2.0 * I * LANES * L * sched.n_steps
        print('L=%d %-8s %7.3f s for %d evaluation mini-batches of %d lanes x %d items (%d events): %.1f us / mini-batch, %.1f TFLOP/s (score GEMM incl. GRU forward + ranking)'
              % (L, name, dt, sched.n_steps, LANES, I, n, dt / sched.n_steps * 1e6, flop / dt / 1e12), flush=True)
        eng.close()
    print('L=%d recall@1,5,20 ffma %s tc %s ; mrr ffma %s tc %s' % (L, out['ffma'][2], out['tc'][2], out['ffma'][3], out['tc'][3]), flush=True)
