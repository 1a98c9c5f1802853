"""Phase breakdown of the persistent kernel from %globaltimer stamps (headline workload)."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import bench
from gru4rec_b200 import _lib
import gru4rec as g4
WL = bench.WORKLOADS['cfg2']
mk = dict(WL['model'])
K = 1000
cfg = _lib.make_config(WL['n_items'], mk, sample_store=bench.SAMPLE_STORE, max_resident_steps=K + 8, step_mode=int(sys.argv[1]) if len(sys.argv) > 1 else 1)
eng = _lib.Engine(cfg)
gru = g4.GRU4Rec(**mk); gru.n_items = WL['n_items']
for name, w in gru._init_host_weights().items():
    eng.set(name, w)
items, offset, order, supports = bench.build_workload(WL, 3 * K)
P = supports.astype(np.float64) ** mk['sample_alpha']; P = P.cumsum() / P.sum(); P[-1] = 1
eng.set_sampling_cdf(P.astype(np.float32)); eng.generate_samples()
sched = _lib.Schedule(items, offset, order, mk['batch_size'], mk['n_sample'], mode=0)
eng.upload_steps(sched, 0, K); eng.run_uploaded(K, False)
eng.persistent_stamps(True)
eng.upload_steps(sched, K, K); c, ms = eng.run_uploaded(K, True)
st = eng.persistent_stamps(True, K).astype(np.int64)
if cfg.step_mode >= 2:
    print('fast windows', eng.fast_windows())
    # step_mode 2: the column-phase slots come from the first column CTA (dSy and its chunk's row update after b1), the GRU
    # slots 4-8 from GRU CTA 0 (b1_done reached, then backward, dense update and forward of the next step)
    names = [('wait h + stage', 0, 1), (' targets+scores', 1, 9), (' partial stats', 9, 10), (' B2 + parallel combine', 10, 2), (' RS load + cost', 2, 11), (' g + dby', 11, 12), (' part', 12, 13), (' B3', 13, 3),
             ('b1 (+release)', 3, 15), (' dSy + row update', 15, 14), ('b1 end -> GRU past b1_done', 15, 4), ('b2 -> dvec', 4, 5), ('dense (resident)', 5, 6), ('f1 + grp', 6, 7), ('f2', 7, 8)]
    if cfg.step_mode == 3:   # GRU phases on one thread-block cluster; dSy and the row update before B3
        names = names[:6] + [(' dSy + part', 12, 13), (' sparse update', 13, 14), (' B3', 14, 3), ('b1 (+release)', 3, 15), ('prefetch issue', 15, 4),
                             ('backward -> dvec', 4, 5), ('dense (resident)', 5, 6), ('f1 (+in_done, barriers)', 6, 7), ('f2', 7, 8)]
    st = st[:-1]
else:
  names = [('gru_rz(f1)', 0, 6), ('gru_h(f2)', 6, 1), ('score', 1, 2), ('stats', 2, 3), ('lossgrad', 3, 4), ('b1', 4, 7), ('b2', 7, 8), ('dense+sparse_in', 8, 5)]
print('ms/step', ms / K)
for n, a, b in names:
    d = (st[:, b] - st[:, a]) / 1000.0
    print('%-16s mean %.2f us  p50 %.2f' % (n, d[10:].mean(), np.median(d[10:])))
print('step total', ((st[1:, 0] - st[:-1, 0]) / 1000.0)[10:].mean())
