"""Worker of tests/test_gpu_tcstep.py::test_tc_step_launch_configurations: runs the named TC_CASES of gpu_utils under the launch
configuration of its environment (G4R_TS_CLUSTER, G4R_TS_CLUSTER_BIG and G4R_TS_PDL are read once per process) and writes the
device outputs and the float64 comparison failures of every case to one npz file.
usage: tc_config_worker.py OUT.npz CASE [CASE ...]"""
import os
import sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle')); sys.path.insert(0, os.path.join(ROOT, 'tests'))
from gpu_utils import TC_CASES, f64_setup, f64_run_steps, f64_failures


def main():
    out, names = sys.argv[1], sys.argv[2:]
    res = {}
    for name in names:
        mk, n_items, step_mode = TC_CASES[name]
        eng, store, steps, P0 = f64_setup(mk, n_items, step_mode, torch_alloc=False)
        checks, outs, _ = f64_run_steps(eng, mk, n_items, store, steps, P0, 'tc')
        failed = ['%s %s' % (name, f) for f in f64_failures(checks)]
        res[name + ':failures'] = np.array('\n'.join(failed))
        res.update({'%s:%s' % (name, k): v for k, v in outs.items()})
        eng.close()
    np.savez(out, **res)


if __name__ == '__main__':
    main()
