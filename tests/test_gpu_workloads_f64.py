"""-m gpu: the training workloads bench.py times (bench.WORKLOADS), each at its own shape, step by step against the float64 oracle
(gpu_utils.f64_run_steps, F64_REL / F64_RTOL).  Everything is set up as bench.py sets it up: make_config(n_items, model,
step_mode=2), the reference's initial weights (GRU4Rec._init_host_weights), the workload's synthetic sessions and schedule
(bench.build_workload, _lib.Schedule), the sampling CDF from the item supports ** sample_alpha, the logQ support, and negative
samples drawn by the device sampler (Engine.generate_samples); on top of that a random hidden state and random non-zero optimizer
state, so that Adagrad's update depends on the size of the gradient.  Three steps of the workload's own schedule: its first step
(M = B; every step of these workloads ends sessions, most synthetic sessions being two events long), the next one (those lanes
start again from the zeroed state) and the first step of the shrinking tail (M < B, compacted lanes).  The handle's counters
must show the kernel STEP_PATHS names for every step.

A float32 run of the oracle on the same inputs is held to the same comparisons; the test prints both worst errors (DESIGN.md,
the table of fp32 kernels against float64).  cfg3 is the one case where the float32 oracle comes within 4x of the bar: 1.1e-5
against 4e-5, in By.acc's update; the device reaches 2.4e-6 there.

Deliberate numeric defects, run once each on an H100 80GB HBM3 (700 W power limit):
  1. the generic kernels' dBh sum (phase_dense) leaving out lanes 64-79, the partial last lane tile at B = 80: cfg4 fails here
     in both step modes, and so do both cfg4 cases of test_gpu_windows.py; test_gpu_fp32_f64.py passes in full.
  2. the embedding-dropout mask of the layer-0 input (phase_gather_in) left out in models of more than one layer: cfg4 fails
     here in both step modes, both cfg4 window cases fail, and test_gpu_fp32_f64.py's two-layer E model (embed64_L96_100) fails.
  3. the logQ correction of the sample columns' bias scaled by 0.99 where the tensor-core step prepares it (k_ts_prep_tab):
     cfg3 fails here and in test_gpu_windows.py, and so do test_gpu_tcstep.py's two logQ product cases.
"""
import subprocess
import sys
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from bench import WORKLOADS, build_workload, ROOT
from gpu_utils import make_cfg, random_opt_state, param_names, f64_run_steps, f64_failures, f64_errors, F64_REL, F64_RTOL

P = 'persistent'

# workload -> {step_mode: kernel path of each step (gpu_utils.STEP_PATHS)}, with the reason from the code
STEP_PATHS = {
    # k_fast's shape (no embedding, one layer of L <= 120, B <= 32, Adagrad), but a window runs it only if no column chunk is
    # wider than FK_CT = 32 (run_window).  At sample_alpha 0.75 over 1,000 Zipf-distributed items the most popular item alone
    # is drawn about 105 times per row of 2,048 samples (the next ones 61, 45, 35), and a chunk never splits an item's
    # duplicate group: every row the device sampler draws for this workload falls back to k_persistent, so the benchmark
    # trains cfg1 on k_persistent throughout.  The fourth step takes a row the same sampler draws from the uniform CDF
    # (sample_alpha 0: about 2 copies per item, no chunk over 32 columns) to hold k_fast to the bar at this shape as well.
    'cfg1': {2: [P, P, P, 'fast']},
    # k_fast's shape, and sample_alpha 0: uniform samples over 37,483 items, no wide chunk
    'cfg2': {2: 'fast'},
    # the shared embedding rules out k_fast (fast_shape: no-embedding models only) and L = 100 the tensor-core step
    # (tc_eligible: L >= 160): the fallback window of k_persistent
    'cfg2x': {2: P},
    # shared embedding, one layer, L = 512 >= 160, B = 240 <= 256, Adagrad: tc_eligible
    'cfg3': {2: 'tc'},
    # shared embedding (no k_fast) and three layers (no tensor-core step): k_persistent; also the per-phase graph (step_mode 0),
    # so that the generic kernels' partial last lane tile (B = 80: lanes 64-79 of GB = 32) is checked on both launch forms
    'cfg4': {2: P, 0: 'phases'},
}
PARAMS = [(name, sm) for name in STEP_PATHS for sm in STEP_PATHS[name]]


def test_every_benchmarked_workload_has_a_case():
    """A workload bench.py can time is held to the float64 bar here; importing bench.py loads neither torch nor the library and
    starts no thread (its main() runs only as a script)."""
    assert sorted(STEP_PATHS) == sorted(WORKLOADS)
    probe = ('import sys, threading; sys.path.insert(0, %r); import bench; '
             'print(sorted(m for m in sys.modules if m.split(".")[0] in ("torch", "gru4rec_b200", "gru4rec")), threading.active_count())' % ROOT)
    out = subprocess.run([sys.executable, '-c', probe], capture_output=True, text=True, timeout=120, check=True).stdout.split()
    assert out == ['[]', '1'], out


def sampling_cdf(supports, alpha):
    """the CDF bench.py's main() hands to Engine.set_sampling_cdf"""
    P = supports.astype(np.float64) ** alpha
    P = P.cumsum() / P.sum()
    P[-1] = 1
    return P.astype(np.float32)


def _schedule(wl):
    """(Schedule, the oracle's steps, indices of the steps to run): the first step, the next one and the first step of the
    shrinking tail, over the workload's whole synthetic epoch"""
    mk = wl['model']
    B, S = mk['batch_size'], mk['n_sample']
    items, offset, order, supports = build_workload(wl, 64)
    sched = _lib.Schedule(items, offset, order, B, S, mode=0)
    steps = orc.build_train_schedule(items, offset, order, B, S)
    M = np.array([st['M'] for st in steps])
    tail = int(np.flatnonzero(M < B)[0])
    idx = [0, 1, tail]
    assert M[0] == B and M[1] == B and steps[0]['R'].any(), 'the first step has no lane whose session ends'
    assert not np.array_equal(steps[tail]['slots'], np.arange(M[tail])), 'the lanes of the tail step are not compacted'
    e = sched.export()
    for i in idx:
        m = steps[i]['M']
        assert e['M'][i] == m
        for key in ('X', 'Y', 'slots'):
            np.testing.assert_array_equal(e[key][i, :m], steps[i][key])
        np.testing.assert_array_equal(e['F'][i, :m] & 1, steps[i]['R'].astype(np.uint8))
    return sched, steps, idx, supports


def _engine(name, step_mode, n_rows, supports, seed=0):
    """the engine bench.py builds for workload `name` (its own sample store of n_rows rows), with a random hidden state and
    random non-zero optimizer state; returns (engine, model keywords, float32 logQ support or None, device-drawn sample rows)"""
    import gru4rec
    wl = WORKLOADS[name]
    mk, n_items = dict(wl['model']), wl['n_items']
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=n_rows * mk['n_sample'], step_mode=step_mode))
    gru = gru4rec.GRU4Rec(**mk)
    gru.n_items = n_items
    for n, w in gru._init_host_weights().items():
        eng.set(n, w)
    rs = np.random.RandomState(seed)
    for i, L in enumerate(mk['layers']):
        eng.set('H%d' % i, rs.randn(mk['batch_size'], L).astype(np.float32) * 0.5)
    m = orc.OracleGRU4Rec(**mk)
    m.E = None              # parameter names only: no workload has a separate embedding table
    random_opt_state(eng, m, np.random.RandomState(seed + 1))
    P0 = None
    if mk.get('logq', 0):
        P0 = np.maximum(supports, 1).astype(np.float32)
        eng.set_logq_support(P0)
    eng.set_sampling_cdf(sampling_cdf(supports, mk.get('sample_alpha', 0.75)))
    eng.generate_samples()
    return eng, mk, P0, eng.get_sample_store()


def worst(checks):
    """(largest max err / max |ref|, largest max relative err above 1 % of max, the checks they come from)"""
    errs = [(f64_errors(dev, ref, extra), what) for what, dev, ref, extra in checks]
    a, wa = max((e[0], w) for e, w in errs)
    r, wr = max((e[1], w) for e, w in errs)
    return a, r, wa, wr


@pytest.mark.gpu
@pytest.mark.parametrize('name,step_mode', PARAMS, ids=['%s-mode%d' % p for p in PARAMS])
def test_workload_steps_match_float64(name, step_mode):
    """Three steps of the workload's schedule (cfg1: four), each against a float64 oracle re-seeded from the device: every
    product the kernel keeps and the updates of every weight and optimizer state tensor, on the kernel STEP_PATHS names."""
    wl = WORKLOADS[name]
    paths = STEP_PATHS[name][step_mode]
    sched, steps, idx, supports = _schedule(wl)
    n_steps = len(paths) if isinstance(paths, list) else len(idx)
    eng, mk, P0, store = _engine(name, step_mode, n_steps, supports)
    if n_steps > len(idx):
        # cfg1's k_fast step: the schedule's third step, on a row the device draws from the uniform CDF
        idx = idx + [2]
        eng.set_sampling_cdf(sampling_cdf(supports, 0.0))
        eng.generate_samples()
        store[len(idx) - 1] = eng.get_sample_store()[0]
        eng.set_sample_store(store)
    M = [len(steps[i]['X']) for i in idx]
    for k, i in enumerate(idx):
        # the widest duplicate group among the step's score columns (k_fast takes chunks of at most 32 columns)
        widest = np.bincount(np.concatenate([steps[i]['Y'], store[k]])).max()
        print('%s step %d (schedule step %d, M = %d): widest duplicate group %d columns' % (name, k + 1, i, M[k], widest))

    def run(k, X, Y, R):
        return eng.train_steps(sched, idx[k], 1)[0]

    f32 = []
    # require_dsy=False: a step of the schedule may have no column chunk wider than a sub tile of the generic kernels
    checks, _, _ = f64_run_steps(eng, mk, wl['n_items'], store, [steps[i] for i in idx], P0, paths, run=run, keep_weights=False,
                                 f32_checks=f32, require_dsy=False)
    eng.close()
    dev, ref32 = worst(checks), worst(f32)
    print('%s-mode%d worst error, device: %.2g / %.2g (%s; %s); float32 oracle: %.2g / %.2g (%s; %s)%s' % (
        name, step_mode, dev[0], dev[1], dev[2], dev[3], ref32[0], ref32[1], ref32[2], ref32[3],
        '  (float32 oracle within 4x of the bar)' if ref32[0] > F64_REL / 4 or ref32[1] > F64_RTOL / 4 else ''))
    failed = f64_failures(checks)
    assert not failed, '\n'.join(failed)
