"""-m gpu: the tensor-core training step (wgmma 3xTF32 GEMMs with fused epilogues, csrc/g4r_tcstep.cuh) against the oracle:
constrained embedding, one layer -- the family of the reference's shipped parameter files (paramfiles/*_best.py)."""
import os
import subprocess
import sys
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions, make_session_arrays
from gpu_utils import make_cfg, push_weights, compare_weights, assert_step_costs, TC_CASES, f64_setup, f64_run_steps, f64_failures

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

SMALL = [
    dict(layers=[16], batch_size=8, n_sample=32, loss='cross-entropy', final_act='softmax', constrained_embedding=True, learning_rate=0.1, momentum=0.2, logq=1.0, sample_alpha=0.5),
    dict(layers=[20], batch_size=12, n_sample=48, loss='bpr-max', final_act='elu-0.5', constrained_embedding=True, learning_rate=0.05, momentum=0.4, bpreg=1.95, sample_alpha=0.4),
    dict(layers=[36], batch_size=5, n_sample=0, loss='bpr-max', final_act='elu-1', constrained_embedding=True, learning_rate=0.05, momentum=0.0),
    dict(layers=[24], batch_size=16, n_sample=64, loss='top1-max', final_act='tanh', constrained_embedding=True, learning_rate=0.1, momentum=0.1, lmbd=0.001,
         dropout_p_hidden=0.2, dropout_p_embed=0.3),
    dict(layers=[16], batch_size=8, n_sample=32, loss='xe_logit', final_act='softmax_logit', constrained_embedding=True, learning_rate=0.1, momentum=0.0, adapt=None),
]


@pytest.mark.parametrize('mk', SMALL)
def test_tensor_core_step_whole_epoch(mk):
    """step_mode 4 forces the tensor-core step at any size: a whole epoch incl. the shrinking tail (M < B), duplicates, logQ, dropout."""
    df = make_sessions(n_items=120, n_events=700, seed=13)
    d = orc.prepare_fit_data(df)
    B, S = mk['batch_size'], mk['n_sample']
    rows = 120
    m = orc.OracleGRU4Rec(**mk)
    m.init(d['n_items'])
    eng = _lib.Engine(make_cfg(d['n_items'], mk, sample_store=rows * S, step_mode=4))
    assert eng.uses_tensor_cores()
    push_weights(eng, m)
    rs = np.random.RandomState(3)
    store = None
    if S:
        store = rs.randint(0, d['n_items'], size=(rows, S)).astype(np.int64)
        store[:, :S // 4] = rs.randint(0, 12, size=(rows, S // 4))          # heavy duplicates, also against the targets
        eng.set_sample_store(store)
    if mk.get('logq', 0):
        P0 = rs.randint(1, 50, size=d['n_items']).astype(np.float32)
        m.P0 = P0
        eng.set_logq_support(P0)
    sched = _lib.Schedule(d['data_items'], d['offset_sessions'], d['base_order'], B, S, mode=0)
    steps = orc.build_train_schedule(d['data_items'], d['offset_sessions'], d['base_order'], B, S)
    n = min(sched.n_steps, rows - 1)
    assert steps[n - 1]['M'] < B or n < sched.n_steps
    costs = eng.train_steps(sched, 0, n)
    ref = [m.train_step(st['X'], st['Y'], st['R'], samples=(store[k] if S else None), slots=st['slots']) for k, st in enumerate(steps[:n])]
    assert_step_costs(costs, ref)
    compare_weights(eng, m, rtol=3e-3, atol=3e-5, what='tensor-core step')
    eng.close()


@pytest.mark.parametrize('L,B,loss,fact,extra', [(224, 80, 'bpr-max', 'elu-0.5', dict(momentum=0.4, bpreg=1.95, sample_alpha=0.4)),
                                                 (512, 240, 'cross-entropy', 'softmax', dict(momentum=0.0, logq=1.0, sample_alpha=0.5, learning_rate=0.065)),
                                                 (480, 48, 'cross-entropy', 'softmax', dict(momentum=0.0, logq=1.0, sample_alpha=0.2, dropout_p_hidden=0.2))])
def test_tensor_core_step_shipped_shapes(L, B, loss, fact, extra):
    """The shapes of paramfiles/{retailrocket,rees46,yoochoose}_*_best.py (2048 samples): picked automatically (step_mode 2)."""
    n_items = 4000
    mk = dict(layers=[L], batch_size=B, n_sample=2048, loss=loss, final_act=fact, constrained_embedding=True, learning_rate=0.05)
    mk.update(extra)
    items, offset, order, supports = make_session_arrays(n_items, 30000, seed=7)
    rows = 12
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=rows * 2048, step_mode=2))
    assert eng.uses_tensor_cores()
    push_weights(eng, m)
    if mk.get('logq', 0):
        P0 = np.maximum(supports, 1).astype(np.float32)
        m.P0 = P0
        eng.set_logq_support(P0)
    P = orc.sampling_cdf(supports, mk['sample_alpha']).astype(np.float32)
    u = np.random.RandomState(4).rand(rows * 2048).astype(np.float32)
    eng.set_sampling_cdf(P)
    eng.generate_samples_from_uniform(u)
    store = orc.searchsorted_k2(P, u).reshape(rows, 2048)
    sched = _lib.Schedule(items, offset, order, B, 2048, mode=0)
    steps = orc.build_train_schedule(items, offset, order, B, 2048)
    n = 6
    costs = eng.train_steps(sched, 0, n)
    ref = [m.train_step(st['X'], st['Y'], st['R'], samples=store[k], slots=st['slots']) for k, st in enumerate(steps[:n])]
    np.testing.assert_allclose(costs, ref, rtol=1e-4, atol=1e-6)
    compare_weights(eng, m, rtol=2e-3, atol=2e-5, what='tensor-core step, shipped shape')
    eng.close()


@pytest.mark.parametrize('name', sorted(TC_CASES))
def test_tc_step_products_match_float64(name):
    """Every product of the tensor-core step against a float64 oracle run on the same float32 inputs, two steps (M = B, then M < B
    with a reset lane and duplicates; the oracle is re-seeded from the device in between): y, H, dvec = [da_h | da_r | da_z], dSx,
    the dSy rows, the cost, and -- plain SGD -- dWx, dWh, dWrz, dBh and the Wy / By row gradients recovered from the updates; the
    Adagrad case compares the updates W1 - W0 of the weights and the optimizer state, from random non-zero state
    (gpu_utils.f64_run_steps).  Failures are listed as 'max err / max |ref|  /  max relative err above 1 % of max' against the
    bar of gpu_utils.F64_REL / F64_RTOL (4e-5 / 1e-3).  Measured on an H100 80GB HBM3 (400 W power limit), worst tensor over all
    cases: the device 4.8e-6 / 7.6e-5 (the Adagrad case, updates from random state: 2.3e-6 / 4.1e-5); a float32 run of the oracle
    9.1e-6 / 2.3e-4 (the Adagrad case, updates from random state: 5.5e-6 / 2.1e-4); the device with the a_lo * b_hi term of every
    product dropped (2xTF32) at least 2.9e-4 / 1.5e-2 in every case, up to 0.23 / 2.5 (the Adagrad case then compared updated
    weights from zero state)."""
    mk, n_items, step_mode = TC_CASES[name]
    eng, store, steps, P0 = f64_setup(mk, n_items, step_mode)
    checks, _, _ = f64_run_steps(eng, mk, n_items, store, steps, P0, 'tc')
    failed = f64_failures(checks)
    assert not failed, '\n'.join(failed)
    eng.close()


def test_tc_step_bitwise_repeatable():
    """Two engines alive in one process, same inputs: the K splits are summed in a fixed order, so every output is bit for bit
    the same."""
    mk, n_items, step_mode = TC_CASES['L344_B48_xe_logq']
    runs = [f64_setup(mk, n_items, step_mode) for _ in range(2)]
    outs = [f64_run_steps(eng, mk, n_items, store, steps, P0, 'tc')[1] for eng, store, steps, P0 in runs]
    for k in outs[0]:
        assert np.array_equal(outs[0][k], outs[1][k]), k
    for r in runs:
        r[0].close()


# (G4R_TS_CLUSTER, G4R_TS_CLUSTER_BIG, G4R_TS_PDL); the first is the default
LAUNCH_CONFIGS = [(8, 16, 1), (8, 16, 0), (8, 8, 1), (1, 16, 1), (2, 8, 1), (4, 16, 1)]


def test_tc_step_launch_configurations(tmp_path):
    """The cluster cap of the K splits, the cluster size of the long-K products and programmatic dependent launch change how the
    products are split and overlapped, not what they compute.  They are read once per process, so every configuration runs the
    L = 344 and L = 512 cases in a worker process (tests/tc_config_worker.py): each passes the float64 comparison, and PDL on / off
    are bitwise identical."""
    res = {}
    for cfg in LAUNCH_CONFIGS:
        out = str(tmp_path / ('cfg_%d_%d_%d.npz' % cfg))
        env = dict(os.environ, G4R_TS_CLUSTER=str(cfg[0]), G4R_TS_CLUSTER_BIG=str(cfg[1]), G4R_TS_PDL=str(cfg[2]))
        p = subprocess.run([sys.executable, os.path.join(HERE, 'tc_config_worker.py'), out, 'L344_B48_xe_logq', 'L512_B256_xelogit'],
                           env=env, capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, '%s: worker failed\n%s' % (cfg, p.stderr[-4000:])
        with np.load(out) as z:
            res[cfg] = {k: z[k] for k in z.files}
        failed = [str(v) for k, v in res[cfg].items() if k.endswith(':failures') and str(v)]
        assert not failed, '%s:\n%s' % (cfg, '\n'.join(failed))
    a, b = res[(8, 16, 1)], res[(8, 16, 0)]
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), 'PDL on / off differ: ' + k
