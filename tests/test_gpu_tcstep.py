"""-m gpu: the tensor-core training step (wgmma 3xTF32 GEMMs with fused epilogues, csrc/g4r_tcstep.cuh) against the oracle:
constrained embedding, one layer -- the family of the reference's shipped parameter files (paramfiles/*_best.py)."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions, make_session_arrays
from gpu_utils import make_cfg, push_weights, compare_weights, assert_step_costs

pytestmark = pytest.mark.gpu

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
