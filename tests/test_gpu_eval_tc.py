"""-m gpu: full-catalogue evaluation on the tensor cores (wgmma 3xTF32 tiles, csrc/g4r_eval_tc.cuh) against the fp32 FFMA
tiles and the oracle's evaluate_gpu restatement (evaluation.py:57-75)."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
from gpu_utils import push_weights

pytestmark = pytest.mark.gpu


def _setup(n_items, L, lanes, seed, final_act='elu-0.5', loss='bpr-max', layers=None):
    mk = dict(layers=layers or [L], batch_size=8, n_sample=16, loss=loss, final_act=final_act)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    df = make_sessions(n_items=n_items, n_events=6 * lanes + 400, seed=seed)
    d = orc.prepare_fit_data(df)
    engs = []
    for tc in (False, True):
        eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=tc))
        push_weights(eng, m)
        engs.append(eng)
    items = d['data_items'] % n_items
    sched = _lib.Schedule(items, d['offset_sessions'], None, lanes, 0, mode=1)
    return m, engs, sched, items, d


@pytest.mark.parametrize('n_items,L,lanes,mode', [(5000, 100, 300, 0), (5000, 100, 300, 1), (3001, 64, 130, 0), (4100, 40, 512, 2), (2500, 224, 96, 0)])
def test_tensor_core_ranking_equals_fp32_tiles(n_items, L, lanes, mode):
    m, (e_ff, e_tc), sched, items, d = _setup(n_items, L, lanes, seed=3)
    cuts = [1, 5, 20]
    r0, q0, n0 = e_ff.eval_schedule(sched, cuts, mode)
    r1, q1, n1 = e_tc.eval_schedule(sched, cuts, mode)
    assert n0 == n1 and n0 > 0
    # 3xTF32 scores agree with fp32 to ~1e-6 relative: a rank moves only on a near-tie between two different items
    np.testing.assert_allclose(r1 / n1, r0 / n0, rtol=1e-4, atol=2.0 / n0)
    np.testing.assert_allclose(q1 / n1, q0 / n0, rtol=1e-4, atol=2.0 / n0)
    e_ff.close(); e_tc.close()


def test_tensor_core_ranking_equals_oracle():
    m, (e_ff, e_tc), sched, items, d = _setup(3000, 100, 200, seed=5, final_act='softmax', loss='cross-entropy')
    cuts = [1, 5, 20]
    r1, q1, n1 = e_tc.eval_schedule(sched, cuts, 0)
    rec, mrr = m.evaluate(items, d['offset_sessions'], batch_size=200, cut_off=cuts, mode='standard')
    np.testing.assert_allclose(r1 / n1, rec, rtol=1e-4, atol=2.0 / n1)
    np.testing.assert_allclose(q1 / n1, mrr, rtol=1e-4, atol=2.0 / n1)
    e_ff.close(); e_tc.close()


def test_tiebreaking_mode_breaks_saturated_ties():
    """mode='tiebreaking' (evaluation.py:55,65): with a relu output most scores saturate at exactly 0; 'standard' ranks the target
    ahead of every tie, 'conservative' behind, the tie-breaking noise puts it in between (about half of the ties ahead)."""
    n_items, lanes = 600, 40
    mk = dict(layers=[16], batch_size=8, n_sample=16, loss='bpr-max', final_act='relu')
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    m.By[:] = -0.35          # pushes most pre-activations below zero
    df = make_sessions(n_items=n_items, n_events=2500, seed=11)
    d = orc.prepare_fit_data(df)
    eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=False))
    push_weights(eng, m)
    sched = _lib.Schedule(d['data_items'] % n_items, d['offset_sessions'], None, lanes, 0, mode=1)
    cuts = [20, 100, 300]
    std = eng.eval_schedule(sched, cuts, 0); cons = eng.eval_schedule(sched, cuts, 1); tb = eng.eval_schedule(sched, cuts, 3); tb2 = eng.eval_schedule(sched, cuts, 3)
    np.testing.assert_array_equal(tb[0], tb2[0])          # deterministic
    assert (cons[0] <= tb[0]).all() and (tb[0] <= std[0]).all()
    assert tb[0][1] < std[0][1] and tb[0][1] > cons[0][1], (std[0], tb[0], cons[0])
    eng.close()
