"""-m gpu: full-catalogue evaluation on the tensor cores (wgmma 3xTF32 tiles, csrc/g4r_eval_tc.cuh) against the fp32 FFMA
tiles and the oracle's evaluate_gpu restatement (evaluation.py:57-75)."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
from gpu_utils import push_weights

pytestmark = pytest.mark.gpu


def _setup(n_items, L, lanes, seed, final_act='elu-0.5', loss='bpr-max', layers=None, by=None):
    mk = dict(layers=layers or [L], batch_size=8, n_sample=16, loss=loss, final_act=final_act)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1 if by is None else by
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


RANKING_CASES = [(5000, 100, 300, 0, 'elu-0.5'), (5000, 100, 300, 1, 'elu-0.5'), (3001, 64, 130, 0, 'elu-0.5'), (4100, 40, 512, 2, 'elu-0.5'),
                 (2500, 224, 96, 0, 'elu-0.5'),
                 # relu below zero: most items tie exactly with the target; the last item tile is mostly padding, which must not
                 # count as ties (cut-offs at the tied ranks)
                 (300, 64, 130, 1, 'relu'), (300, 64, 130, 2, 'relu')]


# ids n_items-L-lanes-mode, with the activation appended when it is not the default elu-0.5
@pytest.mark.parametrize('n_items,L,lanes,mode,act', [pytest.param(*c, id='-'.join(map(str, c[:4] if c[4] == 'elu-0.5' else c)))
                                                      for c in RANKING_CASES])
def test_tensor_core_ranking_equals_fp32_tiles(n_items, L, lanes, mode, act):
    m, (e_ff, e_tc), sched, items, d = _setup(n_items, L, lanes, seed=3, final_act=act, by=-0.35 if act == 'relu' else None)
    cuts = [20, 200, n_items] if act == 'relu' else [1, 5, 20]
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


# ---------------- per-lane counts against float64 ----------------
def _count_setup(n_items, L, M, fact, by, tc, seed=7):
    """One mini-batch of M lanes (M sessions of two events, eval_lanes = M) on an engine with the given scoring tiles."""
    mk = dict(layers=[L], batch_size=8, n_sample=16, loss='cross-entropy' if fact == 'softmax' else 'bpr-max', final_act=fact)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1 + by
    items = rs.randint(0, n_items, size=2 * M).astype(np.int64)
    sched = _lib.Schedule(items, np.arange(0, 2 * M + 1, 2, dtype=np.int32), None, M, 0, mode=1)
    eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=M, step_mode=1, eval_tc=tc))
    push_weights(eng, m)
    return m, eng, sched


def _f64_count_bounds(m, y, Y):
    """Per lane: (#surely greater, #surely equal incl. the target, #ambiguous) from float64 scores of the device's hidden output y.
    A score is only known to within delta_i = 2^-19 (sum_k |y_k w_ik| + |b_i|) -- the fp32 FMA chain of the target score and
    the 3xTF32 tiles both stay far inside -- so a pair is decided when the activation intervals of the two scores do not overlap,
    or when both intervals sit in one flat region of the activation (relu below zero: an exact tie)."""
    Wy, By = m.Wy.astype(np.float64), m.By.astype(np.float64).ravel()
    y = y.astype(np.float64)
    x = y @ Wy.T + By
    delta = 2.0 ** -19 * (np.abs(y) @ np.abs(Wy).T + np.abs(By))
    kind = orc.parse_act(m.final_act)
    act = (lambda v: v) if kind[0] in ('softmax', 'softmax_logit') else (lambda v: orc.act_fwd(kind, v))
    lo, hi = act(x - delta), act(x + delta)
    lo, hi = lo - 2.0 ** -22 * np.abs(lo), hi + 2.0 ** -22 * np.abs(hi)        # fp32 rounding of the activation itself
    b = np.arange(len(Y))
    lo_t, hi_t = lo[b, Y][:, None], hi[b, Y][:, None]
    gt = lo > hi_t
    lt = hi < lo_t
    eq = (lo == hi) & (lo == lo_t) & (lo_t == hi_t)
    amb = ~(gt | lt | eq)
    for a in (gt, eq, amb):
        a[b, Y] = False                   # the target's own column: one tie, always
    return gt.sum(1), eq.sum(1) + 1, amb.sum(1)


COUNT_CASES = [(257, 32, 1, 'linear', 0.0), (256, 31, 128, 'relu', -0.35), (2049, 64, 129, 'relu', 0.0), (3001, 63, 127, 'leaky-0.1', 0.0),
               (2500, 40, 64, 'selu-1.05-1.67', 0.0), (5000, 100, 300, 'elu-0.5', 0.0), (4100, 224, 256, 'tanh', 0.0), (3000, 100, 200, 'softmax', 0.0)]


@pytest.mark.parametrize('n_items,L,M,fact,by', COUNT_CASES)
def test_lane_counts_match_float64(n_items, L, M, fact, by):
    """(#greater, #equal) of every lane from the wgmma tiles (eval_tc 2) and the fp32 tiles (eval_tc 1) against float64 scores of
    the device's own hidden output: sure <= device <= sure + ambiguous, ambiguous pairs under 0.1 %, and both tile kinds
    identical on every lane without an ambiguous pair.  256 and 2049 items: relu ties with and without a padded last tile."""
    counts = {}
    for tc in (True, False):
        m, eng, sched = _count_setup(n_items, L, M, fact, by, tc)
        assert sched.n_steps == 1
        Y = sched.export()['Y'][0, :M]
        eng.eval_schedule(sched, [1, 5, 20], 0)
        c = eng.eval_counts(M)
        gt, eq, amb = _f64_count_bounds(m, eng.get('y0')[:M], Y)
        assert amb.sum() < 1e-3 * M * n_items, (amb.sum(), M * n_items)
        for what, dev, sure in (('#greater', c[:, 0], gt), ('#equal', c[:, 1], eq)):
            bad = np.flatnonzero((dev < sure) | (dev > sure + amb))
            assert bad.size == 0, '%s tiles, %s: lanes %s device %s, float64 sure %s + ambiguous %s' % (
                'wgmma' if tc else 'fp32', what, bad[:8], dev[bad[:8]], sure[bad[:8]], amb[bad[:8]])
        counts[tc] = c
        eng.close()
    clean = amb == 0
    np.testing.assert_array_equal(counts[True][clean], counts[False][clean])


def test_rank_sums_follow_the_counts():
    """k_eval_rank: the Recall / MRR sums of modes 0, 1, 2 are exactly those of the lane counts (evaluation.py:60-75)."""
    n_items, L, M, fact, by = 2049, 64, 129, 'relu', 0.0
    m, eng, sched = _count_setup(n_items, L, M, fact, by, True)
    cuts = [1, 20, 500, n_items]
    for mode in (0, 1, 2):
        rec, mrr, n = eng.eval_schedule(sched, cuts, mode)
        c = eng.eval_counts(M).astype(np.float64)
        gt, eq = c[:, 0], c[:, 1]
        rank = {0: gt + 1, 1: gt + eq, 2: gt + 0.5 * (eq - 1) + 1}[mode]
        hit = rank[:, None] <= np.asarray(cuts)[None, :]
        np.testing.assert_array_equal(rec, hit.sum(0), err_msg='mode %d' % mode)
        np.testing.assert_allclose(mrr, (hit / rank[:, None]).sum(0), rtol=1e-12, err_msg='mode %d' % mode)
    eng.close()
