"""-m gpu: every step of a multi-step training window.  Engine.train_steps runs up to CAP steps in one window -- one launch of
k_fast, of its cluster variant or of k_persistent, or the 16-step unrolled CUDA graph of the per-phase kernels / the tensor-core
step plus the one-step graph for the rest -- and carries data from step s to step s + 1 inside it: rows prefetched or staged for
the next step, GRU weights resident in shared memory, the graphs' device-side step base, dropout masks keyed by the global step.
A window of one step (Engine.train_step, what the float64 tests drive) runs none of that.

The training kernels reduce in a fixed order and use only integer atomics, so the arithmetic of a step does not depend on where
the window boundaries fall: the same N = 37 steps run as one window (A), as 37 one-step windows (B) and as windows of 5 (C,
max_resident_steps = 5: 7 x 5 + 2) must leave bit-identical costs, weights, optimizer state and hidden state.  B is checked step
by step against the float64 oracle (gpu_utils.f64_run_steps, F64_REL / F64_RTOL), so the bitwise equality carries that bar to
every step of the long window.  f64_run_steps fills DSY with NaN before each generic step: the equality also shows that no step
reads a DSY row an earlier step left behind.

Deliberate defects, each invisible to a one-step window, were run once each on an H100 80GB HBM3 (700 W power limit).  In every
failing case run B still met the float64 bar; the bitwise comparison with A failed:
  1. k_fast, fr_dense's row task summing the lanes in reverse order (the row copy of Wh drifts from the column copy in the last
     bit): headline, L120_xe_logq_drop and L50_B13_top1_adagrad-mode2 fail.  The existing -m gpu suite passed in full.
  2. k_fast's F1 of step s + 1 reading the H rows staged for step s (sm.gH[s & 1] instead of hnext): the same three fail.  The
     existing suite: 21 trajectory tests in step_mode 2 fail (golden fixtures, headline-shape parity).
  3. the unrolled graph advancing the step base by 15 instead of 16: adam_embed_2layer_mom_l2, rmsprop_cap_smooth,
     tc_auto_L160_B64 and tc_small_L16_B8 fail.  The existing suite: 26 trajectory tests fail (golden fixtures in step_mode 0,
     the tensor-core whole-epoch runs).
  4. the hidden-dropout mask of the forward keyed on md.wG[0] instead of md.wG[s], in the generic kernels' F2 phase and in
     g4r_tcstep.cuh: rsc15, embed64_2layer_drop, adam_embed_2layer_mom_l2 and tc_small_L16_B8 fail.  The existing suite: 5
     trajectory tests with dropout fail.
Wall time of this module on that H100: 94 to 99 s, about two thirds of it the headline case (the float64 oracle over the
37,483-item tables).  The benchmarked workloads cfg4 and cfg3 were added later, and defects of their edges run once each:
  5. the generic kernels' dBh sum leaving out lanes 64-79 (the partial last lane tile at B = 80): cfg4-mode2 and cfg4-mode0
     fail (run B misses the float64 bar); test_gpu_fp32_f64.py passes in full.
  6. no embedding-dropout mask on the layer-0 input of a model of more than one layer: cfg4-mode2 and cfg4-mode0 fail.
  7. the logQ correction of the sample columns' bias x 0.99 in the tensor-core step's k_ts_prep_tab: cfg3 fails.
With the two workload cases the module takes 164 s on an H100 80GB HBM3 at a 700 W power limit, about 104 s of it the cfg3 case
(37 float64 steps over the full 172,000 x 512 tables, 13.7 GB of host memory at the peak).
"""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from bench import WORKLOADS
from gpu_utils import make_cfg, push_weights, param_names, opt_slots, random_opt_state, f64_run_steps, f64_failures

pytestmark = pytest.mark.gpu

N = 37              # odd; two unrolled graphs (2 x 16) plus 5 steps on the one-step graph; not a multiple of SHORT
SHORT = 5           # max_resident_steps of run C
UNROLL = 16         # steps of the unrolled graph (g4r_lib.cu, graph_unroll)


def _mk(L, B, loss, fact, S=2048, **kw):
    mk = dict(layers=list(L) if isinstance(L, (list, tuple)) else [L], batch_size=B, n_sample=S, loss=loss, final_act=fact, adapt=None,
              learning_rate=0.5, momentum=0.0, sample_alpha=0.5)
    mk.update(kw)
    return mk


ADAGRAD = dict(adapt='adagrad', learning_rate=0.05)
P = 'persistent'

# name -> (model keywords, n_items, {step_mode: kernel path (gpu_utils.STEP_PATHS)}); no embedding unless stated
CASES = {
    # the benched kernel: partner CTAs, rows_done, the resident Wh copies, dropout per global step
    'headline': (_mk(100, 32, 'bpr-max', 'elu-0.5', momentum=0.3, lmbd=1e-3, dropout_p_hidden=0.1, **ADAGRAD), 37483, {2: 'fast'}),
    # the widest GRU group of k_fast
    'L120_xe_logq_drop': (_mk(120, 32, 'cross-entropy', 'softmax', logq=1.0, dropout_p_hidden=0.3), 4000, {2: 'fast'}),
    # L % 4 != 0, odd batch
    'L50_B13_top1_adagrad': (_mk(50, 13, 'top1', 'tanh', momentum=0.3, lmbd=1e-3, **ADAGRAD), 6000, {2: 'fast', 3: 'fast'}),
    # a width only the cluster variant takes
    'L128_top1max': (_mk(128, 32, 'top1-max', 'tanh'), 4000, {3: 'fast'}),
    # k_persistent, shared embedding: X[t+1] = Y[t] reads the Wy row step t just updated
    'rsc15': (_mk(100, 32, 'cross-entropy', 'softmax', constrained_embedding=True, logq=1.0, dropout_p_hidden=0.4, momentum=0.2, **ADAGRAD),
              8000, {1: P}),
    # two layers over E rows, both dropouts
    'embed64_2layer_drop': (_mk([96, 100], 32, 'bpr-max', 'elu-0.5', embedding=64, dropout_p_hidden=0.2, dropout_p_embed=0.3), 5000, {1: P}),
    # the graphs (graphU + graph1) of the per-phase kernels; adam's per-element countt; dropout keyed by the graphs' step base
    'adam_embed_2layer_mom_l2': (_mk([48, 64], 32, 'bpr-max', 'elu-0.5', embedding=32, adapt='adam', adapt_params=[0.9, 0.999],
                                     learning_rate=0.01, momentum=0.3, lmbd=1e-3, dropout_p_hidden=0.1), 4000, {0: 'phases'}),
    # the two-pass graph nodes (grad_cap below the gradient norm) and the smoothing statistics
    'rmsprop_cap_smooth': (_mk(64, 32, 'cross-entropy', 'softmax', adapt='rmsprop', adapt_params=[0.9], learning_rate=0.01, grad_cap=1e-2,
                               smoothing=0.1), 4000, {0: 'phases'}),
    # the tensor-core step, chosen automatically (L >= 160), under graphU
    'tc_auto_L160_B64': (_mk(160, 64, 'bpr-max', 'elu-0.5', constrained_embedding=True, momentum=0.4, **ADAGRAD), 4000, {2: 'tc'}),
    # the tensor-core step with K padding of every operand, under graphU; both dropouts
    'tc_small_L16_B8': (_mk(16, 8, 'cross-entropy', 'softmax', S=32, constrained_embedding=True, logq=1.0, dropout_p_hidden=0.2,
                            dropout_p_embed=0.3), 300, {4: 'tc'}),
    # benchmarked workload cfg4: three shared layers at B = 80 (a partial last lane tile of the generic kernels), both dropouts,
    # Adagrad + momentum, BPR-max; on k_persistent and on the per-phase graphs
    'cfg4': (dict(WORKLOADS['cfg4']['model']), WORKLOADS['cfg4']['n_items'], {2: P, 0: 'phases'}),
    # benchmarked workload cfg3 on the tensor-core step under graphU: Adagrad over the full 172,000-row Wy, embedding dropout on
    # the shared input, logQ, B = 240
    'cfg3': (dict(WORKLOADS['cfg3']['model']), WORKLOADS['cfg3']['n_items'], {2: 'tc'}),
}
PARAMS = [(name, sm) for name in CASES for sm in CASES[name][2]]


def _window(n_items, B, S, seed):
    """(Schedule, the oracle's steps of the window, its first step, sample store of N rows).  Every sample row holds the same
    S / 8 items, 8 copies each, in another order: each row step t updates is read again by step t + 1, and a duplicate group
    stays within a chunk of k_fast (32 columns).  Sessions of one repeated item (X[t+1] = X[t]: the Wx0 / E row step t updated is
    F1's input in step t + 1), sessions drawn from the sampled items (targets among the samples), sessions that end inside the
    window; the window ends in the epoch's shrinking tail (M < B, lanes compacted: slot != lane)."""
    rs = np.random.RandomState(seed)
    pool = rs.choice(n_items, S // 8, replace=False)
    store = np.stack([rs.permutation(np.repeat(pool, 8)) for _ in range(N)]).astype(np.int64)
    n_sess = 12 * B
    lens = rs.randint(2, 10, n_sess)
    sess = []
    for k, n in enumerate(lens):
        if k % 5 == 0:
            sess.append(np.full(n, pool[rs.randint(len(pool))] if k % 10 == 0 else rs.randint(n_items)))
        elif k % 5 == 1:
            sess.append(pool[rs.randint(0, len(pool), n)])
        else:
            sess.append(rs.randint(0, n_items, n))
    items = np.concatenate(sess).astype(np.int64)
    offset = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    order = np.arange(n_sess, dtype=np.int64)
    sched = _lib.Schedule(items, offset, order, B, S, mode=0)
    steps = orc.build_train_schedule(items, offset, order, B, S)
    M = np.array([st['M'] for st in steps])
    last = int(np.flatnonzero(M <= (3 * B) // 4)[0])
    first = last + 1 - N
    win = steps[first:last + 1]
    assert first >= 0 and win[0]['M'] == B and win[-1]['M'] < B, (first, win[0]['M'], win[-1]['M'])
    assert not np.array_equal(win[-1]['slots'], np.arange(win[-1]['M'])), 'the lanes of the last step are not compacted'
    assert sum(st['R'].sum() for st in win) >= B, 'too few sessions end inside the window'
    assert any(np.isin(st['X'], pool).any() for st in win), 'no input item among the samples'
    assert any(np.isin(st['Y'], pool).any() for st in win), 'no target among the samples'
    # the device's schedule is the oracle's
    e = sched.export()
    for k, st in enumerate(win):
        m = st['M']
        assert e['M'][first + k] == m
        for key, dev in (('X', e['X']), ('Y', e['Y']), ('slots', e['slots'])):
            np.testing.assert_array_equal(dev[first + k, :m], st[key])
        np.testing.assert_array_equal(e['F'][first + k, :m] & 1, st['R'].astype(np.uint8))
    return sched, win, first, store


def _engine(mk, n_items, step_mode, store, seed, resident=0):
    """Engine with the state every run of a case starts from: random weights, hidden state and biases, logQ support, random
    non-zero optimizer state and the sample store."""
    rs = np.random.RandomState(seed)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    for h in m.H:
        h[:] = rs.randn(*h.shape).astype(np.float32) * 0.5
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    for b in m.Bh:
        b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=store.size, step_mode=step_mode, max_resident_steps=resident))
    push_weights(eng, m)
    eng.set_sample_store(store)
    P0 = None
    if mk.get('logq', 0):
        P0 = rs.randint(1, 50, size=n_items).astype(np.float32)
        eng.set_logq_support(P0)
    random_opt_state(eng, m, np.random.RandomState(seed + 1))
    return eng, m, P0


def _counters(eng):
    return np.array((eng.kernel_launches(),) + tuple(eng.fast_windows()))


def _expected(path, windows, per_step, step_mode):
    """(kernel launches, role-specialised windows, fallback windows) of `windows` on `path`: k_plan plus one launch of k_fast /
    k_persistent per window (a fallback window in step_modes 2 / 3), or k_plan, `per_step` launches per step, the unrolled
    graphs and the one-step graphs"""
    if path in ('fast', P):
        return np.array((2 * len(windows), len(windows) if path == 'fast' else 0, len(windows) if path == P and step_mode >= 2 else 0))
    return np.array((sum(1 + w * per_step + w // UNROLL + w % UNROLL for w in windows), 0, 0))


def _state(eng, m, costs):
    names = param_names(m)
    out = {n: eng.get(n) for n in names}
    out.update({'%s.%s' % (n, s): eng.get('%s.%s' % (n, s)) for n in names for s in opt_slots(m)})
    out.update({'H%d' % i: eng.get('H%d' % i) for i in range(len(m.layers))})
    out['costs'] = np.asarray(costs, np.float32)
    return out


@pytest.mark.parametrize('name,step_mode', PARAMS, ids=['%s-mode%d' % p for p in PARAMS])
def test_window_equals_one_step_windows(name, step_mode):
    """The same 37 steps as one window (A), as 37 one-step windows (B, each step against the float64 oracle at the step's
    slots) and as windows of 5 (C): bit-identical costs of every step, parameters, optimizer state and hidden state; the
    handle's counters show the intended kernel in every window of every run."""
    mk, n_items, modes = CASES[name]
    path = modes[step_mode]
    sched, steps, first, store = _window(n_items, mk['batch_size'], mk['n_sample'], seed=3)
    seed = 5

    # B: one-step windows, each against float64
    eng, m, P0 = _engine(mk, n_items, step_mode, store, seed)
    c0 = _counters(eng)
    costs_b = []

    def run(k, X, Y, R):
        costs_b.append(eng.train_steps(sched, first + k, 1)[0])
        return costs_b[-1]

    checks, _, scales = f64_run_steps(eng, mk, n_items, store, steps, P0, path, run=run, keep_weights=False)
    failed = f64_failures(checks)
    assert not failed, '\n'.join(failed)
    if mk.get('grad_cap', 0):
        assert max(scales) < 1, scales
    delta = _counters(eng) - c0
    per_step = None if path in ('fast', P) else delta[0] // N - 2
    states = {'B': _state(eng, m, costs_b)}
    counts = {'B': (delta, _expected(path, [1] * N, per_step, step_mode))}
    assert eng.uses_tensor_cores() == (path == 'tc')
    eng.close()

    for run_name, resident, windows in (('A', 0, [N]), ('C', SHORT, [SHORT] * (N // SHORT) + [N % SHORT])):
        eng, m, _ = _engine(mk, n_items, step_mode, store, seed, resident)
        assert eng.uses_tensor_cores() == (path == 'tc')
        c0 = _counters(eng)
        costs = eng.train_steps(sched, first, N)
        counts[run_name] = (_counters(eng) - c0, _expected(path, windows, per_step, step_mode))
        states[run_name] = _state(eng, m, costs)
        eng.close()

    for run_name, (got, want) in counts.items():
        assert np.array_equal(got, want), '%s: kernel launches, role-specialised windows, fallback windows %s, expected %s on the %s path' % (
            run_name, got.tolist(), want.tolist(), path)
    a = states['A']
    assert np.isfinite(a['costs']).all()
    for run_name in ('B', 'C'):
        other = states[run_name]
        differ = [k for k in a if not np.array_equal(a[k].view(np.uint32), other[k].view(np.uint32))]
        if 'costs' in differ:
            diff = np.flatnonzero(a['costs'].view(np.uint32) != other['costs'].view(np.uint32))
            differ.append('first differing step %d of %d' % (diff[0], N))
        assert not differ, 'one window of %d steps and run %s differ: %s' % (N, run_name, differ)
