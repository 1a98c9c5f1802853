"""-m gpu: full-softmax training (full_softmax=True, DESIGN §3n) held to the per-element float64 bound of
tests/full_softmax_oracle.py (full_step_reference / row_update_bounds), every catalogue row at its own scale.

tests/test_gpu_full_softmax.py judges each row table against its largest element; in a full-softmax step at most B target rows
are large, so the other rows -- most of what k_full_stats / k_full_grad / k_full_rows compute -- are barely held.  Here every
element of the update of Wy / By and of each optimizer state tensor, of the gradient recovered from a plain SGD update, and of
dvec / dSx per lane meets the bound, with the row reference built from the step's own final-layer output y (exported after the
hidden dropout: the operand k_full_rows multiplies).  Every case runs on both score tile kinds (eval_tc forced each way), the
launch count of each step showing which ran:
- every case of test_gpu_full_softmax.py, and the RSC15 / Rees46 shapes;
- trained-like spreads (scores spread over about 6-8 per lane) with planted lanes: a target that is the lane's top item by 8
  (p_t ~ 1), hard negatives 0.1 .. 0.5 below the lane's max, targets 40 below the max (p_t ~ 4e-18) and 60 below it
  (p_t ~ 9e-27 < EPS_LOG, where fac = p_t / (p_t + EPS_LOG) collapses the lane's gradient to ~1 %);
- merge edges: one item 100 above every lane's scores in the first tile, then in the padded last tile (the other tiles' sums
  rescale to float32 underflow), and ten items 100 above the rest (every other exp underflows);
- shapes: a catalogue smaller than one tile, more item tiles than 2 x 132 SMs on either kind, B = 65; M < B, duplicated inputs
  and a target that is another lane's input (one Wy row takes both dSx and dSy) come with every case's second step."""
import numpy as np
import pytest

import full_softmax_oracle as fso
import test_gpu_full_softmax as tfs
from gpu_utils import oracle_f64, opt_slots

pytestmark = pytest.mark.gpu

KINDS = {'fp32': False, 'wgmma': True}


def _ulp(a, b):
    return 2.0 ** -23 * (np.abs(a) + np.abs(b))


def _judge_steps(eng, mk, n_items, steps, tc):
    """runs `steps` on the engine, each against the bound from the float64 oracle re-seeded from the device; returns
    {check: worst bound ratio over the steps}"""
    sgd = mk.get('adapt', 'adagrad') is None and not mk.get('momentum', 0) and not mk.get('lmbd', 0)
    lr = mk['learning_rate']
    nl = len(mk['layers'])
    out = {}

    def note(what, r):
        out[what] = max(out.get(what, 0.0), r)
    for k, (X, Y, R) in enumerate(steps):
        m = oracle_f64(eng, mk, n_items, k)
        keys = ['Wy', 'By'] + ['%s.%s' % (n, s) for n in ('Wy', 'By') for s in opt_slots(m)]
        T0 = {n: eng.get(n) for n in keys}
        l0 = eng.kernel_launches()
        eng.train_step(X, Y, R)
        assert eng.kernel_launches() - l0 == tfs._launches(mk, tc), 'expected the %s score tiles' % ('wgmma' if tc else 'fp32')
        M = len(X)
        C, G, E = fso.full_step_reference(m, X, Y, R, eng.get('y%d' % (nl - 1))[:M])
        for i in range(nl):
            note('dvec%d' % i, fso.bound_ratio(eng.get('dvec%d' % i)[:M], G['dvec'][i], E['dvec'][i]))
        if C['mode'] != 'none':
            note('dSx', fso.bound_ratio(eng.get('dSx')[:M], G['dSx'], E['dSx']))
        T1 = {n: eng.get(n) for n in keys}
        shared = C['mode'] == 'shared'
        for lo, hi, cnt, rows in fso.row_update_bounds(m, C, G, E):
            for n, (b, a, allow) in rows.items():
                a0, a1 = T0[n][lo:hi].astype(np.float64), T1[n][lo:hi].astype(np.float64)
                note(n + ' update', fso.bound_ratio(a1 - a0, a - b, allow + cnt[:, None] * _ulp(a0, a1)))
            if sgd:
                for n, g, e in (('Wy', G['dSy'], E['dSy']), ('By', G['dSBy'], E['dSBy'])):
                    g, e = g[lo:hi].copy(), e[lo:hi].copy()
                    if shared and n == 'Wy':
                        sel = (C['X'] >= lo) & (C['X'] < hi)
                        np.add.at(g, C['X'][sel] - lo, G['dSx'][sel])
                        np.add.at(e, C['X'][sel] - lo, E['dSx'][sel])
                    w0, w1 = T0[n][lo:hi].astype(np.float64), T1[n][lo:hi].astype(np.float64)
                    note('d%s recovered' % n, fso.bound_ratio((w0 - w1) / lr, g, e + cnt[:, None] * _ulp(w0, w1) / lr))
    return out


def _check(label, ratios):
    worst = max(ratios.values())
    print('%s: worst bound ratio %.3g (%s)' % (label, worst, ', '.join('%s %.3g' % kv for kv in sorted(ratios.items(), key=lambda kv: -kv[1]))))
    failed = ['%s %.3g' % kv for kv in ratios.items() if not kv[1] <= 1.0]
    assert not failed, label + ': ' + ', '.join(failed)


def _scores(eng, mk, n_items, X, R):
    """float64 scores y . Wy^T + By of the step (X, R) from the engine's state, and the oracle that computed them"""
    m = oracle_f64(eng, mk, n_items, 0)
    M = len(X)
    _, C = fso.forward_full(m, np.asarray(X), M, R=R, masks=m.make_masks(M), H=[h[:M] for h in m.H])
    return C['y_last'] @ m.Wy.T + m.By.reshape(-1), m


def _trained_spread(eng, mk, n_items, X, R):
    """scale Wy and By so that each lane's scores have a standard deviation of about 1.5 (a spread of about 6-8 over the
    catalogue); twice, since with a shared embedding the input rows are Wy rows too"""
    for _ in range(2):
        o, m = _scores(eng, mk, n_items, X, R)
        f = 1.5 / o.std(axis=1).mean()
        eng.set('Wy', (m.Wy * f).astype(np.float32))
        eng.set('By', (m.By * f).astype(np.float32))


def _plant_lanes(eng, mk, n_items, X, Y, R):
    """planted lanes of step 1 (through By only, so y stays): lane 0's target is its top item by 8, lane 1 has hard negatives
    0.1 / 0.3 / 0.5 below its max, lane 2's target is 40 below its max and lane 3's 60 below.  Returns the new Y."""
    Y = np.array(Y)
    o, m = _scores(eng, mk, n_items, X, R)
    By = m.By.reshape(-1).copy()
    used = set(np.asarray(X).tolist())
    rs = np.random.RandomState(11)

    def fresh():
        while True:
            j = int(rs.randint(n_items))
            if j not in used:
                used.add(j)
                return j

    def set_score(b, j, v):            # By_j so that lane b's score of item j is v
        d = v - o[b, j]
        By[j] += d
        o[:, j] += d
    j0 = fresh(); Y[0] = j0
    set_score(0, j0, np.delete(o[0], j0).max() + 8.0)
    for d in (0.1, 0.3, 0.5):
        j = fresh()
        set_score(1, j, np.delete(o[1], j).max() - d)
    Y[1] = fresh()
    for b, d in ((2, 40.0), (3, 60.0)):
        j = fresh(); Y[b] = j
        set_score(b, j, o[b].max() - d)
    eng.set('By', By.astype(np.float32).reshape(-1, 1))
    return Y


def _spike(eng, mk, n_items, X, Y, R, items):
    """items 100 (+ up to 2) above every lane's scores: every other exp underflows in float32.  Half of the lanes take one of
    them as target, the others keep theirs (p_t underflows: the EPS_LOG collapse).  Returns the new Y."""
    Y = np.array(Y)
    o, m = _scores(eng, mk, n_items, X, R)
    By = m.By.reshape(-1).copy()
    top = o.max()
    rs = np.random.RandomState(12)
    for j in items:
        By[j] += top + 100.0 + 2.0 * rs.rand() - o[:, j].min()
    Y[::2] = np.asarray(items)[np.arange(len(Y[::2])) % len(items)]
    eng.set('By', By.astype(np.float32).reshape(-1, 1))
    return Y


def _run(mk, n_items, kind, seed=1, prep=None, n_steps=2):
    eng = tfs._engine(mk, n_items, eval_tc=KINDS[kind])
    steps = tfs._steps(n_items, mk['batch_size'], seed)[:n_steps]
    if prep:
        X, Y, R = steps[0]
        steps[0] = (X, prep(eng, mk, n_items, X, Y, R), R)
    ratios = _judge_steps(eng, mk, n_items, steps, KINDS[kind])
    eng.close()
    return ratios


@pytest.mark.parametrize('kind', sorted(KINDS))
@pytest.mark.parametrize('name', sorted(tfs.CASES))
def test_cases_rows_within_bound(name, kind):
    """every case of test_gpu_full_softmax.py, two steps, on each tile kind"""
    mk, n_items = tfs.CASES[name]
    _check('%s %s' % (name, kind), _run(mk, n_items, kind))


def _trained(eng, mk, n_items, X, Y, R):
    _trained_spread(eng, mk, n_items, X, R)
    return _plant_lanes(eng, mk, n_items, X, Y, R)


@pytest.mark.parametrize('kind', sorted(KINDS))
@pytest.mark.parametrize('name', ['rsc15_xe_shared', 'none_xe_sgd', 'shared_xe_adagrad_drop', 'wide_none_xelogit'])
def test_trained_spread_planted_lanes(name, kind):
    """trained-like spreads with the planted lanes (top target, hard negatives, targets 40 and 60 below the max) in step 1"""
    mk, n_items = dict(tfs.CASES, **tfs.SHIPPED)[name]
    _check('%s trained %s' % (name, kind), _run(mk, n_items, kind, prep=_trained))


def test_rsc15_random_init_fp32_and_wgmma():
    """the RSC15 shape from random init, on each tile kind"""
    mk, n_items = tfs.SHIPPED['rsc15_xe_shared']
    for kind in sorted(KINDS):
        _check('rsc15_xe_shared %s' % kind, _run(mk, n_items, kind, seed=2))


EDGE_MK = tfs._mk(40, 16, constrained_embedding=True, **tfs.ADA)
EDGES = {
    'spike_first_tile': lambda n: [3],
    'spike_last_tile': lambda n: [n - 1],
    'ten_survivors': lambda n: list(range(700, 710)),
}


@pytest.mark.parametrize('kind', sorted(KINDS))
@pytest.mark.parametrize('edge', sorted(EDGES))
def test_merge_edges(edge, kind):
    """one item far above the rest in the first / the padded last tile, ten items above the rest: the other tiles' sums
    rescale to underflow"""
    n_items = 3001
    items = EDGES[edge](n_items)
    prep = lambda eng, mk, n, X, Y, R: _spike(eng, mk, n, X, Y, R, items)
    _check('%s %s' % (edge, kind), _run(EDGE_MK, n_items, kind, prep=prep))


SHAPES = {
    # fewer items than one tile of either kind
    'tiny_catalogue': (tfs._mk(24, 8, constrained_embedding=True, **tfs.ADA), 50),
    # 1094 fp32 tiles / 274 wgmma tiles: more than 2 x 132 SMs on either kind; 70001 is no multiple of 64, 128 or 256
    'many_tiles': (tfs._mk(32, 16, constrained_embedding=True, dropout_p_hidden=0.2, **tfs.ADA), 70001),
    # one lane past a wgmma lane block
    'B65_sgd': (tfs._mk(48, 65), 2500),
}


@pytest.mark.parametrize('kind', sorted(KINDS))
@pytest.mark.parametrize('name', sorted(SHAPES))
def test_shapes(name, kind):
    mk, n_items = SHAPES[name]
    _check('%s %s' % (name, kind), _run(mk, n_items, kind, prep=_trained if name != 'tiny_catalogue' else None))


@pytest.mark.parametrize('spread', ['random', 'trained'])
def test_rees46_one_step(spread):
    """the Rees46 shape (172,000 items, L 512, B 240) on the wgmma tiles, one step"""
    mk, n_items = tfs.SHIPPED['rees46_xe_shared']
    _check('rees46_xe_shared %s wgmma' % spread, _run(mk, n_items, 'wgmma', seed=2, n_steps=1, prep=_trained if spread == 'trained' else None))
