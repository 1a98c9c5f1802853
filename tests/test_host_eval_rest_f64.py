"""CPU checks of the float64 bracket of test_gpu_eval_rest_f64.py, so that a broken bracket cannot pass the GPU tests: the
(#greater, #equal) of a float32 numpy replay of the same weights (a second float32 implementation, summing in another order than
the device) lie inside it on two of its cases, exclude_seen on and off, and its vectorised metric sums restate event_metrics."""
import numpy as np
import pytest

from test_host_eval_rest import event_metrics
from test_gpu_eval_rest import _relevant


@pytest.mark.parametrize('case', ['default_I2049_L100_E100_elu', 'I2049_L64_E300_relu_shift'])
@pytest.mark.parametrize('seen_on', [False, True])
def test_float32_replay_within_bracket(case, seen_on):
    from test_gpu_eval_rest_f64 import CASES, _case, rest_bracket
    n_items, mk = CASES[case][:2]
    m, items, off, sched = _case(case)
    br = rest_bracket(m, mk, n_items, sched, items, off, seen_on=seen_on, f32=True)
    c, miss = br['f32'], br['miss']
    assert miss.any() == seen_on and (c[miss] == -1).all()
    g, e = c[~miss, 0], c[~miss, 1]
    s, q, a = br['gt'][~miss], br['eq'][~miss], br['amb'][~miss]
    for dev, lo in ((g, s), (e, q), (g + e, s + q)):
        bad = np.flatnonzero((dev < lo) | (dev > lo + a))
        assert bad.size == 0, (bad[:8], dev[bad[:8]], lo[bad[:8]], a[bad[:8]])
    assert (a == 0).mean() > 0.5                                          # the bracket decides most pairs
    if case.startswith('I2049_L64_E300_relu'):
        assert (e > 1).mean() > 0.5                                       # ties of the flat region, decided


@pytest.mark.parametrize('seen_on', [False, True])
def test_float32_replay_within_bracket_candidates_and_edges(seen_on):
    """the bracket's candidate-multiset branch (evaluate_rest(items=): unlisted relevant items are misses, each copy of the
    item a tie) and the edge rows of test_rest_edges_inside_one_row"""
    from test_gpu_eval_rest_f64 import CASES, EDGE_ITEMS, _case, _edge_setup, rest_bracket
    from gru4rec_b200 import _lib
    case = 'default_I2049_L100_E100_elu'
    n_items, mk = CASES[case][:2]
    m, items, off, sched = _case(case)
    rs = np.random.RandomState(8)
    cand = np.concatenate([rs.choice(n_items, 1400, replace=False), rs.choice(n_items, 100)])
    runs = [(m, mk, n_items, sched, items, off, cand)]
    emk, em, eitems, eoff = _edge_setup()
    runs.append((em, emk, EDGE_ITEMS, _lib.Schedule(eitems, eoff, None, 16, 0, mode=1 | _lib.SCHED_POSITIONS), eitems, eoff, None))
    for m_, mk_, n_, sched_, items_, off_, cand_ in runs:
        br = rest_bracket(m_, mk_, n_, sched_, items_, off_, cand=cand_, seen_on=seen_on, f32=True)
        c, miss = br['f32'], br['miss']
        assert (c[miss] == -1).all() and miss.any() == (seen_on or cand_ is not None)
        g, e = c[~miss, 0], c[~miss, 1]
        s, q, a = br['gt'][~miss], br['eq'][~miss], br['amb'][~miss]
        for dev, lo in ((g, s), (e, q), (g + e, s + q)):
            bad = np.flatnonzero((dev < lo) | (dev > lo + a))
            assert bad.size == 0, (bad[:8], dev[bad[:8]], lo[bad[:8]], a[bad[:8]])
        assert (a == 0).mean() > 0.5
        if cand_ is not None:
            rel = np.concatenate([_relevant(items_, off_, int(p))[0] for p in sched_.positions()[sched_.counted()]])
            mult = np.bincount(cand_, minlength=n_)[rel]
            assert (miss[mult == 0]).all() and (q[mult[~miss] > 1] >= 2).all()


def test_rest_metrics_restate_event_metrics():
    from test_gpu_eval_rest_f64 import metric_bounds, rest_metrics
    rs = np.random.RandomState(0)
    lens = rs.randint(1, 70, 300)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    r = rs.randint(1, 40, offsets[-1]).astype(np.float64) + 0.5 * rs.randint(0, 2, offsets[-1])   # ties and halves
    r[rs.rand(len(r)) < 0.1] = np.inf                                                            # misses
    cuts = [1, 5, 20, 71]
    want = np.zeros((6, len(cuts)))
    for i in range(len(lens)):
        for j, N in enumerate(cuts):
            want[:, j] += event_metrics(r[offsets[i]:offsets[i + 1]], lens[i], N)
    np.testing.assert_allclose(rest_metrics(r, offsets, cuts), want, rtol=1e-12, atol=0)
    best, worst = metric_bounds(r, r, offsets, cuts)                   # point intervals: the metrics themselves
    np.testing.assert_allclose(best, want, rtol=1e-12, atol=0)
    np.testing.assert_allclose(worst, want, rtol=1e-12, atol=0)
    # wider intervals: the bounds enclose the metrics of every rank vector inside them, MAP across ties included
    lo, hi = np.maximum(r - rs.randint(0, 3, len(r)), 1.0), r + rs.randint(0, 3, len(r))
    best, worst = metric_bounds(lo, hi, offsets, cuts)
    for _ in range(5):
        x = np.where(np.isfinite(r), lo + np.floor(rs.rand(len(r)) * np.where(np.isfinite(r), hi - lo + 1, 0)), np.inf)
        got = rest_metrics(x, offsets, cuts)
        assert (got <= best + 1e-9).all() and (got >= worst - 1e-9).all()
