"""-m gpu: the scoring path -- the evaluation / predict GRU forward (eval_forward: k_gather_in, k_f1, k_f2 with train = 0 on the
scoring state He), the predict kernels (k_eval_score<true>, k_predict_act), whole evaluations (g4r_eval_schedule) and the device
top-k -- against a float64 oracle holding the device's float32 weights, at the shapes users run (37,483 items, 512 scoring lanes
over a model batch of 32) and at the edges of the kernels: feature rows wider than one 128-column slab, partial item tiles,
fewer predict lanes than the engine reserves, lane compaction and session resets, evaluations longer than one staging window,
the switch from the wgmma to the fp32 tiles inside one evaluation, dropout configured but not applied when scoring, candidate
subsets with duplicates.  Last, scoring between two training windows must leave training bitwise unchanged."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays
from gpu_utils import F64_REL, F64_RTOL, f64_errors, assert_f64_close, param_names, oracle_param, push_weights, opt_slots

pytestmark = pytest.mark.gpu


def _mk(final_act, **kw):
    loss = {'softmax': 'cross-entropy', 'softmax_logit': 'xe_logit'}.get(final_act, 'bpr-max')
    mk = dict(batch_size=32, n_sample=0, loss=loss, final_act=final_act)
    mk.update(kw)
    return mk


def _engine(n_items, mk, lanes, seed, by_shift=0.0, tc=None):
    """Engine with random weights, output biases (+ by_shift) and GRU biases; its scoring state He is zero."""
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1 + np.float32(by_shift)
    for b in m.Bh:
        b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=tc))
    push_weights(eng, m)
    return eng, rs


def _oracle(eng, mk, n_items, dtype=np.float64):
    """oracle holding the device's float32 weights (float64: the reference; float32: a second float32 implementation)"""
    m = orc.OracleGRU4Rec(dtype=dtype, **mk)
    m.init(n_items)
    for name in param_names(m):
        p = oracle_param(m, name)
        p[...] = eng.get(name).reshape(p.shape)
    return m


def _gru(m, X, H):
    """predict-mode GRU forward of lanes X from states H (one [M, L] array per layer; no dropout): ([y of every layer],
    [new state of every layer])"""
    X = np.asarray(X, np.int64)
    _, C = m.forward(X, X[:1], len(X), predict=True, H=H)          # one score column: the catalogue is scored separately
    return [lc['inp'] for lc in C['layers'][1:]] + [C['y_last']], C['H_new']


def _final(m, o):
    return orc.act_fwd(('softmax', 0, 0) if m.final_act == 'softmax_logit' else m.fact, o)


def _rowwise_errors(dev, ref):
    """f64_errors row by row (a softmax row is judged at its own scale): the worst row's values"""
    dev = np.asarray(dev, np.float64); ref = np.asarray(ref, np.float64)
    if not (np.isfinite(dev).all() and np.isfinite(ref).all()):
        return np.inf, np.inf
    scale = np.maximum(np.abs(ref).max(1, keepdims=True), 1e-30)
    err = np.abs(dev - ref)
    big = np.abs(ref) > 0.01 * scale
    rel = np.where(big, err / np.where(big, np.abs(ref), 1.0), 0.0)
    return float((err / scale).max()), float(rel.max())


# ---------------- A. predict, step by step, re-seeded from the device ----------------
# name -> (n_items, model keywords, scoring lanes, By shift)
PREDICT_CASES = {
    # run.py's serving shape: 512 scoring lanes over a model batch of 32 (the forward writes scratch rows past B)
    'I37483_L100_E512_elu': (37483, _mk('elu-0.5', layers=[100]), 512, 0.0),
    # ldL = 132 > 128: the slab loop of k_eval_score; 3001 = 46 full item tiles + 57
    'I3001_L130_E129_tanh': (3001, _mk('tanh', layers=[130]), 129, 0.0),
    # two layers over a separate embedding, dropout configured on both: scoring must be the dropout-free forward
    'I5000_L96x64_emb48_E300_xe_drop': (5000, _mk('softmax', layers=[96, 64], embedding=48, dropout_p_hidden=0.3, dropout_p_embed=0.3), 300, 0.0),
    # shared embedding, relu mostly below zero: exact ties at 0
    'I2049_shared_L64_E64_relu': (2049, _mk('relu', layers=[64], constrained_embedding=True), 64, -0.35),
    'I4100_L512_E240_softmax_logit': (4100, _mk('softmax_logit', layers=[512]), 240, 0.0),
    'I700_L24_E40_linear': (700, _mk('linear', layers=[24]), 40, 0.0),
    'I700_L24x16_E40_leaky': (700, _mk('leaky-0.1', layers=[24, 16]), 40, 0.0),
    'I700_shared_L20_E40_selu': (700, _mk('selu-1.05-1.67', layers=[20], constrained_embedding=True), 40, 0.0),
}


def _predict_calls(rs, n_items, lanes):
    """(X, reset_mask) of four calls: all lanes; some lanes reset; fewer lanes than the engine reserves; all lanes again"""
    calls = []
    for k, batch in enumerate((lanes, lanes, max(1, (2 * lanes) // 3 - 1), lanes)):
        X = rs.randint(0, n_items, batch).astype(np.int32)
        reset = None if k == 0 else (rs.rand(batch) < 0.25).astype(np.uint8)
        calls.append((X, reset))
    return calls


@pytest.mark.parametrize('case', list(PREDICT_CASES))
def test_predict_matches_float64(case):
    """predict(): y of every layer, the new scoring state and every output score against the float64 forward from the device's
    own state before the call; He rows at or past the call's batch stay bit-identical."""
    n_items, mk, lanes, by = PREDICT_CASES[case]
    eng, rs = _engine(n_items, mk, lanes, seed=1, by_shift=by)
    nl = len(mk['layers'])
    for i in range(nl):
        eng.set('He%d' % i, (rs.randn(*eng.shape('He%d' % i)) * 0.5).astype(np.float32))
    worst = {}
    for k, (X, reset) in enumerate(_predict_calls(rs, n_items, lanes)):
        tag = 'call %d (batch %d of %d lanes) ' % (k, len(X), lanes)
        He0 = [eng.get('He%d' % i) for i in range(nl)]
        m = _oracle(eng, mk, n_items)
        H = [h[:len(X)].astype(np.float64) for h in He0]
        if reset is not None:
            for h in H:
                h[reset.astype(bool)] = 0.0
        ys, Hn = _gru(m, X, H)
        ref = _final(m, ys[-1] @ m.Wy.T + m.By.ravel())
        out = eng.predict(X, reset)
        assert np.isfinite(out).all(), tag + 'non-finite score'
        for i in range(nl):
            assert_f64_close(eng.get('y%d' % i)[:len(X)], ys[i], tag + 'y%d' % i)
            He1 = eng.get('He%d' % i)
            assert_f64_close(He1[:len(X)], Hn[i], tag + 'He%d' % i)
            assert np.array_equal(He1[len(X):].view(np.uint32), He0[i][len(X):].view(np.uint32)), tag + 'He%d rows >= batch changed' % i
        a, r = _rowwise_errors(out, ref)
        assert a <= F64_REL and r <= F64_RTOL, tag + 'scores: worst row max err / max |ref| = %.3g (bar %g), relative %.3g (bar %g)' % (a, F64_REL, r, F64_RTOL)
        worst[k] = (a, r)
    print('%s: worst row score errors per call %s' % (case, {k: '%.2g / %.2g' % v for k, v in worst.items()}))
    eng.close()


# ---------------- B. whole evaluations against float64 rank bounds ----------------
# A device score is known to within delta = 2^-19 (|y| . |w| + |b|) (fp32 fma chains and 3xTF32 tiles stay far inside, as in
# test_gpu_eval_tc._f64_count_bounds) plus the error of the hidden output y itself, which compounds along a session (nothing is
# re-seeded): HID_REL * max |y| per element, so HID_REL * max |y| * ||w||_1 on a score.  A float32 replay of the oracle ends up to
# 2.4e-7 of max |state| (and 1.3e-5 relative, on the elements above 1 % of the max) away from the float64 replay on EVAL_CASES;
# the device sums in another order than numpy's float32 products, so the bars are 8x that.  The same bars judge the device's
# final scoring state and last hidden output.
HID_REL = 2e-6
HID_RTOL = 1e-4
STRADDLE_MAX = 0.01      # events whose rank interval contains a cut-off (the bound there has no teeth)
ITEM_CHUNK = 4096


def _competitors(m, items=None):
    """the score table of the competitors of _bounds, in chunks of columns: (item indices, W, |W|, ||W||_1 per row, b, |b|)"""
    cols = np.arange(m.n_items) if items is None else np.asarray(items, np.int64)
    out = []
    for c0 in range(0, len(cols), ITEM_CHUNK):
        c = cols[c0:c0 + ITEM_CHUNK]
        W, b = m.Wy[c], m.By.ravel()[c]
        out.append((c, W, np.abs(W).T.copy(), np.abs(W).sum(1), b, np.abs(b)))
    return out


def _flat_regions(fact):
    """Pre-activation ranges over which the device's fp32 final activation (act_fwd) is one constant, so that all scores in one
    of them tie exactly: [(from, to, value)].  relu: 0 at and below 0.  tanhf: +-1 past |x| = 10 (1 - tanh(10) = 4e-9, far
    below half an ulp of 1, 3e-8).  elu / selu: expf(x) - 1 rounds to -1 below x = -20 (expf(-20) = 2e-9, against half an ulp
    of 1 of 6e-8), so the score is -p1 (elu) or p1 * (p2 * -1) (selu) there.  CUDA documents tanhf to 2 ulp and expf to 2 ulp,
    which alone would allow 1 - 6e-8 past |x| = 10: no threshold makes an exact 1 follow from the documented bounds.  That
    these functions round to exactly +-1 / -1 there is what the H100's tanhf and expf (and numpy's float32 ones, in
    test_host_eval_rest_f64.py) do, checked by the tests that use it: a library that did not would count those pairs as
    greater or smaller, outside the bracket, and fail them rather than pass a wrong count."""
    kind, p1, p2 = fact
    return {'relu': [(-np.inf, 0.0, 0.0)], 'tanh': [(-np.inf, -10.0, -1.0), (10.0, np.inf, 1.0)],
            'elu': [(-np.inf, -20.0, -p1)], 'selu': [(-np.inf, -20.0, -p1 * p2)]}.get(kind, [])


def _act_interval(m, x, d):
    """(lo, hi, flat): the interval of the device's activated score for the float64 pre-activation scores x +- d (softmax ranks
    by the pre-activation score), widened by 2^-22 relative for the fp32 rounding of the activation itself; flat: index in
    _flat_regions of the region that holds all of x +- d (-1: none), where the interval is that of the region's one value"""
    kind = orc.parse_act(m.final_act)
    lo, hi = (x - d, x + d) if kind[0] in ('softmax', 'softmax_logit') else (orc.act_fwd(kind, x - d), orc.act_fwd(kind, x + d))
    flat = np.full(np.shape(x), -1, np.int8)
    for k, (a, b, v) in enumerate(_flat_regions(kind)):
        inside = (x - d >= a) & (x + d <= b)
        flat[inside] = k
        lo, hi = np.where(inside, v, lo), np.where(inside, v, hi)
    return lo - 2.0 ** -22 * np.abs(lo), hi + 2.0 ** -22 * np.abs(hi), flat


def _bounds(m, tab, y, Y, hid_abs=0.0):
    """Per lane: (#competitors surely above the target, #surely tied with it, #ambiguous) from float64 scores of the float64 hidden
    output y.  Competitors (`tab`, _competitors): the whole catalogue (the target itself included, one sure tie), or a candidate
    list with its duplicates (the target ties with each copy of itself).  A pair is decided when the activation intervals of the
    two scores do not overlap, or when both sit in one flat region of the activation (_flat_regions: an exact tie)."""
    Wy, By = m.Wy, m.By.ravel()
    ay = np.abs(y)
    wt = Wy[Y]
    lo_t, hi_t, f_t = _act_interval(m, (y * wt).sum(1) + By[Y], 2.0 ** -19 * ((ay * np.abs(wt)).sum(1) + np.abs(By[Y])) + hid_abs * np.abs(wt).sum(1))
    lo_t, hi_t, f_t = lo_t[:, None], hi_t[:, None], f_t[:, None]
    gt = np.zeros(len(Y), np.int64); eq = np.zeros(len(Y), np.int64); amb = np.zeros(len(Y), np.int64)
    for c, W, aWT, l1, b, ab in tab:
        lo, hi, f = _act_interval(m, y @ W.T + b, 2.0 ** -19 * (ay @ aWT + ab) + hid_abs * l1)
        own = c[None, :] == Y[:, None]
        g = (lo > hi_t) & ~own
        e = ((f == f_t) & (f_t >= 0)) | own
        a = ~(g | e | (hi < lo_t))
        gt += g.sum(1); eq += e.sum(1); amb += a.sum(1)
    return gt, eq, amb


def _rank_interval(gt, eq, amb, mode):
    lo = {0: gt + 1.0, 1: (gt + eq).astype(np.float64), 2: gt + 0.5 * (eq - 1) + 1.0}[mode]
    return lo, lo + amb


def _replay(eng, mk, n_items, sched, items=None):
    """The device's evaluation schedule (Schedule.export(): X, Y, slots, flags, M) replayed in float64 from zero state, and the
    hidden state of a float32 replay beside it: per event (gt, eq, amb) of _bounds; the final state of every scoring lane; y of
    the last mini-batch (float64); the same two of the float32 replay."""
    ex = sched.export()
    m = _oracle(eng, mk, n_items)
    m32 = _oracle(eng, mk, n_items, np.float32)
    nl = len(mk['layers'])
    Be = eng.shape('He0')[0]
    H = [np.zeros((Be, L)) for L in mk['layers']]
    H32 = [np.zeros((Be, L), np.float32) for L in mk['layers']]
    tab = _competitors(m, items)
    counts = []
    hid_abs = 0.0
    for s in range(sched.n_steps):
        M = int(ex['M'][s])
        X, Y, sl = ex['X'][s, :M], ex['Y'][s, :M].astype(np.int64), ex['slots'][s, :M]
        zero = sl[(ex['F'][s, :M] & 2) != 0]
        for h in H + H32:
            h[zero] = 0
        ys, Hn = _gru(m, X, [h[sl] for h in H])
        ys32, Hn32 = _gru(m32, X, [h[sl] for h in H32])
        for i in range(nl):
            H[i][sl] = Hn[i]; H32[i][sl] = Hn32[i]
        hid_abs = HID_REL * max(float(np.abs(ys[-1]).max()), 1e-30)
        counts.append(_bounds(m, tab, ys[-1], Y, hid_abs))
    gt, eq, amb = (np.concatenate(c) for c in zip(*counts))
    return dict(gt=gt, eq=eq, amb=amb, last=counts[-1], H=H, y=ys, H32=H32, y32=ys32, M=M, hid_abs=hid_abs)


def _cuts(n_items):
    """64 cut-offs (the ABI maximum) spread from 1 to n_items: almost a rank CDF"""
    c = np.unique(np.concatenate([np.arange(1, 17), np.round(np.geomspace(17, n_items, 48))]).astype(np.int32))
    assert len(c) <= 64 and c[-1] == n_items
    return c


def _assert_sums_in_bounds(rec, mrr, n, rp, cuts, mode, tag):
    lo, hi = _rank_interval(rp['gt'], rp['eq'], rp['amb'], mode)
    assert n == len(lo), tag + 'events: device %d, schedule %d' % (n, len(lo))
    c = cuts[None, :].astype(np.float64)
    in_lo, in_hi = hi[:, None] <= c, lo[:, None] <= c
    rec_lo, rec_hi = in_lo.sum(0), in_hi.sum(0)
    with np.errstate(divide='ignore'):
        mrr_lo = np.where(in_lo, 1.0 / hi[:, None], 0.0).sum(0)
        mrr_hi = np.where(in_hi, 1.0 / lo[:, None], 0.0).sum(0)
    bad = np.flatnonzero((rec < rec_lo) | (rec > rec_hi))
    assert bad.size == 0, tag + 'recall sums outside the float64 bounds at cut-offs %s: device %s, bounds %s .. %s' % (
        cuts[bad[:6]], rec[bad[:6]], rec_lo[bad[:6]], rec_hi[bad[:6]])
    tol = 1e-12 * np.maximum(mrr_hi, 1.0)
    bad = np.flatnonzero((mrr < mrr_lo - tol) | (mrr > mrr_hi + tol))
    assert bad.size == 0, tag + 'MRR sums outside the float64 bounds at cut-offs %s: device %s, bounds %s .. %s' % (
        cuts[bad[:6]], mrr[bad[:6]], mrr_lo[bad[:6]], mrr_hi[bad[:6]])
    straddle = float(((lo[:, None] <= c) & (hi[:, None] > c)).any(1).mean())
    assert straddle <= STRADDLE_MAX, tag + '%.3g of the events straddle a cut-off (at most %g): the bounds have no teeth' % (straddle, STRADDLE_MAX)
    return straddle


def _sessions(n_items, n_events, seed):
    """(items, session offsets) of about n_events events in sessions of 2 + Geometric(0.5) - 1 events (at most 20), items drawn
    Zipf-like over the catalogue (synth.make_session_arrays, which needs more events than items)"""
    rs = np.random.RandomState(seed)
    lens = np.minimum(1 + rs.geometric(0.5, size=n_events // 2 + 1), 20)
    lens = lens[:np.searchsorted(np.cumsum(lens), n_events) + 1]
    offset = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    p = 1.0 / np.arange(1.0, n_items + 1)
    items = rs.permutation(n_items)[rs.choice(n_items, size=int(offset[-1]), p=p / p.sum())].astype(np.int64)
    return items, offset


# name -> (n_items, model keywords, scoring lanes, schedule lanes, events, By shift, eval_tc values, modes, candidate subset)
EVAL_CASES = {
    # run.py's evaluation: auto tile choice, wgmma tiles until M < 64, then the fp32 tiles
    'run_py_I37483_L100_E512': (37483, _mk('elu-0.5', layers=[100]), 512, 512, 4500, 0.0, (None,), (0,), False),
    # more than one staging window of 512 mini-batches, on both tile kinds; ldL = 132
    'two_windows_I3000_L130_E64': (3000, _mk('elu-0.5', layers=[130]), 64, 64, 52000, 0.0, (False, True), (0,), False),
    'xe_L96x64_emb48_drop_E200': (5000, _mk('softmax', layers=[96, 64], embedding=48, dropout_p_hidden=0.3, dropout_p_embed=0.3), 200, 200, 2500, 0.0,
                                  (None,), (0,), False),
    'shared_relu_I2049_E64_modes': (2049, _mk('relu', layers=[64], constrained_embedding=True), 64, 64, 1500, -0.35, (None,), (0, 1, 2), False),
    # conservative ranks against a subset can be 0 (evaluation.py:55-56): modes 0 and 2 only
    'tanh_subset_I3000_E100': (3000, _mk('tanh', layers=[48]), 100, 100, 2000, 0.0, (None,), (0, 2), True),
    # a schedule of 300 lanes staged at the stride of 512 scoring lanes
    'strided_B300_E512_I4100': (4100, _mk('elu-0.5', layers=[40]), 512, 300, 2500, 0.0, (None,), (0,), False),
}


@pytest.mark.parametrize('case', list(EVAL_CASES))
def test_evaluation_within_float64_bounds(case):
    """eval_schedule end to end: the Recall / MRR sums at 64 cut-offs inside the float64 rank bounds of every event, the final
    scoring state of every lane and y of the last mini-batch at the hidden-state bar, and the last mini-batch's per-lane counts
    inside their bounds."""
    n_items, mk, lanes, Bs, n_events, by, tcs, modes, subset = EVAL_CASES[case]
    items, offset = _sessions(n_items, n_events, seed=3)
    sched = _lib.Schedule(items, offset, None, Bs, 0, mode=1)
    if case.startswith('two_windows'):
        assert sched.n_steps > 512, sched.n_steps
    cand = None
    if subset:
        rs = np.random.RandomState(4)
        cand = rs.randint(0, n_items, 700)
        cand[:40] = cand[40:80]                                  # duplicates
        ex = sched.export()
        cand[80:120] = np.concatenate([ex['Y'][s, :ex['M'][s]] for s in range(sched.n_steps)])[-40:]   # targets of the last events
    cuts = _cuts(n_items)
    nl = len(mk['layers'])
    rp = None
    for tc in tcs:
        eng, _ = _engine(n_items, mk, lanes, seed=2, by_shift=by, tc=tc)
        if rp is None:
            rp = _replay(eng, mk, n_items, sched, cand)
            d32 = [f64_errors(rp['H32'][i], rp['H'][i]) for i in range(nl)]
        if cand is not None:
            eng.set_eval_items(cand)
        for mode in modes:
            tag = 'eval_tc=%s mode %d: ' % (tc, mode)
            rec, mrr, n = eng.eval_schedule(sched, cuts, mode)
            straddle = _assert_sums_in_bounds(rec, mrr, n, rp, cuts, mode, tag)
            derr = []
            for i in range(nl):
                for what, dev, ref in (('He%d' % i, eng.get('He%d' % i), rp['H'][i]), ('y%d' % i, eng.get('y%d' % i)[:rp['M']], rp['y'][i])):
                    a, r = f64_errors(dev, ref)
                    derr.append((what, a, r))
                    assert a <= HID_REL and r <= HID_RTOL, tag + '%s: max err / max |ref| = %.3g (bar %g), relative %.3g (bar %g)' % (what, a, HID_REL, r, HID_RTOL)
            c = eng.eval_counts(rp['M'])
            gt, eq, amb = rp['last']
            for what, dev, sure in (('#greater', c[:, 0], gt), ('#equal', c[:, 1], eq), ('#greater + #equal', c.sum(1), gt + eq)):
                bad = np.flatnonzero((dev < sure) | (dev > sure + amb))
                assert bad.size == 0, tag + 'last mini-batch %s: lanes %s device %s, float64 sure %s + ambiguous %s' % (
                    what, bad[:8], dev[bad[:8]], sure[bad[:8]], amb[bad[:8]])
            print('%s %s%d mini-batches, %d events, straddling %.4f, ambiguous pairs / event %.3g; state errors device %s, float32 oracle %s' % (
                case, tag, sched.n_steps, n, straddle, rp['amb'].mean(),
                ' '.join('%s %.2g/%.2g' % e for e in derr), ' '.join('%.2g/%.2g' % e for e in d32)))
        eng.close()


# ---------------- C. top-k at the serving shape against float64 ----------------
def _key_intervals(m, y, cols, hid_abs):
    """float64 keys of the device's top-k order (the activated score; the pre-activation score for softmax) of columns `cols` and
    their uncertainty: (key - delta, key + delta) of the scores, through the activation"""
    W, B = m.Wy[cols], m.By.ravel()[cols]
    x = y @ W.T + B
    d = 2.0 ** -19 * (np.abs(y) @ np.abs(W).T + np.abs(B)) + hid_abs * np.abs(W).sum(1)
    kind = orc.parse_act(m.final_act)
    act = (lambda v: v) if kind[0] in ('softmax', 'softmax_logit') else (lambda v: orc.act_fwd(kind, v))
    return act(x - d), act(x + d), x


@pytest.mark.parametrize('tc', [False, True])
def test_topk_serving_shape_is_a_float64_topk(tc):
    """predict_topk at 37,483 items x 512 lanes, k = 20 and 100, unfiltered and filtered (candidates and per-lane exclusions): every
    lane's list is a float64 top-k up to the score uncertainty -- no eligible item left out is surely above a returned one -- of
    eligible, distinct items, best first, and the returned scores meet the float64 bar."""
    n_items, mk, lanes, by = PREDICT_CASES['I37483_L100_E512_elu']
    eng, rs = _engine(n_items, mk, lanes, seed=5, by_shift=by, tc=tc)
    eng.set('He0', (rs.randn(*eng.shape('He0')) * 0.5).astype(np.float32))
    for k, filtered in ((20, False), (100, False), (20, True), (100, True)):
        tag = 'eval_tc=%s k=%d %s: ' % (tc, k, 'filtered' if filtered else 'unfiltered')
        X = rs.randint(0, n_items, lanes).astype(np.int32)
        reset = (rs.rand(lanes) < 0.1).astype(np.uint8)
        He0 = eng.get('He0').astype(np.float64)
        He0[reset.astype(bool)] = 0.0
        m = _oracle(eng, mk, n_items)
        ys, _ = _gru(m, X, [He0])
        y = ys[-1]
        hid_abs = F64_REL * float(np.abs(y).max())
        elig = np.ones((lanes, n_items), bool)
        cand = excl = None
        if filtered:
            cand = rs.choice(n_items, n_items // 3, replace=False)
            mask = np.zeros(n_items, bool); mask[cand] = True
            lo, hi, x = _key_intervals(m, y, cand, hid_abs)
            best = cand[np.argsort(-x, axis=1)[:, :3 * k]]
            # each lane excludes a third of its float64 best candidates and random items
            excl = [np.concatenate([best[b, rs.rand(3 * k) < 1 / 3], rs.randint(0, n_items, 30)]) for b in range(lanes)]
            elig[:] = mask[None, :]
            for b in range(lanes):
                elig[b, excl[b]] = False
        items, scores = eng.predict_topk(X, k, reset, items=cand, exclude=excl)
        assert (items >= 0).all(), tag + 'a lane came back short'
        assert all(len(np.unique(r)) == k for r in items), tag + 'duplicate item in a list'
        assert np.take_along_axis(elig, items.astype(np.int64), 1).all(), tag + 'an ineligible item was returned'
        assert (np.diff(scores, axis=1) <= 0).all(), tag + 'scores are not best first'
        lo, hi, x = _key_intervals(m, y, np.arange(n_items), hid_abs)
        ref = _final(m, x)                 # an elementwise activation: the filters do not change a score
        assert_f64_close(scores, np.take_along_axis(ref, items.astype(np.int64), 1), tag + 'returned scores')
        ret = np.zeros_like(elig); np.put_along_axis(ret, items.astype(np.int64), True, 1)
        floor = np.take_along_axis(hi, items.astype(np.int64), 1).min(1)               # the weakest returned item, at its best
        above = np.where(elig & ~ret, lo, -np.inf).max(1)                              # the strongest item left out, at its worst
        bad = np.flatnonzero(above > floor)
        assert bad.size == 0, tag + 'lanes %s leave out an item surely above a returned one (%s > %s)' % (bad[:8], above[bad[:8]], floor[bad[:8]])
    eng.close()


# ---------------- D. scoring between training windows leaves training unchanged ----------------
# step_mode -> model keywords, n_items
TRAIN_CASES = {
    2: (dict(layers=[100], batch_size=32, n_sample=2048, loss='bpr-max', final_act='elu-0.5', learning_rate=0.2, momentum=0.3), 37483),   # k_fast
    4: (dict(layers=[64], batch_size=48, n_sample=256, loss='cross-entropy', final_act='softmax', constrained_embedding=True, learning_rate=0.05,
             dropout_p_hidden=0.2, dropout_p_embed=0.3), 3000),                                                                            # tensor-core step
    0: (dict(layers=[48, 32], batch_size=24, n_sample=128, loss='top1-max', final_act='tanh', embedding=40, adapt='adam', adapt_params=[0.9, 0.999],
             learning_rate=0.01, dropout_p_hidden=0.1), 3000),                                                                             # per-phase kernels
}


@pytest.mark.parametrize('step_mode', sorted(TRAIN_CASES))
def test_scoring_between_training_windows_changes_nothing(step_mode):
    """The scoring forward reuses the training step's scratch: evaluate + predict + predict_topk between two train_steps windows
    must leave the costs, every parameter, every optimizer state tensor and the training hidden state bit-identical to a twin
    that runs the same two windows without scoring."""
    mk, n_items = TRAIN_CASES[step_mode]
    B, S, n = mk['batch_size'], mk['n_sample'], 6
    lanes = 2 * B + 7
    items, offset, order, _ = make_session_arrays(n_items, 20 * B + 4 * n_items, seed=8)
    sched = _lib.Schedule(items, offset, order, B, S, mode=0)
    esched = _lib.Schedule(*_sessions(n_items, 600, seed=11), None, lanes, 0, mode=1)
    store = np.random.RandomState(9).randint(0, n_items, size=(2 * n + 2, S)).astype(np.int64)
    engs, outs = [], []
    for scoring in (True, False):
        m = orc.OracleGRU4Rec(**mk)
        m.init(n_items)
        eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=store.size, eval_lanes=lanes, step_mode=step_mode))
        push_weights(eng, m)
        eng.set_sample_store(store)
        costs = [eng.train_steps(sched, 0, n)]
        if scoring:
            eng.eval_schedule(esched, [1, 5, 20], 0)
            X = np.random.RandomState(10).randint(0, n_items, lanes).astype(np.int32)
            eng.predict(X)
            eng.predict_topk(X[:B + 3], 20)
        costs.append(eng.train_steps(sched, n, n))
        names = param_names(m)
        state = {nm: eng.get(nm) for nm in names}
        state.update({'%s.%s' % (nm, s): eng.get('%s.%s' % (nm, s)) for nm in names for s in opt_slots(m)})
        state.update({'H%d' % i: eng.get('H%d' % i) for i in range(len(mk['layers']))})
        state['costs'] = np.concatenate(costs)
        outs.append(state)
        engs.append(eng)
    if step_mode == 4:
        assert engs[0].uses_tensor_cores()
    a, b = outs
    assert np.isfinite(a['costs']).all()
    changed = [nm for nm in a if not np.array_equal(a[nm].view(np.uint32), b[nm].view(np.uint32))]
    assert not changed, 'step_mode %d: scoring between the windows changed %s' % (step_mode, changed)
    for e in engs:
        e.close()
