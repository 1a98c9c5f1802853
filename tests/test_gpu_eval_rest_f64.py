"""-m gpu: rest-of-session ranking (Engine.eval_rest; csrc/g4r_rest.cuh, DESIGN §3m) against a float64
restatement at the shapes users run.  test_gpu_eval_rest.py pins the fp32 counts bitwise at one small shape; here:

- the float64 bracket: the evaluation schedule replayed in float64 from zero state (test_gpu_scoring_f64: _oracle, _gru, the
  HID_REL error model of a hidden output compounded along a session); every counted event's score row and its error half-width
  computed once, every relevant item of the event judged against it: (#surely greater, #surely equal -- itself, each copy of
  itself in a candidate list, and every score of the same flat activation region, _flat_regions --, #ambiguous) over the
  device's competitors (the catalogue or a candidate multiset, less the session's inputs under exclude_seen); a seen or
  unlisted relevant item is a miss
- CASES: several lane blocks of 128 on the wgmma tiles, passes 1 and 2 on more than 128 rows, padded last item tiles, a layer
  width whose bias column falls in a later or partial K chunk, more item tiles than SMs (a CTA sweeps several per lane block),
  every final activation with flat or saturated regions, two forwards (two layers over an embedding, a constrained embedding),
  history schedules; each on the fp32 tiles, the wgmma tiles and the automatic choice (shown by the launch counts: +2 per fp32
  pass, +3 per wgmma pass, a unit with pass 0 on wgmma and a later pass on fp32), modes 0 / 1 / 2, exclude_seen off and on
- every pair's counts inside the bracket; equal on every decided pair across the tile choices; the fp32 counts bitwise the
  pair-replication workaround (test_gpu_eval_rest._workaround) on a sample of events; the miss pattern the host's
- the six metric sums inside the sums of the metrics at the two ends of the float64 rank intervals, which differ by < 1 %
- edges inside one row, on both tile kinds: the padded last tile and item 0, exact twins, the row's lowest threshold (the
  skipped search), rows of exactly 32, 33 and 64 relevant items, seen items mixed into a long row
- evaluation.evaluate_rest with default arguments and with items= on a GRU4Rec holding the weights
The bracket itself is checked on the CPU (test_host_eval_rest_f64.py): a float32 numpy replay of the same weights lies inside
it (the catalogue, a candidate multiset, the edge rows), and the vectorised metric sums restate event_metrics."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gpu_utils import push_weights, oracle_param
from test_gpu_scoring_f64 import HID_REL, _act_interval, _flat_regions, _gru, _mk, _oracle, _rank_interval, _sessions
from test_gpu_eval_rest import _relevant, _workaround

pytestmark = pytest.mark.gpu

PAIR_CHUNK = 1 << 22        # pair x item elements judged at once
TC_N = 256                  # items per wgmma tile (csrc/g4r_eval_tc.cuh)


class _Weights(object):
    """the weights of a float32 oracle model behind Engine.get, for _oracle"""

    def __init__(self, m):
        self.m = m

    def get(self, name):
        return oracle_param(self.m, name)


# name -> (n_items, model keywords, lanes, (long sessions, their length), short-session events, By shift, tanh-saturated Wy
#          scale, history)
CASES = {
    # evaluate_rest's default: 100 lanes; 2049 = 8 full item tiles + 1; L + 1 = 101 spans four K chunks
    'default_I2049_L100_E100_elu': (2049, _mk('elu-0.5', layers=[100]), 100, (12, 80), 1500, 0.0, 0.0, False),
    # a second lane block holding one row; a history schedule
    'I3001_L63_E129_leaky': (3001, _mk('leaky-0.1', layers=[63]), 129, (10, 76), 1800, 0.0, 0.0, True),
    # relu mostly below zero: wide flat-region intervals and ties everywhere; three lane blocks, passes 1 and 2 on > 128 rows
    'I2049_L64_E300_relu_shift': (2049, _mk('relu', layers=[64]), 300, (140, 76), 1200, -0.35, 0.0, False),
    # more item tiles (147) than SMs; a third of the catalogue scaled into tanh's saturated tails
    'I37483_L100_E512_tanh_sat': (37483, _mk('tanh', layers=[100]), 512, (6, 72), 2500, 0.0, 60.0, False),
    'I4100_L130_E240_softmax_logit': (4100, _mk('softmax_logit', layers=[130]), 240, (20, 75), 1500, 0.0, 0.0, False),
    # 128 lanes: one full lane block; a history schedule
    'I2500_L40_E128_selu': (2500, _mk('selu-1.05-1.67', layers=[40]), 128, (10, 70), 1500, 0.0, 0.0, True),
    'I2300_L48x32_emb40_E160_elu': (2300, _mk('elu-1', layers=[48, 32], embedding=40), 160, (10, 70), 1500, 0.0, 0.0, False),
    'I2200_shared_L56_E200_linear': (2200, _mk('linear', layers=[56], constrained_embedding=True), 200, (10, 70), 1500, 0.0, 0.0, False),
}


def _model(n_items, mk, seed, by_shift=0.0, sat=0.0):
    """float32 oracle model with random weights, output biases (+ by_shift) and GRU biases; sat: every third item's Wy row
    scaled by it (its scores mostly in tanh's saturated tails)"""
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1 + np.float32(by_shift)
    for b in m.Bh:
        b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    if sat:
        m.Wy[::3] *= np.float32(sat)
        m.By *= np.float32(10.0)                  # a wider spread of the other items' scores: fewer of them within the error bar
    return m


def _engine(n_items, mk, m, lanes, tc):
    eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=lanes, step_mode=1, eval_tc=tc))
    push_weights(eng, m)
    return eng


def _data(n_items, n_long, long_len, n_short, seed):
    """n_long sessions of long_len events first (they fill the first lanes together: rows of more than 32 and 64 distinct later
    items in the same mini-batch), mostly distinct items with some repeats; then short sessions (_sessions) of n_short events"""
    rs = np.random.RandomState(seed)
    items, lens = [], []
    for _ in range(n_long):
        seq = rs.choice(n_items, long_len, replace=False)
        rep = rs.rand(long_len) < 0.03
        seq[rep] = seq[np.maximum(0, np.arange(long_len)[rep] - rs.randint(1, 20, rep.sum()))]
        items.append(seq)
        lens.append(long_len)
    si, so = _sessions(n_items, n_short, seed + 1)
    items = np.concatenate(items + [si]).astype(np.int64) if n_long else si
    off = np.concatenate([[0], np.cumsum(lens), np.sum(lens) + so[1:]]).astype(np.int32)
    return items, off


def _history(off, seed):
    """leading history events of every session: none for a third, else up to half of it"""
    rs = np.random.RandomState(seed)
    lens = np.diff(off)
    return np.where(rs.rand(len(lens)) < 1 / 3, 0, (lens * rs.rand(len(lens)) / 2).astype(np.int32)).astype(np.int32)


def _case(case):
    n_items, mk, lanes, (n_long, long_len), n_short, by, sat, hist = CASES[case]
    m = _model(n_items, mk, seed=1, by_shift=by, sat=sat)
    items, off = _data(n_items, n_long, long_len, n_short, seed=2)
    nh = _history(off, seed=3) if hist else None
    sched = _lib.Schedule(items, off, None, lanes, 0, mode=1 | _lib.SCHED_POSITIONS, n_history=nh)
    return m, items, off, sched


def rest_bracket(m, mk, n_items, sched, items, off, cand=None, seen_on=False, f32=False):
    """The float64 bracket of every (counted event, relevant item) pair of eval_rest, in its order.  Returns a dict: gt, eq, amb
    (int64 per pair, #surely greater / #surely equal / #ambiguous competitors), miss (bool per pair), offsets (int64, each
    event's pairs), rows (per mini-batch of the schedule, the pair count of each counted row), and with f32 the (#greater,
    #equal) of a float32 numpy replay of the same weights (f32: int64 [pairs, 2], -1 on misses).
    The error bar is test_gpu_scoring_f64's: HID_REL was set there on sessions of at most 20 events, and the hidden output's
    error compounds along a session.  It was checked again at the 65 - 80-event sessions of CASES and the edge rows: the float32
    replay lies inside the bracket there (test_host_eval_rest_f64.py), and so do the device's counts on both tile kinds."""
    m64 = _oracle(_Weights(m), mk, n_items)
    m32 = _oracle(_Weights(m), mk, n_items, np.float32) if f32 else None
    ex, P, cnt = sched.export(), sched.positions(), sched.counted()
    W, B = m64.Wy, m64.By.ravel()
    aWT, l1, ab = np.abs(W).T.copy(), np.abs(W).sum(1), np.abs(B)
    w = np.ones(n_items) if cand is None else np.bincount(np.asarray(cand, np.int64), minlength=n_items).astype(np.float64)
    w32 = w.astype(np.float32)                          # counts below 2^24: exact in float32 sums
    nf = len(_flat_regions(orc.parse_act(m.final_act)))
    soft = m.final_act in ('softmax', 'softmax_logit')
    H = [np.zeros((sched.batch_size, L)) for L in mk['layers']]
    H32 = [np.zeros((sched.batch_size, L), np.float32) for L in mk['layers']]
    seen = {}
    out = dict(gt=[], eq=[], amb=[], miss=[], f32=[], lens=[], rows=[])
    for s in range(sched.n_steps):
        M = int(ex['M'][s])
        X, sl = ex['X'][s, :M], ex['slots'][s, :M].astype(np.int64)
        zero = (ex['F'][s, :M] & 2) != 0
        for h in H + H32:
            h[sl[zero]] = 0
        ys, Hn = _gru(m64, X, [h[sl] for h in H])
        for i in range(len(H)):
            H[i][sl] = Hn[i]
        if f32:
            ys32, Hn32 = _gru(m32, X, [h[sl] for h in H32])
            for i in range(len(H)):
                H32[i][sl] = Hn32[i]
        for b in range(M):
            if zero[b] or sl[b] not in seen:
                seen[sl[b]] = set()
            seen[sl[b]].add(int(X[b]))
        rows = np.flatnonzero(cnt[s, :M])
        if not len(rows):
            continue
        y = ys[-1][rows]
        hid_abs = HID_REL * max(float(np.abs(ys[-1]).max()), 1e-30)
        lo, hi, flat = _act_interval(m64, y @ W.T + B, 2.0 ** -19 * (np.abs(y) @ aWT + ab) + hid_abs * l1)
        elig = np.broadcast_to(w > 0, lo.shape).copy()
        seen_r = [seen[sl[b]] if seen_on else set() for b in rows]
        for r, sr in enumerate(seen_r):
            elig[r, list(sr)] = False
        S = np.full((len(rows), max([len(x) for x in seen_r] + [1])), n_items, np.int64)
        for r, sr in enumerate(seen_r):
            S[r, :len(sr)] = sorted(sr)
        lo_x = np.concatenate([lo, np.full((len(rows), 1), -np.inf)], 1)       # column n_items: the padding of S, never counted
        hi_x = np.concatenate([hi, np.full((len(rows), 1), np.inf)], 1)
        ew = np.where(elig, w[None, :], 0.0)
        tot = ew.sum(1)
        F = np.stack([np.where(flat == k, ew, 0.0).sum(1) for k in range(nf)], 1) if nf else None
        if f32:
            sc = ys32[-1][rows] @ m32.Wy.T + m32.By.ravel()
            if not soft:
                sc = orc.act_fwd(orc.parse_act(m.final_act), sc)
        pr, pj = [], []
        for r, b in enumerate(rows):
            rel = _relevant(items, off, int(P[s, b]))[0]
            out['lens'].append(len(rel))
            pr += [r] * len(rel); pj += rel
        out['rows'].append(np.array(out['lens'][-len(rows):]))
        pr, pj = np.array(pr, np.int64), np.array(pj, np.int64)
        miss = np.array([j in seen_r[r] for r, j in zip(pr, pj)], bool) | (w[pj] == 0)
        step = max(1, PAIR_CHUNK // n_items)
        for c0 in range(0, len(pr), step):
            r, j = pr[c0:c0 + step], pj[c0:c0 + step]
            lo_t, hi_t, f_t = lo[r, j], hi[r, j], flat[r, j]
            if cand is None:              # the catalogue: count over it, then take the row's seen items back out (S: padded lists)
                gt = np.count_nonzero(lo[r] > hi_t[:, None], axis=1) - (lo_x[r[:, None], S[r]] > hi_t[:, None]).sum(1)
                lt = np.count_nonzero(hi[r] < lo_t[:, None], axis=1) - (hi_x[r[:, None], S[r]] < lo_t[:, None]).sum(1)
            else:
                E = elig[r]
                gt = ((lo[r] > hi_t[:, None]) & E).astype(np.float32) @ w32
                lt = ((hi[r] < lo_t[:, None]) & E).astype(np.float32) @ w32
            eq = w[j] if not nf else np.where(f_t >= 0, F[r, np.maximum(f_t, 0)], w[j])
            amb = tot[r] - gt - lt - eq
            out['gt'].append(gt); out['eq'].append(eq); out['amb'].append(amb)
            if f32:
                t = sc[r, j][:, None]
                E = elig[r]
                out['f32'].append(np.stack([((sc[r] > t) & E).astype(np.float32) @ w32, ((sc[r] == t) & E).astype(np.float32) @ w32], 1))
        out['miss'].append(miss)
    res = {k: np.concatenate(out[k]).astype(np.int64) for k in ('gt', 'eq', 'amb')}
    res['miss'] = np.concatenate(out['miss'])
    for k in ('gt', 'eq', 'amb'):
        res[k][res['miss']] = 0
    res['offsets'] = np.concatenate([[0], np.cumsum(out['lens'])]).astype(np.int64)
    res['rows'] = out['rows']
    assert (res['amb'] >= 0).all() and (res['eq'][~res['miss']] >= 1).all()
    if f32:
        c = np.concatenate(out['f32']).astype(np.int64)
        c[res['miss']] = -1
        res['f32'] = c
    return res


def rest_metrics(r, offsets, cuts, ap=None):
    """per cut-off the sums over the events of HitRate, Precision, Recall, MRR, NDCG and MAP (event_metrics, vectorised) of the
    pair ranks r (inf: a miss); offsets: each event's pairs.  MAP's term of pair k is |{i: a_i <= q_k}| / c_k over the pairs
    with c_k <= N, ap = (a, q, c); by default a = q = c = r"""
    r = np.asarray(r, np.float64)
    a, q, c = (r, r, r) if ap is None else ap
    n_ev = len(offsets) - 1
    lens = np.diff(offsets)
    ev = np.repeat(np.arange(n_ev), lens)
    fin = np.concatenate([x[np.isfinite(x)] for x in (a, q, c)] + [[0.0]])
    S = 4.0 * (fin.max() + 2.0)                       # events apart on one sorted axis
    keys = np.sort(ev * S + a)
    start = np.searchsorted(keys, ev * S - 0.5, side='left')
    below = np.searchsorted(keys, ev * S + q, side='right') - start
    idcg = np.concatenate([[0.0], np.cumsum(1.0 / np.log2(np.arange(2, int(lens.max()) + 2)))])
    first = np.minimum.reduceat(r, offsets[:-1])
    out = np.zeros((6, len(cuts)))
    for j, N in enumerate(cuts):
        hit = r <= N
        hits = np.bincount(ev, weights=hit, minlength=n_ev)
        mm = np.minimum(lens, N)
        with np.errstate(divide='ignore', invalid='ignore'):
            dcg = np.bincount(ev, weights=np.where(hit, 1.0 / np.log2(r + 1.0), 0.0), minlength=n_ev)
            apk = np.bincount(ev, weights=np.where(c <= N, below / c, 0.0), minlength=n_ev)
            mrr = np.where(first <= N, 1.0 / first, 0.0)
        out[:, j] = [(hits > 0).sum(), hits.sum() / N, (hits / lens).sum(), mrr.sum(), (dcg / idcg[mm]).sum(), (apk / mm).sum()]
    return out


def metric_bounds(lo, hi, offsets, cuts):
    """(best, worst): the six metric sums per cut-off at the lower and at the upper end of every pair's rank interval (misses:
    inf at both).  Every metric but MAP is non-increasing in each rank.  MAP is not where ranks tie ({2, 3} -> {3, 3} raises
    AP from 7/6 to 4/3), so its bounds take each term's count and divisor from opposite ends: |{i: lo_i <= hi_k}| / lo_k over
    lo_k <= N, and |{i: hi_i <= lo_k}| / hi_k over hi_k <= N; both are AP itself when every interval is a point"""
    best = rest_metrics(lo, offsets, cuts, ap=(lo, hi, lo))
    worst = rest_metrics(hi, offsets, cuts, ap=(hi, lo, hi))
    return best, worst


def _bracket_ranks(br, mode):
    lo, hi = _rank_interval(br['gt'], br['eq'], br['amb'], mode)
    lo, hi = lo.astype(np.float64), hi.astype(np.float64)
    lo[br['miss']] = np.inf
    hi[br['miss']] = np.inf
    return lo, hi


def assert_in_bracket(c, br, tag):
    """(#greater, #equal) of every pair inside the bracket; misses (-1, -1) exactly where the host has them"""
    miss = br['miss']
    np.testing.assert_array_equal(c[:, 0] < 0, miss, err_msg=tag + 'miss pattern')
    assert (c[miss] == -1).all(), tag + 'misses must count (-1, -1)'
    g, e = c[~miss, 0], c[~miss, 1]
    s, q, a = br['gt'][~miss], br['eq'][~miss], br['amb'][~miss]
    for what, dev, lo in (('#greater', g, s), ('#equal', e, q), ('#greater + #equal', g + e, s + q)):
        bad = np.flatnonzero((dev < lo) | (dev > lo + a))
        assert bad.size == 0, tag + '%s outside the float64 bracket at pairs %s: device %s, sure %s + ambiguous %s' % (
            what, np.flatnonzero(~miss)[bad[:8]], dev[bad[:8]], lo[bad[:8]], a[bad[:8]])
    assert (e >= 1).all(), tag + 'a relevant item does not tie itself'


def assert_sums_in_bounds(sums, br, cuts, mode, tag, gap_max=0.01):
    """the device's six metric sums between the float64 bound sums, which differ by less than gap_max of their value; exactly
    (rtol 1e-12) the bound where every pair is decided.  Returns the largest relative gap"""
    lo, hi = _bracket_ranks(br, mode)
    best, worst = metric_bounds(lo, hi, br['offsets'], cuts)
    tol = 1e-12 * np.maximum(np.abs(best), 1.0)
    names = ('HitRate', 'Precision', 'Recall', 'MRR', 'NDCG', 'MAP')
    for i, nm in enumerate(names):
        bad = np.flatnonzero((sums[i] < worst[i] - tol[i]) | (sums[i] > best[i] + tol[i]))
        assert bad.size == 0, tag + '%s sums outside the float64 bounds at cut-offs %s: device %s, bounds %s .. %s' % (
            nm, np.asarray(cuts)[bad], sums[i][bad], worst[i][bad], best[i][bad])
    gap = (best - worst) / np.maximum(best, 1e-300)
    assert gap.max() < gap_max, tag + 'the bound sums differ by %.3g of their value (at most %g): the bracket has no teeth' % (gap.max(), gap_max)
    if not br['amb'][~br['miss']].any():
        np.testing.assert_allclose(sums, best, rtol=1e-12, atol=0, err_msg=tag + 'every pair decided')
    return float(gap.max())


def _units(br, cfg_tc, I, lanes):
    """launches the wgmma tiles add to an eval_rest call over the fp32 tiles' (plain schedules: a unit is a mini-batch): +1 per
    unit whose next-item ranking takes them (k_tc_split + k_eval_tc for k_eval_score), +1 per rest pass (k_tc_split + k_rest_tc
    + the gather, for k_rest_score + the gather); and whether a unit ranked pass 0 on wgmma and a later pass on fp32"""
    def tc(n):
        return cfg_tc == 2 or (cfg_tc == 0 and n >= 64 and I >= 2048)
    if not tc(lanes) and cfg_tc == 0:
        return 0, False
    extra, mixed = 0, False
    for lens in br['rows']:
        passes = [int((lens > k * 32).sum()) for k in range((int(lens.max()) + 31) // 32)]
        extra += int(tc(len(lens))) + sum(int(tc(n)) for n in passes)
        mixed |= tc(passes[0]) and any(not tc(n) for n in passes[1:])
    return extra, mixed


@pytest.mark.parametrize('seen_on', [False, True])
@pytest.mark.parametrize('case', list(CASES))
def test_rest_counts_and_sums_within_float64(case, seen_on):
    """every pair's (#greater, #equal) inside the float64 bracket on the fp32 tiles, the wgmma tiles and the automatic choice,
    equal across them wherever the bracket decides, the fp32 counts bitwise the workaround on a sample of events, and the six
    metric sums of modes 0 / 1 / 2 inside the float64 bound sums"""
    n_items, mk, lanes = CASES[case][:3]
    hist = CASES[case][-1]
    m, items, off, sched = _case(case)
    br = rest_bracket(m, mk, n_items, sched, items, off, seen_on=seen_on)
    lens = np.diff(br['offsets'])
    cuts = [1, 20, int(lens.max()) + 1]
    tag0 = '%s seen=%s: ' % (case, seen_on)
    assert (lens > 32).sum() >= 8 and (lens > 64).sum() >= 2, tag0 + 'too few rows of several passes'
    assert br['miss'].any() == seen_on
    ranked = ~br['miss']
    decided = ranked & (br['amb'] == 0)
    assert decided.sum() > 0.5 * ranked.sum(), tag0 + 'the bracket decides %d of %d pairs' % (decided.sum(), ranked.sum())
    counts, launches = {}, {}
    for tc in (False, True, None):
        eng = _engine(n_items, mk, m, lanes, tc)
        eng.set_eval_exclude_seen(seen_on)
        tag = tag0 + 'eval_tc=%s ' % tc
        got = []
        for mode in (0, 1, 2):
            n0 = eng.kernel_launches()
            sums, n, n_pairs, c, offsets = eng.eval_rest(sched, cuts, mode)
            launches[tc] = eng.kernel_launches() - n0                  # mode 0 made the item table's split
            np.testing.assert_array_equal(offsets, br['offsets'])
            assert n == len(lens) and n_pairs == len(c)
            got.append(c)
            assert_in_bracket(c, br, tag + 'mode %d: ' % mode)
            gap = assert_sums_in_bounds(sums, br, cuts, mode, tag + 'mode %d: ' % mode)
        assert all(np.array_equal(got[0], g) for g in got[1:]), tag + 'counts depend on the mode'
        counts[tc] = got[0]
        if tc is False and n_items < 10000:
            rs = np.random.RandomState(4)
            inp = sched.positions()[sched.counted()]
            long_ev = np.flatnonzero(lens > 32)
            pick = np.unique(np.concatenate([rs.choice(long_ev, min(30, len(long_ev)), replace=False), rs.choice(len(lens), 60, replace=False)]))
            want = _workaround(eng, items, off, inp[pick], 0)
            idx = np.concatenate([np.arange(br['offsets'][e], br['offsets'][e + 1]) for e in pick])
            np.testing.assert_array_equal(c[idx], want, err_msg=tag + 'fp32 counts vs the workaround')
        eng.close()
    for tc in (True, None):
        np.testing.assert_array_equal(counts[tc][decided], counts[False][decided], err_msg=tag0 + 'eval_tc=%s vs fp32 on decided pairs' % tc)
    assert launches[True] > launches[False]
    if not hist:
        for tc, cfg_tc in ((True, 2), (None, 0)):
            extra, mixed = _units(br, cfg_tc, n_items, lanes)
            assert launches[tc] - launches[False] == extra, tag0 + 'eval_tc=%s: %d launches over fp32, want %d' % (tc, launches[tc] - launches[False], extra)
            if cfg_tc == 0 and case.startswith('default'):
                assert mixed, tag0 + 'no unit takes pass 0 on wgmma and a later pass on fp32 under auto'
        many = max(int((r > 64).sum()) for r in br['rows'])
        if CASES[case][3][0] > 128:
            assert many > 128, tag0 + 'pass 2 ranks at most %d rows' % many
    if n_items > 128 * TC_N:
        import torch
        assert (n_items + TC_N - 1) // TC_N > torch.cuda.get_device_properties(0).multi_processor_count, tag0 + 'no CTA sweeps several item tiles'
    print('%s: %d events, %d pairs, %d misses, decided %d, ambiguous %d (%.2f per undecided pair), launches %s, largest sum gap %.3g' % (
        tag0, len(lens), len(c), br['miss'].sum(), decided.sum(), (ranked & ~decided).sum(),
        br['amb'][ranked & ~decided].mean() if (ranked & ~decided).any() else 0.0, launches, gap))


# ---------------- edges inside one row ----------------
EDGE_ITEMS = 2049           # the last item tile holds one live column (2048) and 255 padded ones
TWINS, LOW, LOW_TWIN, BELOW = (7, 1500), 5, 6, 8


def _edge_setup():
    """a linear model whose special items score exactly (zero Wy rows: the fp32 and the 3xTF32 score are the bias itself):
    twins 7 and 1500 at 50 (above every other item), item 5 at -50 with a non-relevant twin 6, item 8 at -60; item 2048
    (the padded last tile) at -0.25, below the padded columns' 0.  Sessions: A = [11, 0, 2048, 7, 1500, 5, 12, 13] (its first
    row ranks item 0, the padded tile's item, the twins and item 5, the row's lowest threshold); B, C, D of 33, 34 and 65
    distinct items (rows of exactly 32, 33 and 64 relevant items); E of 40 distinct items and then its own earlier items
    interleaved with new ones (seen items mixed into a long row); short sessions after them"""
    mk = _mk('linear', layers=[40])
    m = _model(EDGE_ITEMS, mk, seed=5)
    for it, b in ((TWINS[0], 50.0), (TWINS[1], 50.0), (LOW, -50.0), (LOW_TWIN, -50.0), (BELOW, -60.0), (EDGE_ITEMS - 1, -0.25)):
        m.Wy[it] = 0.0
        m.By[it] = b
    rs = np.random.RandomState(6)
    pool = np.setdiff1d(np.arange(EDGE_ITEMS), [0, 5, 6, 7, 8, 11, 12, 13, 1500, EDGE_ITEMS - 1])
    sess = [np.array([11, 0, EDGE_ITEMS - 1, TWINS[0], TWINS[1], LOW, 12, 13])]
    sess += [rs.choice(pool, n, replace=False) for n in (33, 34, 65)]
    e = rs.choice(pool, 60, replace=False)
    tail = np.empty(40, np.int64)
    tail[0::2], tail[1::2] = e[np.concatenate([[0, 1], 2 + rs.choice(38, 18, replace=False)])], e[40:]
    sess.append(np.concatenate([e[:40], tail]))
    si, so = _sessions(EDGE_ITEMS, 300, seed=7)
    items = np.concatenate(sess + [si]).astype(np.int64)
    off = np.concatenate([[0], np.cumsum([len(x) for x in sess]), sum(len(x) for x in sess) + so[1:]]).astype(np.int32)
    return mk, m, items, off


@pytest.mark.parametrize('seen_on', [False, True])
def test_rest_edges_inside_one_row(seen_on):
    """both tile kinds: every pair inside the float64 bracket and equal across the kinds where it decides; the twins count
    each other as a tie, (0, 2) exactly (the own-column correction of k_rest_tc must not swallow the twin); item 5, the row's
    lowest threshold, ties itself and its twin at exactly its score and counts nothing below it (the search skipped under
    tlow / lolast must not skip a score equal to it); item 2048 of the padded last tile is not outranked by the padded
    columns; rows of exactly 32, 33 and 64 relevant items (one pass, one pass + 1, two full passes); seen items as misses
    inside a row of more than 32 pairs"""
    mk, m, items, off = _edge_setup()
    sched = _lib.Schedule(items, off, None, 16, 0, mode=1 | _lib.SCHED_POSITIONS)
    br = rest_bracket(m, mk, EDGE_ITEMS, sched, items, off, seen_on=seen_on)
    inp = sched.positions()[sched.counted()]
    first = {s: int(np.flatnonzero(inp == off[s])[0]) for s in range(5)}      # the first event of sessions A .. E
    lens = np.diff(br['offsets'])
    assert [lens[first[s]] for s in (1, 2, 3)] == [32, 33, 64]
    e2 = int(np.flatnonzero(inp == off[4] + 1)[0])
    eE = slice(br['offsets'][e2], br['offsets'][e2 + 1])                       # E's second row: its first two inputs seen
    assert not seen_on or (br['miss'][eE].any() and (~br['miss'][eE]).sum() > 32)
    a0 = br['offsets'][first[0]]
    rel = items[1:8]                                               # session A's first row, first occurrence order
    at = {int(j): a0 + k for k, j in enumerate(rel)}
    out = {}
    for tc in (False, True):
        eng = _engine(EDGE_ITEMS, mk, m, 16, tc)
        eng.set_eval_exclude_seen(seen_on)
        n0 = eng.kernel_launches()
        c = eng.eval_rest(sched, [1, 20, 66], 0)[3]
        out[tc] = (c, eng.kernel_launches() - n0)
        tag = 'eval_tc=%s seen=%s: ' % (tc, seen_on)
        assert_in_bracket(c, br, tag)
        for t in TWINS:
            assert tuple(c[at[t]]) == (0, 2), tag + 'twin %d counts %s' % (t, c[at[t]])
        n_comp = EDGE_ITEMS - (1 if seen_on else 0)                # item 11, the input, leaves the competitors
        assert tuple(c[at[LOW]]) == (n_comp - 3, 2), tag + 'item %d counts %s' % (LOW, c[at[LOW]])
        eng.close()
    assert out[True][1] > out[False][1]                              # the wgmma passes (k_tc_split + k_rest_tc)
    decided = ~br['miss'] & (br['amb'] == 0)
    np.testing.assert_array_equal(out[True][0][decided], out[False][0][decided])


# ---------------- the Python surface ----------------
def _gru_holding(m, mk, n_items):
    import gru4rec
    import pandas as pd
    gru = gru4rec.GRU4Rec(**mk)
    gru.n_items = n_items
    gru.itemidmap = pd.Series(data=np.arange(n_items), index=np.array(['i%d' % i for i in range(n_items)]), name='ItemIdx')
    gru._host = {name: oracle_param(m, name) for name in gru._param_names()}
    gru.error_during_train = False
    gru.predict = None
    return gru


@pytest.mark.parametrize('subset', [False, True])
def test_evaluate_rest_within_float64(subset):
    """evaluation.evaluate_rest with default arguments (100 lanes, Recall@20 etc., standard mode, the automatic tile choice at
    2049 items) on a GRU4Rec holding the weights, and with items= (a candidate multiset: unlisted relevant items are misses):
    the pairs frame lists every event's relevant item ids in frame order, each rank inside its float64 rank interval (inf
    exactly for the misses), and every metric between the float64 bounds"""
    import contextlib
    import io
    import pandas as pd
    import evaluation
    case = 'default_I2049_L100_E100_elu'
    n_items, mk = CASES[case][:2]
    m, items, off, sched = _case(case)
    assert sched.batch_size == 100
    gru = _gru_holding(m, mk, n_items)
    ids = gru.itemidmap.index.values
    sid = np.repeat(np.arange(len(off) - 1), np.diff(off))
    test = pd.DataFrame({'SessionId': sid, 'ItemId': ids[items], 'Time': np.arange(len(items), dtype=np.float64)})
    kw, cand = {}, None
    if subset:
        rs = np.random.RandomState(8)
        cand = np.concatenate([rs.choice(n_items, 1400, replace=False), rs.choice(n_items, 100)])
        kw['items'] = ids[cand]
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_rest(gru, test.copy(), **kw)
    br = rest_bracket(m, mk, n_items, sched, items, off, cand=cand)
    assert br['miss'].any() == subset
    inp = sched.positions()[sched.counted()]
    order = np.argsort(inp, kind='stable')
    idx = np.concatenate([np.arange(br['offsets'][e], br['offsets'][e + 1]) for e in order])
    rel = np.concatenate([_relevant(items, off, int(inp[e]))[0] for e in order])
    p = res['pairs']
    assert res['n_events'] == len(inp) and res['n_pairs'] == len(p) == len(idx)
    np.testing.assert_array_equal(p['ItemId'].values, ids[rel])
    lo, hi = _bracket_ranks(br, 0)
    r = p['rank'].values
    np.testing.assert_array_equal(np.isinf(r), br['miss'][idx])
    fin = np.isfinite(r)
    bad = np.flatnonzero(fin & ((r < lo[idx]) | (r > hi[idx])))
    assert bad.size == 0, 'ranks outside the float64 intervals: %s not in %s .. %s' % (r[bad[:8]], lo[idx][bad[:8]], hi[idx][bad[:8]])
    best, worst = metric_bounds(lo, hi, br['offsets'], [20])
    n = res['n_events']
    for i, name in enumerate(('hitrate', 'precision', 'recall', 'mrr', 'ndcg', 'map')):
        got = res[name][0]
        assert worst[i, 0] / n - 1e-12 <= got <= best[i, 0] / n + 1e-12, '%s: %r not in %r .. %r' % (name, got, worst[i, 0] / n, best[i, 0] / n)
    assert ((best - worst) / best).max() < 0.01
