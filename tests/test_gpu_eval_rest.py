"""-m gpu: rest-of-session evaluation (Engine.eval_rest, csrc/g4r_rest.cuh, DESIGN §3m).  A lane's forward and tile scores do not
depend on the other lanes, so the pair-replication workaround -- one session per (event, relevant item j), made of the event's
prefix followed by j, ranked by eval_events -- is an exact oracle for every pair's (#greater, #equal):
- fp32 tiles, modes standard / conservative / median, with and without exclude_seen and a candidate list with duplicates, an
  elementwise and a softmax final activation, and a session with more relevant items than one pass holds: bitwise
- wgmma tiles (eval_tc = 2, shown by the launch count) and fp32 tiles: pair counts within the float64 bar of the weights' scores,
  and equal wherever the bar is unambiguous, rows of several passes included
- tiebreaking where the noise decides (a block of items scoring exactly 0, with and without a reordered candidate list):
  deterministic, every ranked item ties itself, the block's ties resolved
- |R| = 1 reductions against eval_schedule / eval_events; the device sums against a host recomputation from the counts
- history schedules (leave-one-out included), determinism, and eval_events unchanged after an eval_rest call
These run at one shape (16 lanes, one K chunk, full item tiles).  test_gpu_eval_rest_f64.py holds every pair's counts and the
metric sums to a float64 bracket at the shapes users run, on both tile kinds and the automatic choice."""
import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gpu_utils import push_weights
from test_host_eval_rest import event_metrics, rank_of

pytestmark = pytest.mark.gpu

LANES = 16


def _model(n_items, act, seed):
    loss = {'softmax': 'cross-entropy'}.get(act, 'bpr-max')
    mk = dict(batch_size=8, n_sample=0, loss=loss, final_act=act, layers=[24])
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    rs = np.random.RandomState(seed)
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    return mk, m


def _engine(n_items, mk, m, tc=False):
    eng = _lib.Engine(_lib.make_config(n_items, mk, sample_store=0, eval_lanes=LANES, step_mode=1, eval_tc=tc))
    push_weights(eng, m)
    return eng


def _data(n_items, n_sessions, seed, long_len=90):
    """sessions of 1 .. 12 events that repeat items, and one session of long_len events (more than 32 distinct later items)"""
    rs = np.random.RandomState(seed)
    items, off = [], [0]
    for s in range(n_sessions):
        n = long_len if s == 3 else rs.randint(1, 13)
        seq = [rs.randint(n_items)]
        while len(seq) < n:
            seq.append(seq[-1] if rs.rand() < 0.1 else rs.choice(seq) if rs.rand() < 0.3 else rs.randint(n_items))
        items += seq
        off.append(len(items))
    return np.array(items, np.int64), np.array(off, np.int32)


def _rest(eng, items, off, cuts, mode, n_hist=None):
    sched = _lib.Schedule(items, off, None, LANES, 0, mode=1 | _lib.SCHED_POSITIONS, n_history=n_hist)
    sums, n, n_pairs, counts, offsets = eng.eval_rest(sched, cuts, mode)
    pos = sched.positions()
    inp = pos[sched.counted()]
    return sums, n, n_pairs, counts, offsets, inp


def _relevant(items, off, p):
    """(the distinct items of rows p+1 .. end of p's session, first occurrence first; the session's first row)"""
    s = np.searchsorted(off, p, side='right') - 1
    rest = np.asarray(items[p + 1:off[s + 1]])
    first = np.sort(np.unique(rest, return_index=True)[1])
    return [int(v) for v in rest[first]], off[s]


def _workaround(eng, items, off, inp, mode):
    """counts of every (event, relevant item) from eval_events on one session per pair: the prefix, then the item"""
    data, woff = [], [0]
    for p in inp:
        rel, a = _relevant(items, off, p)
        for j in rel:
            data += list(items[a:p + 1]) + [j]
            woff.append(len(data))
    data, woff = np.array(data, np.int64), np.array(woff, np.int32)
    sched = _lib.Schedule(data, woff, None, LANES, 0, mode=1 | _lib.SCHED_POSITIONS)
    counts = eng.eval_events(sched, [20], mode)[3]
    tgt = sched.positions()[sched.counted()] + 1
    last = dict(zip(tgt.tolist(), range(len(tgt))))
    return counts[[last[e - 1] for e in woff[1:]]]


@pytest.mark.parametrize('act', ['softmax', 'elu-0.5'])
@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('seen', [False, True])
@pytest.mark.parametrize('subset', [False, True])
def test_fp32_counts_bitwise_the_workaround(act, mode, seen, subset):
    n_items = 700
    mk, m = _model(n_items, act, seed=1)
    eng = _engine(n_items, mk, m, tc=False)
    items, off = _data(n_items, 30, seed=2)
    cand = None
    if subset:
        rs = np.random.RandomState(5)
        cand = np.concatenate([rs.choice(n_items, 300, replace=False), rs.choice(n_items, 20)])   # duplicates
        eng.set_eval_items(cand)
    eng.set_eval_exclude_seen(seen)
    sums, n, n_pairs, counts, offsets, inp = _rest(eng, items, off, [5, 20], mode)
    assert n == len(inp) and n_pairs == offsets[-1] == len(counts)
    assert np.diff(offsets).max() > 32                                  # a row takes more than one pass
    want = _workaround(eng, items, off, inp, mode)
    miss = counts[:, 0] < 0
    k = 0
    for e, p in enumerate(inp):
        rel, a = _relevant(items, off, p)
        for j in rel:
            is_miss = (seen and j in set(items[a:p + 1].tolist())) or (subset and j not in set(cand.tolist()))
            assert miss[k] == is_miss, (e, j)
            k += 1
    assert miss.any() == (seen or subset)
    np.testing.assert_array_equal(counts[~miss], want[~miss])


def _float64_bar(m, items, off, seen_on, inp_len):
    """per (event, relevant item) in eval_rest's order (plain schedule): competitors surely above the item's float64 score and
    competitors within the tolerance of it (the item itself included), over the eligible items"""
    sched = _lib.Schedule(items, off, None, LANES, 0, mode=1 | _lib.SCHED_POSITIONS)
    e, P = sched.export(), sched.positions()
    H = [np.zeros((LANES, L), dtype=np.float32) for L in m.layers]
    sure, amb, seen = [], [], {}
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        slots, zero = e['slots'][s, :M].astype(np.int64), (e['F'][s, :M] & 2) != 0
        m.predict_step(e['X'][s, :M].astype(np.int64), H, slots=slots, zero=zero)
        y = H[-1][slots].astype(np.float64)
        sc = y @ m.Wy.astype(np.float64).T + m.By.reshape(-1).astype(np.float64)
        for b in range(M):
            if zero[b] or slots[b] not in seen:
                seen[slots[b]] = set()
            seen[slots[b]].add(int(e['X'][s, b]))
            row = np.delete(sc[b], sorted(seen[slots[b]])) if seen_on else sc[b]
            for j in _relevant(items, off, int(P[s, b]))[0]:
                t = sc[b, j]
                tol = 1e-5 * (abs(t) + 1.0)
                sure.append((row > t + tol).sum()); amb.append((np.abs(row - t) <= tol).sum())
    assert len(sure) == inp_len
    return np.array(sure), np.array(amb)


@pytest.mark.parametrize('act', ['linear', 'softmax'])
@pytest.mark.parametrize('seen_on', [False, True])
def test_wgmma_and_fp32_counts_within_float64_bar(act, seen_on):
    """eval_tc = 2 ranks the pairs on the wgmma tiles (k_tc_split + k_rest_tc: more launches than the fp32 passes); the pair counts
    of both tile kinds lie within the float64 bar of the trained weights' scores, and are equal wherever the bar is unambiguous,
    rows of more than one pass included"""
    n_items = 4096
    mk, m = _model(n_items, act, seed=12)
    items, off = _data(n_items, 60, seed=13)
    out = {}
    for tc in (False, True):
        eng = _engine(n_items, mk, m, tc=tc)
        eng.set_eval_exclude_seen(seen_on)
        _rest(eng, items, off, [20], 0)                                  # the item table's split, once
        n0 = eng.kernel_launches()
        out[tc] = _rest(eng, items, off, [20], 0) + (eng.kernel_launches() - n0,)
    cf, ct = out[False][3], out[True][3]
    offsets = out[False][4]
    assert np.diff(offsets).max() > 32
    assert out[True][-1] > out[False][-1]
    sure, amb = _float64_bar(m, items, off, seen_on, len(cf))
    miss = cf[:, 0] < 0
    np.testing.assert_array_equal(miss, ct[:, 0] < 0)
    assert miss.any() == seen_on
    for c in (cf, ct):
        g = c[~miss, 0]
        assert np.all(g >= sure[~miss]) and np.all(g <= sure[~miss] + amb[~miss])
        assert np.all(c[~miss, 1] >= 1)                                  # the item ties itself
    clear = ~miss & (amb == 1)
    assert clear.mean() > 0.5
    np.testing.assert_array_equal(ct[clear], cf[clear])
    long_rows = np.repeat(np.diff(offsets) > 32, np.diff(offsets))
    assert (clear & long_rows).any()


@pytest.mark.parametrize('subset', [False, True])
def test_tiebreaking_resolves_exact_ties(subset):
    """a block of items with all-zero rows and bias scores exactly 0: standard ranking ties them, tiebreaking's noise (keyed by the
    competitor's column) separates them.  A relevant item's threshold carries its own column's noise, so every ranked pair ties
    at least itself; deterministic"""
    n_items, G = 600, 60
    mk, m = _model(n_items, 'linear', seed=14)
    m.Wy[:G] = 0.0
    m.By[:G] = 0.0
    rs = np.random.RandomState(15)
    items, off = [], [0]
    for s in range(40):
        seq = list(rs.choice(G, rs.randint(2, 10))) + list(rs.randint(n_items, size=rs.randint(0, 4)))
        rs.shuffle(seq)
        items += seq
        off.append(len(items))
    items, off = np.array(items, np.int64), np.array(off, np.int32)
    eng = _engine(n_items, mk, m, tc=False)
    if subset:
        eng.set_eval_items(np.concatenate([np.arange(n_items)[::-1], np.arange(G)]))   # reordered, the zero block twice
    std = _rest(eng, items, off, [20], 0)
    a = _rest(eng, items, off, [20], 3)
    b = _rest(eng, items, off, [20], 3)
    assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[3], b[3])
    rel = np.concatenate([_relevant(items, off, int(p))[0] for p in std[5]])
    zero = rel < G
    cs, ct = std[3], a[3]
    assert zero.sum() > 100
    dup = 2 if subset else 1
    np.testing.assert_array_equal(cs[zero, 1], G * dup)                 # standard: the whole block ties
    assert np.all(ct[:, 1] >= 1)                                         # tiebreaking: every item ties itself ...
    assert (ct[zero, 1] == 1).mean() > 0.95                              # ... and almost nothing else
    assert np.all(ct[zero, 0] >= cs[zero, 0]) and np.all(ct[zero, 0] <= cs[zero, 0] + cs[zero, 1] - 1)


def test_reductions_and_host_sums():
    n_items = 500
    mk, m = _model(n_items, 'elu-0.5', seed=7)
    eng = _engine(n_items, mk, m, tc=False)
    rs = np.random.RandomState(8)
    items = np.concatenate([rs.choice(n_items, 2, replace=False) for _ in range(70)]).astype(np.int64)
    off = np.arange(0, len(items) + 1, 2, dtype=np.int32)
    cuts = [1, 5, 20]
    for mode in (0, 1, 2):
        sums, n, n_pairs, counts, offsets, inp = _rest(eng, items, off, cuts, mode)
        sched = _lib.Schedule(items, off, None, LANES, 0, mode=1 | _lib.SCHED_POSITIONS)
        rec, mrr, ne, ecounts = eng.eval_events(sched, cuts, mode)[:4]
        assert n == ne == n_pairs
        np.testing.assert_array_equal(counts, ecounts)
        r = rank_of(ecounts, mode)
        ndcg = [np.where(r <= c, 1.0 / np.log2(r + 1.0), 0.0).sum() for c in cuts]
        for got, want in ((sums[0], rec), (sums[2], rec), (sums[3], mrr), (sums[5], mrr), (sums[4], ndcg), (sums[1], np.array(rec) / cuts)):
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    items, off = _data(n_items, 40, seed=9)
    for mode in (0, 2):
        sums, n, n_pairs, counts, offsets, inp = _rest(eng, items, off, cuts, mode)
        r = rank_of(counts, mode)
        host = np.zeros((6, len(cuts)))
        for i in range(n):
            for j, c in enumerate(cuts):
                host[:, j] += event_metrics(r[offsets[i]:offsets[i + 1]], offsets[i + 1] - offsets[i], c)
        np.testing.assert_allclose(sums, host, rtol=1e-12, atol=0)


def test_history_determinism_and_next_item_unchanged():
    n_items = 800
    mk, m = _model(n_items, 'softmax', seed=10)
    eng = _engine(n_items, mk, m, tc=False)
    items, off = _data(n_items, 50, seed=11)
    lens = np.diff(off)
    sched = _lib.Schedule(items, off, None, LANES, 0, mode=1 | _lib.SCHED_POSITIONS)
    ev0 = eng.eval_events(sched, [5, 20], 0)
    for nh in (np.minimum(lens, np.arange(len(lens)) % 4).astype(np.int32), np.maximum(lens - 1, 0).astype(np.int32)):
        sums, n, n_pairs, counts, offsets, inp = _rest(eng, items, off, [5, 20], 0, n_hist=nh)
        hs = _lib.Schedule(items, off, None, LANES, 0, mode=1 | _lib.SCHED_POSITIONS, n_history=nh)
        ecounts = eng.eval_events(hs, [5, 20], 0)[3]
        np.testing.assert_array_equal(counts[offsets[:-1]], ecounts)     # every event's first pair is its next item
        if (nh == np.maximum(lens - 1, 0)).all():
            assert n_pairs == n                                           # leave-one-out: |R| = 1
        again = _rest(eng, items, off, [5, 20], 0, n_hist=nh)
        assert again[0].tobytes() == sums.tobytes() and np.array_equal(again[3], counts)
    ev1 = eng.eval_events(sched, [5, 20], 0)
    for a, b in zip(ev0[:4], ev1[:4]):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
