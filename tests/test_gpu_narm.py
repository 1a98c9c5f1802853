"""NARM on the device (DESIGN §3s) against the float64 oracle (tests/narm_oracle.py), at the shapes of tests/narm_cases.py (whose
branch reach tests/test_host_narm_shapes.py checks without a GPU).  One mini-batch's loss and every gradient per element within a
bound built from the magnitudes of the summed terms, at the shipped shape (37,483 items, d 50, H 100, max_len 50, 512 RSC15-like
pieces: backward products split 4 ways, dL/dq 64 ways, attention triangles past 256 pairs, an input-embedding run of ~300
positions) and at trained-model scale (a logit spread >= 30), 172,000 items, H 300 and 1024, max_len 512 with a 512-event piece,
d 130 and 1024, d = H = 1 with max_len 2, P and the catalogue at 64 and 65 / 128 and 129 with a piece repeated in the batch, and
the original small rows (dropout on and off throughout); Adam step by step against float64 Adam on the device's own parameters
and gradients for 200 steps (past c1 = 1.0 in float32) and for 8 steps at the shipped shape with every step's gradient against
float64, each epoch's loss bitwise narm_grads'; an epoch whose last batch is short; a 20-step window and a small epoch within a
stated drift; two fits bitwise equal; every counted event's exported q against the float64 encoder (plain, history=, prefixes
longer than max_len) and, over several evaluation chunks, at the shipped shape and at H 300 / max_len 512; q bitwise the same
for a session alone, inside a many-chunk call, as a prefix, as a window behind other items and under any history= count; the
ranking bitwise the NumPy float64 ranking of the exported q in all four modes x plain / items= / exclude_seen / history=, with
evaluate_gpu's sums recomputed from the counts; and a learning check against Pop on sessions whose next item is fixed by an
item three steps back."""
import numpy as np
import pandas as pd
import pytest

import narm_cases as nc
import narm_oracle as no
from gru4rec_b200 import _lib, baselines, evaluation

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _csr(pieces):
    off = np.r_[0, np.cumsum([len(p) for p in pieces])].astype(np.int64)
    return off, np.concatenate(pieces).astype(np.int32)


def _device(NI, d, H, max_len, bs, pieces, th):
    dev = _lib.Baselines('narm', NI, d)
    dev.narm_begin(H, max_len, bs, *_csr(pieces), th)
    return dev


def _check_grads(dev, p, batch, order, seed, step, drop, max_len, label):
    """the device's loss and every gradient element of one mini-batch against the float64 oracle; returns (loss, flat gradient)"""
    NI, d = p['E'].shape
    H = p['Wh'].shape[0]
    loss, g = dev.narm_grads(order, seed, step, *drop)
    l64, g64 = no.loss_and_grads(p, batch, seed, step, drop[0], drop[1], max_len)
    _, mag = no.loss_and_grads(p, batch, seed, step, drop[0], drop[1], max_len, mag=True)
    assert abs(loss - l64) <= 1e-5 * abs(l64), (label, loss, l64)
    worst = {}
    for name, gd in no.unpack(g, NI, d, H).items():
        bound = 1024 * U * mag[name] + 1e-30
        ratio = np.abs(gd - g64[name]) / bound
        worst[name] = float(ratio.max())
        assert (ratio <= 1.0).all(), (label, name, worst[name], np.unravel_index(ratio.argmax(), ratio.shape))
    print('NARM grads %s (NI=%d d=%d H=%d max_len=%d batch=%d P=%d drop=%s step %d): loss %.6f vs %.6f, worst |err| / bound %.4f %s'
          % (label, NI, d, H, max_len, len(batch), sum(len(b) - 1 for b in batch), drop, step, loss, l64, max(worst.values()),
             {k: round(v, 4) for k, v in worst.items()}))
    return loss, g


def _case_params(case, rs):
    """float32 flat parameters of a case: the init, or at a trained model's scale init x scale with a random Bh"""
    NI, d, H = case['NI'], case['d'], case['H']
    th = no.init(NI, d, H, rs)
    if case['scale'] != 1.0:
        p = {k: v * case['scale'] for k, v in no.unpack(th, NI, d, H).items()}
        p['Bh'] = rs.randn(3 * H) * 0.3
        th = no.pack(p).astype(np.float32)
    return th


@pytest.mark.parametrize('case', [pytest.param(c, id=c['id']) for c in nc.GRAD_CASES])
def test_one_batch_loss_and_gradients_against_float64(case):
    NI, d, H, max_len, drop = case['NI'], case['d'], case['H'], case['max_len'], case['drop']
    pieces, order, bs, rs = nc.grad_batch(case)
    th = _case_params(case, rs)
    dev = _device(NI, d, H, max_len, bs, pieces, th)
    p = no.unpack(th, NI, d, H)
    batch = [pieces[k] for k in order]
    if case['scale'] != 1.0:
        _, Q, _ = no.batch_forward(p, batch, 77, 5, drop[0], drop[1], max_len)
        spread = max(float(np.ptp(Q[r:r + 256] @ p['E'].T, axis=1).max()) for r in range(0, len(Q), 256))
        print('NARM %s: largest logit spread in a row %.1f' % (case['id'], spread))
        assert spread >= 30.0
    _check_grads(dev, p, batch, order, 77, 5, drop, max_len, case['id'])


def test_one_adam_step_is_float64_adam_on_the_device_gradients():
    NI, d, H, nb, max_len = 1500, 32, 40, 29, 9
    rs = np.random.RandomState(1)
    pieces = nc.uniform_pieces(rs, nb, NI, max_len)
    th = no.init(NI, d, H, rs)
    dev = _device(NI, d, H, max_len, nb, pieces, th)
    _, g = dev.narm_grads(np.arange(nb), 3, 0, 0.25, 0.5)
    losses, _ = dev.narm_epoch(np.arange(nb), 3, 0.001, 0.25, 0.5)
    th1 = dev.narm_export()
    want, _, _ = no.adam(th.astype(np.float64), g.astype(np.float64), 0.0, 0.0, 1, 0.001)
    err = np.abs(th1 - want)
    assert (err <= 4 * U * np.abs(want) + 1e-6 * 0.001).all(), float(err.max())


def _adam_steps(dev, n_steps, orders, seed, lr, drop, grad_check=None):
    """n_steps single-batch epochs (orders in turn).  Each step: θ_(t-1) exported, narm_grads at step t - 1, narm_epoch; θ_t per
    element against float64 Adam on the device's θ_(t-1) and gradient, m and v carried in float64 from the device gradients.
    The bound follows the float32 arithmetic of k_nm_adam: m's absolute error em_t = 0.9 em_(t-1) + 3u mm_t, with mm the EMA
    of |g| (m itself can cancel), from three roundings and the constants 0.9f / 0.1f; v's relative error grows by 6u a step
    (four roundings, 0.999f and 0.001f); the update adds 8u relative (c1 and c2 as floats, m c1, lr, v c2, the square root, + eps,
    the division) and the subtraction u |θ_t|."""
    lr = float(np.float32(lr))
    th = dev.narm_export()
    m, v, mm, em, ev = (np.zeros(th.size) for _ in range(5))
    worst = 0.0
    for t in range(1, n_steps + 1):
        order = orders[(t - 1) % len(orders)]
        lg, g = dev.narm_grads(order, seed, t - 1, *drop)
        if grad_check is not None:
            grad_check(order, t - 1, th)
        le, _ = dev.narm_epoch(order, seed, lr, *drop)
        assert le.shape == (1,) and le[0] == np.float32(lg), (t, le, lg)     # the epoch's step is narm_grads' batch, bitwise
        th1 = dev.narm_export()
        g64 = g.astype(np.float64)
        want, m, v = no.adam(th.astype(np.float64), g64, m, v, t, lr)
        mm = no.B1 * mm + (1.0 - no.B1) * np.abs(g64)
        em = no.B1 * em + 3 * U * mm
        ev = ev + 6 * U
        c1, c2 = 1.0 / (1.0 - no.B1 ** t), 1.0 / (1.0 - no.B2 ** t)
        bound = U * np.abs(want) + lr * c1 * (em + mm * (ev / 2 + 8 * U)) / (np.sqrt(c2 * v) + no.EPS) + 1e-30
        ratio = np.abs(th1 - want) / bound
        worst = max(worst, float(ratio.max()))
        assert (ratio <= 1.0).all(), (t, float(ratio.max()), int(ratio.argmax()), th1[ratio.argmax()], want[ratio.argmax()])
        th = th1
    return worst


def test_adam_step_by_step_for_200_steps_against_float64_adam():
    # 200 steps: c1 = 1 / (1 - 0.9^t) reaches 1.0 in float32 after about 160, c2 is still 1 / (1 - 0.999^200) = 5.5
    NI, d, H, nb, max_len, bs = 1500, 32, 40, 57, 9, 19
    rs = np.random.RandomState(21)
    pieces = nc.uniform_pieces(rs, nb, NI, max_len)
    dev = _device(NI, d, H, max_len, bs, pieces, no.init(NI, d, H, rs))
    worst = _adam_steps(dev, 200, [np.arange(k, k + bs) for k in range(0, nb, bs)], 3, 0.001, (0.25, 0.5))
    print('NARM Adam, 200 steps: worst |err| / bound %.4f' % worst)


def test_adam_steps_and_gradients_at_the_shipped_shape():
    case = next(c for c in nc.GRAD_CASES if c['id'] == 'shipped')
    NI, d, H, max_len, drop = case['NI'], case['d'], case['H'], case['max_len'], case['drop']
    pieces, order, bs, rs = nc.grad_batch(case)
    dev = _device(NI, d, H, max_len, bs, pieces, _case_params(case, rs))

    def grad_check(o, step, th):
        _check_grads(dev, no.unpack(th, NI, d, H), [pieces[k] for k in o], o, 5, step, drop, max_len, 'shipped Adam step %d' % (step + 1))

    worst = _adam_steps(dev, 8, [order], 5, 0.001, drop, grad_check)
    print('NARM Adam at the shipped shape, 8 steps: worst |err| / bound %.4f' % worst)


def test_an_epoch_whose_last_batch_is_short():
    NI, d, H, max_len, bs, lr = 300, 16, 24, 8, 10, 0.002
    rs = np.random.RandomState(22)
    pieces = nc.uniform_pieces(rs, 23, NI, max_len)
    th0, orders = no.plan(NI, d, H, len(pieces), 5, 1)
    a, b = _device(NI, d, H, max_len, bs, pieces, th0), _device(NI, d, H, max_len, bs, pieces, th0)
    la, _ = a.narm_epoch(orders[0], 5, lr, 0.25, 0.5)
    assert la.shape == (3,)
    # the same steps one ABI call each; before the third (3 pieces), its gradient against float64
    lb = [b.narm_epoch(orders[0][k:k + bs], 5, lr, 0.25, 0.5)[0][0] for k in (0, 10)]
    short = orders[0][20:]
    _check_grads(b, no.unpack(b.narm_export(), NI, d, H), [pieces[k] for k in short], short, 5, 2, (0.25, 0.5), max_len, 'short last batch')
    lb.append(b.narm_epoch(short, 5, lr, 0.25, 0.5)[0][0])
    assert np.array_equal(la, np.array(lb, np.float32)) and np.array_equal(a.narm_export(), b.narm_export())
    th64, ol = no.train(th0, (NI, d, H), pieces, orders, bs, lr, 5, 0.25, 0.5, max_len)
    assert (np.abs(la - ol) <= 1e-4 * np.abs(ol)).all(), np.abs(la - ol).max()
    assert np.abs(a.narm_export() - th64).max() <= 0.05 * lr      # the window test's drift bound


def test_a_window_and_a_small_epoch_against_the_oracle():
    NI, d, H, max_len, bs = 300, 16, 24, 8, 10
    rs = np.random.RandomState(2)
    pieces = nc.uniform_pieces(rs, 200, NI, max_len)
    th0, orders = no.plan(NI, d, H, len(pieces), 9, 2)
    dev = _device(NI, d, H, max_len, bs, pieces, th0)
    lr = 0.002
    dl = []
    for order in orders:
        dl.extend(dev.narm_epoch(order, 9, lr, 0.25, 0.5)[0])
    th_dev = dev.narm_export()
    th64, ol = no.train(th0, (NI, d, H), pieces, orders, bs, lr, 9, 0.25, 0.5, max_len)
    dl, ol = np.array(dl, np.float64), np.array(ol)
    print('NARM 40 steps (2 epochs of 20): device losses', np.round(dl, 5).tolist())
    print('                                 float64      ', np.round(ol, 5).tolist())
    # drift: each step's loss within 1e-4 relative; each parameter within 0.05 lr (an Adam step moves up to about lr, so a
    # gradient near 0 that takes the other sign in float32 moves a parameter by up to 2 lr), the typical one within 1e-3 lr
    assert (np.abs(dl - ol) <= 1e-4 * np.abs(ol)).all(), np.abs(dl - ol).max()
    diff = np.abs(th_dev - th64)
    print('NARM parameter drift after 40 steps: max %.3g, median %.3g (lr %g)' % (diff.max(), np.median(diff), lr))
    assert diff.max() <= 0.05 * lr and np.median(diff) <= 1e-3 * lr


def test_a_batch_past_the_scratch_is_refused_before_any_device_write():
    NI, d, H, max_len = 400, 8, 12, 50
    rs = np.random.RandomState(4)
    pieces = [list(rs.randint(0, NI, 50))] + [list(rs.randint(0, NI, 2)) for _ in range(5)]
    th = no.init(NI, d, H, rs)
    dev = _device(NI, d, H, max_len, 2, pieces, th)              # scratch for 49 + 1 positions
    with pytest.raises(ValueError, match='positions'):
        dev.narm_epoch(np.array([0, 0, 1, 2]), 1, 0.001, 0.0, 0.0)
    with pytest.raises(ValueError, match='positions'):
        dev.narm_grads(np.array([0, 0]), 1, 0, 0.0, 0.0)
    assert np.array_equal(dev.narm_export(), th)                # nothing was stepped
    losses, _ = dev.narm_epoch(np.array([0, 1, 2, 0]), 1, 0.001, 0.0, 0.0)   # a piece repeated across batches fits
    assert np.isfinite(losses).all()


def _sessions(rs, n, NI, lo=1, hi=15):
    rows = []
    for s in range(n):
        for t in range(rs.randint(lo, hi)):
            rows.append((s, 5000 + rs.randint(NI), float(s * 1000 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


def test_two_fits_are_bitwise_equal(capsys):
    data = _sessions(np.random.RandomState(3), 400, 517)
    a = baselines.NARM(embedding=20, hidden=30, n_epochs=2, batch_size=37, max_len=6, seed=4)
    b = baselines.NARM(embedding=20, hidden=30, n_epochs=2, batch_size=37, max_len=6, seed=4)
    a.fit(data)
    b.fit(data)
    assert np.array_equal(a.params, b.params)
    assert all(np.array_equal(x[2], y[2]) for x, y in zip(a.fit_stats, b.fit_stats))


@pytest.fixture(scope='module')
def model():
    train = _sessions(np.random.RandomState(5), 300, 517)
    m = baselines.NARM(embedding=24, hidden=32, n_epochs=1, batch_size=50, max_len=5, seed=6)
    m.fit(train)
    test = _sessions(np.random.RandomState(6), 60, 517, 1, 14)
    test = test[test.ItemId.isin(train.ItemId.unique())]
    test = test.assign(Time=test.Time + 1e9)
    hist = _sessions(np.random.RandomState(7), 60, 517, 0, 5)
    hist = hist[hist.ItemId.isin(train.ItemId.unique())]
    return m, train, test, hist


def _arrays(m, frame):
    frame = frame.sort_values(['SessionId', 'Time'], kind='stable')
    items = m.itemidmap[frame.ItemId.values].values.astype(np.int32)
    lens = frame.groupby('SessionId', sort=True).size().values
    return items, np.r_[0, np.cumsum(lens)].astype(np.int64)


def _with_history(m, test, hist):
    both = pd.concat([hist.assign(h=1), test.assign(h=0)]).sort_values(['SessionId', 'h', 'Time'], ascending=[True, False, True], kind='stable')
    items = m.itemidmap[both.ItemId.values].values.astype(np.int32)
    g = both.groupby('SessionId', sort=True)
    lens, nh = g.size().values, g.h.sum().values.astype(np.int32)
    return items, np.r_[0, np.cumsum(lens)].astype(np.int64), nh


def test_exported_q_against_the_float64_encoder(model):
    m, _, test, hist = model
    dev = m._device()
    p = m.params64()
    for items, off, nh in [(*_arrays(m, test), None), _with_history(m, test, hist)]:
        q = dev.narm_encode(items, off, nh)
        want = no.encode_events(p, items, off, nh, m.max_len)
        assert q.shape == want.shape and q.shape[0] > 100
        lens = np.diff(off)
        assert lens.max() > m.max_len + 1                         # windows of the last max_len inputs are covered
        mag = np.abs(p['B']).sum(axis=1)[None, :] * np.abs(want).max() + np.abs(want)
        assert (np.abs(q - want) <= 1e-4 * mag).all(), float((np.abs(q - want) / mag).max())


def _prefixes(off, nh):
    """per counted event (evaluate's order) its session and the index of its last input"""
    out = []
    for s in range(len(off) - 1):
        i0 = max(int(nh[s]) if nh is not None else 0, 1) - 1
        out += [(s, i) for i in range(i0, int(off[s + 1] - off[s]) - 1)]
    return out


def _straddling(chunks):
    """the sessions whose pieces lie in more than one chunk"""
    seen = {}
    for c, ch in enumerate(chunks):
        for s, _, _ in ch:
            seen.setdefault(s, set()).add(c)
    return sorted(s for s, cs in seen.items() if len(cs) > 1)


@pytest.fixture(scope='module', params=[pytest.param(c, id=c['id']) for c in nc.EVAL_CASES])
def encoded(request):
    """an evaluation case encoded in one narm_encode call: (case, device, parameters, items, offsets, history, q, plan)"""
    case = request.param
    NI, d, H = case['NI'], case['d'], case['H']
    items, off, nh = nc.eval_sessions(case)
    th = no.init(NI, d, H, np.random.RandomState(case['seed']))
    dev = _lib.Baselines('narm', NI, d)
    dev.narm_import(H, case['max_len'], th)
    q = dev.narm_encode(items, off, nh)
    return case, dev, no.unpack(th, NI, d, H), items, off, nh, q, nc.eval_plan(off, nh, case['max_len'])


def test_encoded_q_across_chunks_against_the_float64_encoder(encoded):
    case, dev, p, items, off, nh, q, (chunks, where) = encoded
    assert len(chunks) >= 2 and q.shape == (len(where), case['d'])
    # every event of the sessions whose pieces lie in two chunks, the first and last events of every chunk, a sample of the rest
    straddle = set(_straddling(chunks))
    assert straddle
    pre = _prefixes(off, nh)
    chunk_of = np.array([c for c, _ in where])
    edges = np.flatnonzero(np.diff(chunk_of))
    rs = np.random.RandomState(0)
    pick = set(e for e, (s, _) in enumerate(pre) if s in straddle) | set(edges) | set(edges + 1) | {0, len(pre) - 1}
    pick = np.array(sorted(pick | set(rs.choice(len(pre), min(len(pre), 400 if case['max_len'] <= 50 else 40), replace=False))))
    want = np.array([no.encode(p, items[off[pre[e][0]]:off[pre[e][0]] + pre[e][1] + 1], case['max_len']) for e in pick])
    got = q[pick]
    mag = np.abs(p['B']).sum(axis=1)[None, :] * np.abs(want).max() + np.abs(want)
    ratio = np.abs(got - want) / (1e-4 * mag)
    print('NARM encode %s: %d chunks, %d events, %d compared (sessions across chunks %s), worst |err| / bound %.4f'
          % (case['id'], len(chunks), len(pre), len(pick), sorted(straddle), ratio.max()))
    assert (ratio <= 1.0).all(), (float(ratio.max()), int(pick[np.unravel_index(ratio.argmax(), ratio.shape)[0]]))


def test_encoded_q_is_bitwise_independent_of_the_call(encoded):
    # q of an event depends only on the last max_len inputs of its prefix: the encoder's products never split k, and each piece
    # runs its own recurrence and attention, so neither the chunk, the other pieces nor the piece's length change it
    case, dev, p, items, off, nh, q, (chunks, where) = encoded
    L = case['max_len']
    pre = _prefixes(off, nh)
    ev0 = np.searchsorted([s for s, _ in pre], np.arange(len(off)))
    lens = np.diff(off)
    chosen = sorted(set(_straddling(chunks)) | set(np.flatnonzero(lens > L + 1)[:3]) | {int(np.flatnonzero((lens >= 3) & (lens <= L))[0])})
    other = items[:7]
    n_win = 0
    for s in chosen:
        seq = items[off[s]:off[s + 1]]
        n = len(seq)
        alone = dev.narm_encode(seq, [0, n])                    # the session alone, every event counted
        i0 = max(int(nh[s]), 1) - 1
        assert np.array_equal(q[ev0[s]:ev0[s] + n - 1 - i0], alone[i0:]), s
        for h in sorted({0, 1, 2, 5, L - 1, L, L + 1, L + 7, n - 1} & set(range(n))):
            assert np.array_equal(dev.narm_encode(seq, [0, n], [h]), alone[max(h, 1) - 1:]), (s, h)
        for k in sorted({0, 1, 5, L - 2, L - 1} & set(range(n - 1))):   # a prefix of k + 1 inputs, alone as the last event
            assert np.array_equal(dev.narm_encode(seq[:k + 2], [0, k + 2])[-1], alone[k]), (s, k)
        for i in sorted({L, L + 3, n - 2} & set(range(L, n - 1))):      # a window: behind other items, and as a session's start
            w = seq[i - L + 1:i + 2]
            behind = np.r_[other, w].astype(np.int32)
            assert np.array_equal(dev.narm_encode(behind, [0, len(behind)], [len(behind) - 1])[0], alone[i]), (s, i)
            assert np.array_equal(dev.narm_encode(w, [0, len(w)])[-1], alone[i]), (s, i)
            n_win += 1
    assert n_win > 0
    print('NARM encode %s: sessions %s bitwise alone, inside the call, by history count, as prefixes and as windows' % (case['id'], chosen))


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
def test_ranking_is_bitwise_the_float64_ranking_of_the_exported_q(model, mode):
    m, train, test, hist = model
    dev = m._device()
    E = m.params64()['E']
    cand = m.itemidmap[train.ItemId.unique()[::3]].values.astype(np.int32)
    cand = np.r_[cand, cand[:5], np.unique(_arrays(m, test)[0])]      # duplicates; every target a candidate (rank >= 1)
    name = ('standard', 'conservative', 'median', 'tiebreaking')[mode]
    plain = _arrays(m, test)
    for (items, off), nh, cd, ex in [(plain, None, None, False), (plain, None, cand, False), (plain, None, None, True),
                                      (_with_history(m, test, hist)[:2], _with_history(m, test, hist)[2], None, False)]:
        q = dev.narm_encode(items, off, nh)
        rec, mrr, n, cnt, ti, ts = dev.evaluate(items, off, nh, [1, 5, 20], mode, cd, ex, k=7)
        oc, oi, os_ = no.rank_events(E, q, items, off, nh, name, cd, ex, 7)
        assert np.array_equal(cnt, oc) and np.array_equal(ti, oi)
        assert np.array_equal(np.nan_to_num(ts, nan=7.5), np.nan_to_num(os_, nan=7.5))
        ok = cnt[:, 0] >= 0
        gt, eq = cnt[ok, 0].astype(np.float64), cnt[ok, 1].astype(np.float64)
        rank = gt + eq if mode == 1 else (gt + 0.5 * (eq - 1) + 1 if mode == 2 else gt + 1)
        for c, cut in enumerate([1, 5, 20]):
            assert rec[c] == (rank <= cut).sum() and abs(mrr[c] - np.where(rank <= cut, 1.0 / rank, 0.0).sum()) <= 1e-9 * max(1.0, mrr[c])


def test_evaluate_gpu_and_events_accept_a_narm(model):
    m, train, test, hist = model
    r = evaluation.evaluate_events(m, test, cut_off=[5, 20], k=10, exclude_seen=True)
    rec, mrr = evaluation.evaluate_gpu(m, test, cut_off=[5, 20])
    assert 0.0 <= rec[1] <= 1.0
    evaluation.evaluate_gpu(m, test, cut_off=[20], history=hist, items=train.ItemId.unique()[:100])
    assert len(r['topk_items']) > 0


def _lagged(rs, n, NI, lag=3, length=9):
    rows = []
    for s in range(n):
        x = list(rs.randint(0, NI, lag))
        while len(x) < length:
            x.append((x[-lag] * 7 + 3) % NI)
        rows.extend((s, 100 + it, float(t)) for t, it in enumerate(x))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


def test_narm_learns_an_item_three_steps_back_better_than_pop(capsys):
    rs = np.random.RandomState(8)
    NI = 200
    train, test = _lagged(rs, 4000, NI), _lagged(rs, 300, NI)
    test = test.assign(SessionId=test.SessionId + 10 ** 6)
    m = baselines.NARM(embedding=32, hidden=64, n_epochs=10, batch_size=64, learning_rate=0.005, dropout_emb=0.1, dropout_ct=0.1,
                       max_len=10, seed=1)
    m.fit(train)
    pop = baselines.Pop(top_n=NI)
    pop.fit(train)
    # every event past the third is determined three steps back; evaluate only those
    hist = test.groupby('SessionId').head(3)
    later = test.drop(hist.index)
    r_narm = evaluation.evaluate_gpu(m, later, cut_off=[20], history=hist)[0][0]
    r_pop = evaluation.evaluate_gpu(pop, later, cut_off=[20], history=hist)[0][0]
    with capsys.disabled():
        print('\nlagged-item check: Recall@20 NARM %.4f, Pop %.4f (%d items, 10 epochs)' % (r_narm, r_pop, NI))
    assert r_narm > r_pop + 0.3
