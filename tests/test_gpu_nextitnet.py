"""NextItNet on the device (DESIGN §3w) against the float64 oracle (tests/nextitnet_oracle.py), at the shapes of
tests/nextitnet_cases.py (whose branch reach tests/test_host_nextitnet_shapes.py checks without a GPU).  One mini-batch's loss and
every gradient element within C 2^-24 times the sum of its terms' magnitudes, one C for every row, and every tensor's error norm
within 10^-4 of its norm; Adam step by step against float64 Adam on the device's own parameters and gradients at the shipped
shape, each epoch's loss bitwise nextitnet_grads'; two fits bitwise equal and an epoch whose last batch is short bitwise the same
steps run one call each; a batch past the scratch refused before any device write; every counted event's exported q against the
float64 encoder across several evaluation chunks (plain, history=, windows) and bitwise independent of the call; the ranking
bitwise the NumPy float64 ranking of the exported q against W and bW in all four modes x plain / items= / exclude_seen / history=;
and a learning check against Pop on sessions whose next item is fixed by an item four steps back."""
import numpy as np
import pandas as pd
import pytest

import nextitnet_cases as nic
import nextitnet_oracle as nio
from gru4rec_b200 import _lib, baselines, evaluation

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C = 8192                    # the gradient bound's constant, the same for every row
REL = 1e-4                  # a gradient tensor's error norm over its norm, the same for every row


def _csr(pieces):
    off = np.r_[0, np.cumsum([len(p) for p in pieces])].astype(np.int64)
    return off, np.concatenate(pieces).astype(np.int32)


def _device(case, bs, pieces, th):
    dev = _lib.Baselines('nextitnet', case['NI'], case['d'])
    dev.nextitnet_begin(case['dil'], case['K'], case['max_len'], bs, *_csr(pieces), th)
    return dev


def _unpack(th, case):
    return nio.unpack(th, case['NI'], case['d'], case['dil'], case['K'])


def _check_grads(dev, case, p, batch, order, label):
    """the device's loss and every gradient element of one mini-batch against the float64 oracle; returns (loss, flat gradient)"""
    dil, K = case['dil'], case['K']
    loss, g = dev.nextitnet_grads(order)
    l64, g64 = nio.loss_and_grads(p, batch, dil, K)
    _, mag = nio.loss_and_grads(p, batch, dil, K, mag=True)
    assert abs(loss - l64) <= 1e-5 * abs(l64), (label, loss, l64)
    worst, rel = {}, {}
    gmax = max(np.linalg.norm(v) for v in g64.values())
    for name, gd in _unpack(g, case).items():
        err = np.abs(gd - g64[name])
        ratio = err / (C * U * mag[name] + 1e-30)
        worst[name] = float(ratio.max())
        assert (ratio <= 1.0).all(), (label, name, worst[name], np.unravel_index(ratio.argmax(), ratio.shape))
        # per tensor, the error's norm against the gradient's; a tensor whose gradient is zero but for rounding (a convolution
        # bias right before a layer norm, which removes any constant) is held by the element bound alone
        n64 = np.linalg.norm(g64[name])
        if n64 > 1e-6 * gmax:
            rel[name] = float(np.linalg.norm(err) / n64)
            assert rel[name] <= REL, (label, name, rel[name])
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print('NextItNet grads %s (NI=%d d=%d dil=%s K=%d max_len=%d batch=%d P=%d): loss %.6f vs %.6f, worst |err| / bound %.4f %s, '
          'worst tensor |err| / |g| %.2e (%s)' % (label, case['NI'], case['d'], case['dil'], K, case['max_len'], len(batch),
                                                 sum(len(b) - 1 for b in batch), loss, l64, top[0][1], [(k, round(v, 4)) for k, v in top],
                                                 max(rel.values()), max(rel, key=rel.get)))
    return loss, g


def _case_params(case, rs):
    """float32 flat parameters of a case: the init, or at a trained model's scale E and W x scale, the kernels x 2 and random gains
    and biases"""
    th = nio.init(case['NI'], case['d'], case['dil'], case['K'], rs)
    if case['scale'] != 1.0:
        p = _unpack(th, case)
        for k, v in p.items():
            if v.ndim == 2:
                p[k] = v * (case['scale'] if k in ('E', 'W') else 2.0)
            elif k[0] == 'g':
                p[k] = 1.0 + 0.3 * rs.randn(v.size)
            else:
                p[k] = 0.3 * rs.randn(v.size)
        th = nio.pack(p, case['dil'], case['K']).astype(np.float32)
    return th


@pytest.mark.parametrize('case', [pytest.param(c, id=c['id']) for c in nic.GRAD_CASES])
def test_one_batch_loss_and_gradients_against_float64(case):
    pieces, order, bs, rs = nic.grad_batch(case)
    th = _case_params(case, rs)
    dev = _device(case, bs, pieces, th)
    p = _unpack(th, case)
    batch = [pieces[k] for k in order]
    if case['scale'] != 1.0:
        _, Q, _ = nio.batch_forward(p, batch, case['dil'], case['K'])
        spread = float(np.ptp(Q @ p['W'].T + p['bW'], axis=1).max())
        print('NextItNet %s: largest logit spread in a row %.1f' % (case['id'], spread))
        assert spread >= 30.0
    _check_grads(dev, case, p, batch, order, case['id'])


def _adam_steps(dev, n_steps, order, lr, grad_check):
    """n_steps single-batch epochs.  Each step: θ_(t-1) exported, nextitnet_grads (checked against float64), nextitnet_epoch; θ_t
    per element against float64 Adam on the device's θ_(t-1) and gradient, with NARM's bound for k_nm_adam's float32 arithmetic
    (tests/test_gpu_narm.py)"""
    lr = float(np.float32(lr))
    th = dev.nextitnet_export()
    m, v, mm, em, ev = (np.zeros(th.size) for _ in range(5))
    worst = 0.0
    for t in range(1, n_steps + 1):
        lg, g = dev.nextitnet_grads(order)
        grad_check(t - 1, th)
        le, _ = dev.nextitnet_epoch(order, lr)
        assert le.shape == (1,) and le[0] == np.float32(lg), (t, le, lg)     # the epoch's step is nextitnet_grads' batch, bitwise
        th1 = dev.nextitnet_export()
        g64 = g.astype(np.float64)
        want, m, v = nio.adam(th.astype(np.float64), g64, m, v, t, lr)
        mm = nio.B1 * mm + (1.0 - nio.B1) * np.abs(g64)
        em = nio.B1 * em + 3 * U * mm
        ev = ev + 6 * U
        c1, c2 = 1.0 / (1.0 - nio.B1 ** t), 1.0 / (1.0 - nio.B2 ** t)
        bound = U * np.abs(want) + lr * c1 * (em + mm * (ev / 2 + 8 * U)) / (np.sqrt(c2 * v) + nio.EPS) + 1e-30
        ratio = np.abs(th1 - want) / bound
        worst = max(worst, float(ratio.max()))
        assert (ratio <= 1.0).all(), (t, float(ratio.max()), int(ratio.argmax()), th1[ratio.argmax()], want[ratio.argmax()])
        th = th1
    return worst


def test_adam_steps_and_gradients_at_the_shipped_shape():
    case = next(c for c in nic.GRAD_CASES if c['id'] == 'shipped')
    pieces, order, bs, rs = nic.grad_batch(case)
    dev = _device(case, bs, pieces, _case_params(case, rs))

    def grad_check(step, th):
        if step in (0, 7):
            _check_grads(dev, case, _unpack(th, case), [pieces[k] for k in order], order, 'shipped Adam step %d' % (step + 1))

    worst = _adam_steps(dev, 8, order, 0.001, grad_check)
    print('NextItNet Adam at the shipped shape, 8 steps: worst |err| / bound %.4f' % worst)


def _small():
    return dict(NI=300, d=16, dil=(1, 2, 4), K=3, max_len=8)


def test_an_epoch_whose_last_batch_is_short_is_the_same_steps_one_call_each():
    case, bs, lr = _small(), 10, 0.002
    rs = np.random.RandomState(22)
    pieces = nic._uniform(rs, 23, case['NI'], case['max_len'])
    th0, orders = nio.plan(case['NI'], case['d'], case['dil'], case['K'], len(pieces), 5, 1)
    a, b = _device(case, bs, pieces, th0), _device(case, bs, pieces, th0)
    la, _ = a.nextitnet_epoch(orders[0], lr)
    assert la.shape == (3,)
    lb = [b.nextitnet_epoch(orders[0][k:k + bs], lr)[0][0] for k in (0, 10, 20)]
    assert np.array_equal(la, np.array(lb, np.float32)) and np.array_equal(a.nextitnet_export(), b.nextitnet_export())
    shape = (case['NI'], case['d'], case['dil'], case['K'])
    th64, ol = nio.train(th0, shape, pieces, orders, bs, lr)
    assert (np.abs(la - ol) <= 1e-4 * np.abs(ol)).all(), np.abs(la - ol).max()
    # a convolution bias right before a layer norm has a zero gradient in exact arithmetic, so Adam turns rounding noise of either
    # sign into steps of up to lr: c1 and c2 move by at most lr a step, every other parameter stays within NARM's drift bound of
    # 0.05 lr
    diff = _unpack(np.abs(a.nextitnet_export() - th64), case)
    for k, v in diff.items():
        assert v.max() <= (3 * lr if k[:2] in ('c1', 'c2') else 0.05 * lr), (k, float(v.max()))


def test_a_batch_past_the_scratch_is_refused_before_any_device_write():
    case = dict(NI=400, d=8, dil=(1, 2), K=3, max_len=50)
    rs = np.random.RandomState(4)
    pieces = [list(rs.randint(0, 400, 51))] + [list(rs.randint(0, 400, 2)) for _ in range(5)]
    th = nio.init(400, 8, (1, 2), 3, rs)
    dev = _device(case, 2, pieces, th)                                # scratch for P_max = 50 + 1 positions
    with pytest.raises(ValueError, match='positions'):
        dev.nextitnet_epoch(np.array([0, 0, 1, 2]), 0.001)            # P_max + 49: the long piece twice
    with pytest.raises(ValueError, match='positions'):
        dev.nextitnet_grads(np.array([0, 0]))
    assert np.array_equal(dev.nextitnet_export(), th)                 # nothing was stepped
    pieces2 = [list(rs.randint(0, 400, 3)), list(rs.randint(0, 400, 2)), list(rs.randint(0, 400, 2))]
    dev2 = _device(case, 2, pieces2, th)                              # P_max = 2 + 1
    with pytest.raises(ValueError, match='positions'):
        dev2.nextitnet_grads(np.array([0, 0]))                        # P_max + 1
    loss, _ = dev2.nextitnet_grads(np.array([0, 1]))                  # P_max exactly
    assert np.isfinite(loss)
    losses, _ = dev.nextitnet_epoch(np.array([0, 1, 2, 0]), 0.001)    # a piece repeated across batches fits
    assert np.isfinite(losses).all()


def _sessions(rs, n, NI, lo=1, hi=15):
    rows = []
    for s in range(n):
        for t in range(rs.randint(lo, hi)):
            rows.append((s, 5000 + rs.randint(NI), float(s * 1000 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


def test_two_fits_are_bitwise_equal():
    data = _sessions(np.random.RandomState(3), 400, 517)
    kw = dict(embedding=20, dilations=(1, 2, 1), kernel_size=3, n_epochs=2, batch_size=37, max_len=6, seed=4)
    a, b = baselines.NextItNet(**kw), baselines.NextItNet(**kw)
    a.fit(data)
    b.fit(data)
    assert np.array_equal(a.params, b.params)
    assert all(np.array_equal(x[2], y[2]) for x, y in zip(a.fit_stats, b.fit_stats))


@pytest.fixture(scope='module')
def model():
    train = _sessions(np.random.RandomState(5), 300, 517)
    m = baselines.NextItNet(embedding=24, dilations=(1, 2), kernel_size=3, n_epochs=1, batch_size=50, max_len=5, seed=6)
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


def _q_bound(want, p, n_blocks):
    """q = h after the last block: each block adds a ReLU of a normalised vector, O(|g| + |n|), whose rounding is relative"""
    scale = sum(np.abs(p['g2_%d' % b]) + np.abs(p['n2_%d' % b]) for b in range(n_blocks))
    return 1e-4 * (scale[None, :] + np.abs(want) + np.abs(p['E']).max())


def test_exported_q_against_the_float64_encoder(model):
    m, _, test, hist = model
    dev = m._device()
    p = m.params64()
    for items, off, nh in [(*_arrays(m, test), None), _with_history(m, test, hist)]:
        q = dev.nextitnet_encode(items, off, nh)
        want = nio.encode_events(p, items, off, nh, m.dilations, m.kernel_size, m.max_len)
        assert q.shape == want.shape and q.shape[0] > 100
        assert np.diff(off).max() > m.max_len + 1                 # windows of the last max_len inputs are covered
        bound = _q_bound(want, p, len(m.dilations))
        assert (np.abs(q - want) <= bound).all(), float((np.abs(q - want) / bound).max())


def _prefixes(off, nh):
    """per counted event (evaluate's order) its session and the index of its last input"""
    out = []
    for s in range(len(off) - 1):
        i0 = max(int(nh[s]) if nh is not None else 0, 1) - 1
        out += [(s, i) for i in range(i0, int(off[s + 1] - off[s]) - 1)]
    return out


def _straddling(chunks):
    seen = {}
    for c, ch in enumerate(chunks):
        for s, _, _ in ch:
            seen.setdefault(s, set()).add(c)
    return sorted(s for s, cs in seen.items() if len(cs) > 1)


@pytest.fixture(scope='module', params=[pytest.param(c, id=c['id']) for c in nic.EVAL_CASES])
def encoded(request):
    """an evaluation case encoded in one nextitnet_encode call: (case, device, parameters, items, offsets, history, q, plan)"""
    case = request.param
    items, off, nh = nic.eval_sessions(case)
    th = nio.init(case['NI'], case['d'], case['dil'], case['K'], np.random.RandomState(case['seed']))
    dev = _lib.Baselines('nextitnet', case['NI'], case['d'])
    dev.nextitnet_import(case['dil'], case['K'], case['max_len'], th)
    q = dev.nextitnet_encode(items, off, nh)
    return case, dev, _unpack(th, case), items, off, nh, q, nic.eval_plan(off, nh, case['max_len'])


def test_encoded_q_across_chunks_against_the_float64_encoder(encoded):
    case, dev, p, items, off, nh, q, (chunks, where) = encoded
    assert len(chunks) >= 2 and q.shape == (len(where), case['d'])
    straddle = set(_straddling(chunks))
    assert straddle
    pre = _prefixes(off, nh)
    chunk_of = np.array([c for c, _ in where])
    edges = np.flatnonzero(np.diff(chunk_of))
    rs = np.random.RandomState(0)
    pick = set(e for e, (s, _) in enumerate(pre) if s in straddle) | set(edges) | set(edges + 1) | {0, len(pre) - 1}
    if case['max_len'] > 50:
        pick = set(sorted(pick)[::max(1, len(pick) // 60)])
    pick = np.array(sorted(pick | set(rs.choice(len(pre), min(len(pre), 300 if case['max_len'] <= 50 else 30), replace=False))))
    want = np.array([nio.encode(p, items[off[pre[e][0]]:off[pre[e][0]] + pre[e][1] + 1], case['dil'], case['K'], case['max_len']) for e in pick])
    bound = _q_bound(want, p, len(case['dil']))
    ratio = np.abs(q[pick] - want) / bound
    print('NextItNet encode %s: %d chunks, %d events, %d compared (sessions across chunks %s), worst |err| / bound %.4f'
          % (case['id'], len(chunks), len(pre), len(pick), sorted(straddle), ratio.max()))
    assert (ratio <= 1.0).all(), (float(ratio.max()), int(pick[np.unravel_index(ratio.argmax(), ratio.shape)[0]]))


def test_encoded_q_is_bitwise_independent_of_the_call(encoded):
    # q of an event depends only on the last max_len inputs of its prefix: every step is per position or per piece, and the
    # encoder's products never split k, so neither the chunk, the other pieces nor the piece's length change it
    case, dev, p, items, off, nh, q, (chunks, where) = encoded
    L = case['max_len']
    pre = _prefixes(off, nh)
    ev0 = np.searchsorted([s for s, _ in pre], np.arange(len(off)))
    lens = np.diff(off)
    chosen = sorted(set(_straddling(chunks)[:4]) | set(np.flatnonzero(lens > L + 1)[:2]) | {int(np.flatnonzero((lens >= 3) & (lens <= L))[0])})
    other = items[:7]
    n_win = 0
    for s in chosen:
        seq = items[off[s]:off[s + 1]]
        n = len(seq)
        alone = dev.nextitnet_encode(seq, [0, n])
        i0 = max(int(nh[s]), 1) - 1
        assert np.array_equal(q[ev0[s]:ev0[s] + n - 1 - i0], alone[i0:]), s
        for h in sorted({0, 1, 2, 5, L - 1, L, L + 1, L + 7, n - 1} & set(range(n))):
            assert np.array_equal(dev.nextitnet_encode(seq, [0, n], [h]), alone[max(h, 1) - 1:]), (s, h)
        for k in sorted({0, 1, 5, L - 2, L - 1} & set(range(n - 1))):
            assert np.array_equal(dev.nextitnet_encode(seq[:k + 2], [0, k + 2])[-1], alone[k]), (s, k)
        for i in sorted({L, L + 3, n - 2} & set(range(L, n - 1))):
            w = seq[i - L + 1:i + 2]
            behind = np.r_[other, w].astype(np.int32)
            assert np.array_equal(dev.nextitnet_encode(behind, [0, len(behind)], [len(behind) - 1])[0], alone[i]), (s, i)
            assert np.array_equal(dev.nextitnet_encode(w, [0, len(w)])[-1], alone[i]), (s, i)
            n_win += 1
    assert n_win > 0


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
def test_ranking_is_bitwise_the_float64_ranking_of_the_exported_q(model, mode):
    m, train, test, hist = model
    dev = m._device()
    p = m.params64()
    cand = m.itemidmap[train.ItemId.unique()[::3]].values.astype(np.int32)
    cand = np.r_[cand, cand[:5], np.unique(_arrays(m, test)[0])]
    name = ('standard', 'conservative', 'median', 'tiebreaking')[mode]
    plain = _arrays(m, test)
    wh = _with_history(m, test, hist)
    for (items, off), nh, cd, ex in [(plain, None, None, False), (plain, None, cand, False), (plain, None, None, True), (wh[:2], wh[2], None, False)]:
        q = dev.nextitnet_encode(items, off, nh)
        rec, mrr, n, cnt, ti, ts = dev.evaluate(items, off, nh, [1, 5, 20], mode, cd, ex, k=7)
        oc, oi, os_ = nio.rank_events(p['W'], p['bW'], q, items, off, nh, name, cd, ex, 7)
        assert np.array_equal(cnt, oc) and np.array_equal(ti, oi)
        assert np.array_equal(np.nan_to_num(ts, nan=7.5), np.nan_to_num(os_, nan=7.5))
        ok = cnt[:, 0] >= 0
        gt, eq = cnt[ok, 0].astype(np.float64), cnt[ok, 1].astype(np.float64)
        rank = gt + eq if mode == 1 else (gt + 0.5 * (eq - 1) + 1 if mode == 2 else gt + 1)
        for c, cut in enumerate([1, 5, 20]):
            assert rec[c] == (rank <= cut).sum() and abs(mrr[c] - np.where(rank <= cut, 1.0 / rank, 0.0).sum()) <= 1e-9 * max(1.0, mrr[c])


def test_evaluate_gpu_and_events_accept_a_nextitnet(model):
    m, train, test, hist = model
    assert np.abs(m.params64()['bW']).max() > 0                  # the fit moved the output bias, which the ranking must add
    r = evaluation.evaluate_events(m, test, cut_off=[5, 20], k=10, exclude_seen=True)
    rec, mrr = evaluation.evaluate_gpu(m, test, cut_off=[5, 20])
    assert 0.0 <= rec[1] <= 1.0
    evaluation.evaluate_gpu(m, test, cut_off=[20], history=hist, items=train.ItemId.unique()[:100])
    assert len(r['topk_items']) > 0


def _lagged(rs, n, NI, lag=4, length=10):
    rows = []
    for s in range(n):
        x = list(rs.randint(0, NI, lag))
        while len(x) < length:
            x.append((x[-lag] * 7 + 3) % NI)
        rows.extend((s, 100 + it, float(t)) for t, it in enumerate(x))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


def test_nextitnet_learns_an_item_four_steps_back_better_than_pop(capsys):
    rs = np.random.RandomState(8)
    NI = 200
    train, test = _lagged(rs, 4000, NI), _lagged(rs, 300, NI)
    test = test.assign(SessionId=test.SessionId + 10 ** 6)
    m = baselines.NextItNet(embedding=32, dilations=(1, 2), kernel_size=3, n_epochs=10, batch_size=64, learning_rate=0.005, max_len=10, seed=1)
    m.fit(train)
    pop = baselines.Pop(top_n=NI)
    pop.fit(train)
    hist = test.groupby('SessionId').head(4)                      # every later event is determined four steps back
    later = test.drop(hist.index)
    r_ni = evaluation.evaluate_gpu(m, later, cut_off=[20], history=hist)[0][0]
    r_pop = evaluation.evaluate_gpu(pop, later, cut_off=[20], history=hist)[0][0]
    with capsys.disabled():
        print('\nlagged-item check: Recall@20 NextItNet %.4f, Pop %.4f (%d items, 10 epochs)' % (r_ni, r_pop, NI))
    assert r_ni > r_pop + 0.6
