"""STAMP on the device (DESIGN §3v) against the float64 oracle (tests/stamp_oracle.py), at the shapes of tests/stamp_cases.py (whose
branch reach tests/test_host_stamp_shapes.py checks without a GPU).  One mini-batch's loss and every gradient element within
C 2^-24 times the sum of its terms' magnitudes, one C for every row, and each tensor's error norm against its norm; Adam step by
step against float64 at the shipped shape, each epoch's loss bitwise stamp_grads'; training over several epochs against float64
through the ABI and through STAMP.fit; two fits bitwise equal and an epoch whose last batch is short bitwise the same steps run
one call each; a batch past the scratch refused before any device write; every counted event's exported q against the float64
encoder across several evaluation chunks (plain, history=, windows) and bitwise independent of the call; the ranking bitwise
the NumPy float64 ranking of the exported q in all four modes x plain / items= / exclude_seen / history=; and a learning check
against Pop."""
import numpy as np
import pandas as pd
import pytest

import stamp_cases as sc
import stamp_oracle as so
from gru4rec_b200 import _lib, baselines, evaluation

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C = 8192                    # the gradient bound's constant, the same for every row
REL = 1e-4                  # a gradient tensor's error norm over its norm, the same for every row


def _csr(sessions):
    off = np.r_[0, np.cumsum([len(s) for s in sessions])].astype(np.int64)
    return off, np.concatenate(sessions).astype(np.int32)


def _device(case, bs, sessions, th):
    dev = _lib.Baselines('stamp', case['NI'], case['d'])
    dev.stamp_begin(case['max_len'], bs, *_csr(sessions), th)
    return dev


def _unpack(th, case):
    return so.unpack(th, case['NI'], case['d'])


def _check_grads(dev, case, p, batch, order, label):
    """the device's loss and every gradient element of one mini-batch against the float64 oracle; returns (loss, flat gradient)"""
    loss, g = dev.stamp_grads(order)
    l64, g64 = so.loss_and_grads(p, batch)
    _, mag = so.loss_and_grads(p, batch, mag=True)
    assert abs(loss - l64) <= 1e-5 * abs(l64), (label, loss, l64)
    worst, rel = {}, {}
    gmax = max(np.linalg.norm(v) for v in g64.values())
    for name, gd in _unpack(g, case).items():
        err = np.abs(gd - g64[name])
        ratio = err / (C * U * mag[name] + 1e-30)
        worst[name] = float(ratio.max())
        assert (ratio <= 1.0).all(), (label, name, worst[name], np.unravel_index(ratio.argmax(), ratio.shape))
        n64 = np.linalg.norm(g64[name])
        if n64 > 1e-9 * gmax:
            rel[name] = float(np.linalg.norm(err) / n64)
            assert rel[name] <= REL, (label, name, rel[name])
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print('STAMP grads %s (NI=%d d=%d max_len=%d batch=%d P=%d): loss %.6f vs %.6f, worst |err| / bound %.4f %s, worst tensor '
          '|err| / |g| %.2e (%s)' % (label, case['NI'], case['d'], case['max_len'], len(batch), sum(len(x) for x, _ in batch), loss, l64,
                                     top[0][1], [(k, round(v, 4)) for k, v in top], max(rel.values()), max(rel, key=rel.get)))
    return loss, g


@pytest.mark.parametrize('case', [pytest.param(c, id=c['id']) for c in sc.GRAD_CASES])
def test_one_batch_loss_and_gradients_against_float64(case):
    sessions, order, bs, rs = sc.grad_batch(case)
    th = sc.case_params(case, rs)
    dev = _device(case, bs, sessions, th)
    p = _unpack(th, case)
    smp = so.samples(sessions, case['max_len'])
    batch = [smp[k] for k in order]
    if case['scale'] != 1.0:
        Q = np.array([so.forward(p, x)[1] for x, _ in batch])
        spread = float(np.ptp(Q @ p['E'].T, axis=1).max())
        print('STAMP %s: largest logit spread in a row %.1f' % (case['id'], spread))
        assert spread >= 30.0
    _check_grads(dev, case, p, batch, order, case['id'])


def test_adam_steps_and_gradients_at_the_shipped_shape():
    case = next(c for c in sc.GRAD_CASES if c['id'] == 'shipped')
    sessions, order, bs, rs = sc.grad_batch(case)
    dev = _device(case, bs, sessions, sc.case_params(case, rs))
    smp = so.samples(sessions, case['max_len'])
    batch = [smp[k] for k in order]
    lr = float(np.float32(0.005))
    th = dev.stamp_export()
    m, v, mm, em, ev = (np.zeros(th.size) for _ in range(5))
    worst = 0.0
    for t in range(1, 9):
        lg, g = dev.stamp_grads(order)
        _check_grads(dev, case, _unpack(th, case), batch, order, 'shipped Adam step %d' % t)
        le, _ = dev.stamp_epoch(order, lr)
        assert le.shape == (1,) and le[0] == np.float32(lg), (t, le, lg)     # the epoch's step is stamp_grads' batch, bitwise
        th1 = dev.stamp_export()
        g64 = g.astype(np.float64)
        want, m, v = so.adam(th.astype(np.float64), g64, m, v, t, lr)
        mm = so.B1 * mm + (1.0 - so.B1) * np.abs(g64)
        em = so.B1 * em + 3 * U * mm
        ev = ev + 6 * U
        c1, c2 = 1.0 / (1.0 - so.B1 ** t), 1.0 / (1.0 - so.B2 ** t)
        bound = U * np.abs(want) + lr * c1 * (em + mm * (ev / 2 + 8 * U)) / (np.sqrt(c2 * v) + so.EPS) + 1e-30
        ratio = np.abs(th1 - want) / bound
        worst = max(worst, float(ratio.max()))
        assert (ratio <= 1.0).all(), (t, float(ratio.max()), int(ratio.argmax()), th1[ratio.argmax()], want[ratio.argmax()])
        th = th1
    print('STAMP Adam at the shipped shape, 8 steps: worst |err| / bound %.4f' % worst)


def _small():
    return dict(NI=300, d=16, max_len=8)


def _small_sessions(rs, n, NI):
    return [list(rs.randint(0, NI, rs.randint(2, 12))) for _ in range(n)]


def test_epochs_against_float64_training_through_the_abi_and_fit():
    case, bs, lr, std = _small(), 10, 0.004, 0.3
    rs = np.random.RandomState(21)
    sessions = _small_sessions(rs, 9, case['NI'])
    smp = so.samples(sessions, case['max_len'])
    th0, orders = so.plan(case['NI'], case['d'], std, len(smp), 5, 4)
    dev = _device(case, bs, sessions, th0)
    losses = np.concatenate([dev.stamp_epoch(o, lr)[0] for o in orders])
    th64, ol = so.train(th0, case['NI'], case['d'], smp, orders, bs, lr)
    assert (np.abs(losses - ol) <= 1e-4 * np.abs(ol)).all(), np.abs(losses - ol).max()
    drift = np.abs(dev.stamp_export() - th64).max()
    assert drift <= 0.05 * lr, drift
    # the same training through the class's fit, on the same data
    frame = pd.DataFrame([(s, 100 + it, float(t)) for s, seq in enumerate(sessions) for t, it in enumerate(seq)], columns=['SessionId', 'ItemId', 'Time'])
    m = baselines.STAMP(embedding=16, n_epochs=4, batch_size=bs, learning_rate=lr, init_std=std, max_len=8, seed=5)
    m.fit(frame)
    ids = m.itemidmap.index.values
    remap = [[int(np.flatnonzero(ids == 100 + it)[0]) for it in seq] for seq in sessions]
    th0m, ordm = so.plan(m.n_items, 16, std, len(smp), 5, 4)
    thm, olm = so.train(th0m, m.n_items, 16, so.samples(remap, 8), ordm, bs, lr)
    assert np.abs(np.concatenate([s[2] for s in m.fit_stats]) - olm).max() <= 1e-4 * np.abs(olm).max()
    assert np.abs(m.params - thm).max() <= 0.05 * lr


def test_an_epoch_whose_last_batch_is_short_is_the_same_steps_one_call_each():
    case, bs, lr = _small(), 10, 0.002
    rs = np.random.RandomState(22)
    sessions = _small_sessions(rs, 7, case['NI'])
    n = len(so.samples(sessions, case['max_len']))
    assert n % bs
    th0, orders = so.plan(case['NI'], case['d'], 0.05, n, 5, 1)
    a, b = _device(case, bs, sessions, th0), _device(case, bs, sessions, th0)
    la, _ = a.stamp_epoch(orders[0], lr)
    assert la.shape == (-(-n // bs),)
    lb = [b.stamp_epoch(orders[0][k:k + bs], lr)[0][0] for k in range(0, n, bs)]
    assert np.array_equal(la, np.array(lb, np.float32)) and np.array_equal(a.stamp_export(), b.stamp_export())


def test_a_batch_past_the_scratch_is_refused_before_any_device_write():
    case = dict(NI=400, d=8, max_len=50)
    rs = np.random.RandomState(4)
    sessions = [list(rs.randint(0, 400, 51))] + [list(rs.randint(0, 400, 2)) for _ in range(5)]
    th = so.init(400, 8, 0.05, rs)
    dev = _device(case, 2, sessions, th)                              # scratch for 50 + 49 positions
    with pytest.raises(ValueError, match='positions'):
        dev.stamp_epoch(np.array([49, 49, 1, 2]), 0.001)
    with pytest.raises(ValueError, match='positions'):
        dev.stamp_grads(np.array([49, 49]))
    assert np.array_equal(dev.stamp_export(), th)                     # nothing was stepped
    losses, _ = dev.stamp_epoch(np.array([49, 1, 2, 49]), 0.001)      # a sample repeated across batches fits
    assert np.isfinite(losses).all()


def _sessions(rs, n, NI, lo=1, hi=15):
    rows = []
    for s in range(n):
        for t in range(rs.randint(lo, hi)):
            rows.append((s, 5000 + rs.randint(NI), float(s * 1000 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


def test_two_fits_are_bitwise_equal():
    data = _sessions(np.random.RandomState(3), 400, 517)
    kw = dict(embedding=20, n_epochs=2, batch_size=37, max_len=6, seed=4)
    a, b = baselines.STAMP(**kw), baselines.STAMP(**kw)
    a.fit(data)
    b.fit(data)
    assert np.array_equal(a.params, b.params)
    assert all(np.array_equal(x[2], y[2]) for x, y in zip(a.fit_stats, b.fit_stats))


@pytest.fixture(scope='module')
def model():
    train = _sessions(np.random.RandomState(5), 300, 517)
    m = baselines.STAMP(embedding=24, n_epochs=1, batch_size=50, max_len=5, seed=6)
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


def _q_bound(p, prefixes, max_len):
    """(want, bound): q in float64 and 1e-4 times the magnitude of its rounding error (the oracle's magnitude pass)"""
    want, bound = [], []
    for x in prefixes:
        c, q = so.forward(p, list(x)[-max_len:])
        want.append(q)
        bound.append(1e-4 * so._magnitudes(p, c)['q'])
    return np.array(want), np.array(bound)


def _prefixes(items, off, nh):
    out = []
    for s in range(len(off) - 1):
        i0 = max(int(nh[s]) if nh is not None else 0, 1) - 1
        out += [items[off[s]:off[s] + i + 1] for i in range(i0, int(off[s + 1] - off[s]) - 1)]
    return out


def test_exported_q_against_the_float64_encoder(model):
    m, _, test, hist = model
    dev = m._device()
    p = m.params64()
    for items, off, nh in [(*_arrays(m, test), None), _with_history(m, test, hist)]:
        q = dev.stamp_encode(items, off, nh)
        want, bound = _q_bound(p, _prefixes(items, off, nh), m.max_len)
        assert q.shape == want.shape and q.shape[0] > 100
        assert np.diff(off).max() > m.max_len + 1                 # windows of the last max_len inputs are covered
        assert (np.abs(q - want) <= bound).all(), float((np.abs(q - want) / bound).max())


@pytest.fixture(scope='module', params=[pytest.param(c, id=c['id']) for c in sc.EVAL_CASES])
def encoded(request):
    """an evaluation case encoded in one stamp_encode call: (case, device, parameters, items, offsets, history, q, chunks)"""
    case = request.param
    items, off, nh = sc.eval_sessions(case)
    rs = np.random.RandomState(case['seed'])
    th = sc.case_params(dict(NI=case['NI'], d=case['d'], scale=4.0), rs)
    dev = _lib.Baselines('stamp', case['NI'], case['d'])
    dev.stamp_import(case['max_len'], th)
    q = dev.stamp_encode(items, off, nh)
    return case, dev, _unpack(th, case), items, off, nh, q, sc.eval_chunks(off, nh, case['max_len'], sc.constants()['ST_EVAL_POS'])


def test_encoded_q_across_chunks_against_the_float64_encoder(encoded):
    case, dev, p, items, off, nh, q, chunk = encoded
    assert chunk.max() >= 1 and q.shape == (len(chunk), case['d'])
    pre = _prefixes(items, off, nh)
    edges = np.flatnonzero(np.diff(chunk))
    rs = np.random.RandomState(0)
    pick = set(edges) | set(edges + 1) | {0, len(pre) - 1} | set(np.flatnonzero([len(x) > case['max_len'] for x in pre])[:20])
    pick = np.array(sorted(pick | set(rs.choice(len(pre), min(len(pre), 200), replace=False))))
    want, bound = _q_bound(p, [pre[e] for e in pick], case['max_len'])
    ratio = np.abs(q[pick] - want) / bound
    print('STAMP encode %s: %d chunks, %d events, %d compared, worst |err| / bound %.4f' % (case['id'], chunk.max() + 1, len(pre), len(pick), ratio.max()))
    assert (ratio <= 1.0).all(), (float(ratio.max()), int(pick[np.unravel_index(ratio.argmax(), ratio.shape)[0]]))


def test_encoded_q_is_bitwise_independent_of_the_call(encoded):
    # q of an event depends only on the last max_len inputs of its prefix: every kernel works per piece, per query or per
    # position, and the encoder's products never split k, so neither the chunk nor the other pieces change it
    case, dev, p, items, off, nh, q, chunk = encoded
    L = case['max_len']
    pre = _prefixes(items, off, nh)
    ev0 = np.r_[0, np.cumsum([max(0, int(off[s + 1] - off[s]) - max(int(nh[s]), 1)) for s in range(len(off) - 1)])]
    lens = np.diff(off)
    sess_chunks = [set(chunk[ev0[s]:ev0[s + 1]]) for s in range(len(off) - 1)]
    chosen = sorted(set([s for s in range(len(off) - 1) if len(sess_chunks[s]) > 1][:3]) | set(np.flatnonzero(lens > L + 1)[:2]))
    other = items[:7]
    n_win = 0
    for s in chosen:
        seq = items[off[s]:off[s + 1]]
        n = len(seq)
        alone = dev.stamp_encode(seq, [0, n])
        i0 = max(int(nh[s]), 1) - 1
        assert np.array_equal(q[ev0[s]:ev0[s + 1]], alone[i0:]), s
        for h in sorted({0, 1, 2, L, L + 1, n - 1} & set(range(n))):
            assert np.array_equal(dev.stamp_encode(seq, [0, n], [h]), alone[max(h, 1) - 1:]), (s, h)
        for k in sorted({0, 1, 5, L - 1} & set(range(n - 1))):
            assert np.array_equal(dev.stamp_encode(seq[:k + 2], [0, k + 2])[-1], alone[k]), (s, k)
        for i in sorted({L, L + 3, n - 2} & set(range(L, n - 1))):
            w = seq[i - L + 1:i + 2]
            behind = np.r_[other, w].astype(np.int32)
            assert np.array_equal(dev.stamp_encode(behind, [0, len(behind)], [len(behind) - 1])[0], alone[i]), (s, i)
            n_win += 1
    assert n_win > 0 and len(pre) == len(q)


@pytest.mark.parametrize('mode', [0, 1, 2, 3])
def test_ranking_is_bitwise_the_float64_ranking_of_the_exported_q(model, mode):
    m, train, test, hist = model
    dev = m._device()
    E = m.params64()['E']
    cand = m.itemidmap[train.ItemId.unique()[::3]].values.astype(np.int32)
    cand = np.r_[cand, cand[:5], np.unique(_arrays(m, test)[0])]
    name = ('standard', 'conservative', 'median', 'tiebreaking')[mode]
    plain = _arrays(m, test)
    wh = _with_history(m, test, hist)
    for (items, off), nh, cd, ex in [(plain, None, None, False), (plain, None, cand, False), (plain, None, None, True), (wh[:2], wh[2], None, False)]:
        q = dev.stamp_encode(items, off, nh)
        rec, mrr, n, cnt, ti, ts = dev.evaluate(items, off, nh, [1, 5, 20], mode, cd, ex, k=7)
        oc, oi, os_ = so.rank_events(E, q, items, off, nh, name, cd, ex, 7)
        assert np.array_equal(cnt, oc) and np.array_equal(ti, oi)
        assert np.array_equal(np.nan_to_num(ts, nan=7.5), np.nan_to_num(os_, nan=7.5))
        ok = cnt[:, 0] >= 0
        gt, eq = cnt[ok, 0].astype(np.float64), cnt[ok, 1].astype(np.float64)
        rank = gt + eq if mode == 1 else (gt + 0.5 * (eq - 1) + 1 if mode == 2 else gt + 1)
        for c, cut in enumerate([1, 5, 20]):
            assert rec[c] == (rank <= cut).sum() and abs(mrr[c] - np.where(rank <= cut, 1.0 / rank, 0.0).sum()) <= 1e-9 * max(1.0, mrr[c])


def test_evaluate_gpu_and_events_accept_a_stamp(model):
    m, train, test, hist = model
    r = evaluation.evaluate_events(m, test, cut_off=[5, 20], k=10, exclude_seen=True)
    rec, mrr = evaluation.evaluate_gpu(m, test, cut_off=[5, 20])
    assert 0.0 <= rec[1] <= 1.0
    evaluation.evaluate_gpu(m, test, cut_off=[20], history=hist, items=train.ItemId.unique()[:100])
    assert len(r['topk_items']) > 0


def _chains(rs, n, NI, length=8):
    """sessions whose next item is fixed by the current one: x' = (7 x + 3) mod NI from a random start (synth.py draws every item
    independently of its session, so on its sessions no model can beat Pop's ranking)"""
    rows = []
    for s in range(n):
        x = [int(rs.randint(NI))]
        while len(x) < length:
            x.append((x[-1] * 7 + 3) % NI)
        rows.extend((s, 100 + it, float(t)) for t, it in enumerate(x))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


def test_stamp_learns_the_next_item_better_than_pop(capsys):
    rs = np.random.RandomState(8)
    NI = 200
    train, test = _chains(rs, 3000, NI), _chains(rs, 300, NI)
    test = test.assign(SessionId=test.SessionId + 10 ** 6)
    m = baselines.STAMP(embedding=32, n_epochs=6, batch_size=100, learning_rate=0.005, max_len=10, seed=1)
    m.fit(train)
    pop = baselines.Pop(top_n=NI)
    pop.fit(train)
    r_st = evaluation.evaluate_gpu(m, test, cut_off=[20])[0][0]
    r_pop = evaluation.evaluate_gpu(pop, test, cut_off=[20])[0][0]
    with capsys.disabled():
        print('\nnext-item chain check: Recall@20 STAMP %.4f, Pop %.4f (%d items, 6 epochs)' % (r_st, r_pop, NI))
    assert r_st > r_pop + 0.5
