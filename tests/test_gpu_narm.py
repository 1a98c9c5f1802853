"""NARM on the device (DESIGN §3s) against the float64 oracle (tests/narm_oracle.py): one mini-batch's loss and every gradient per
element within a bound built from the magnitudes of the summed terms (dropout on and off, catalogues from about 1k to 37,483
items, pieces of 2 .. max_len events in one batch, batch sizes not a multiple of 32); one Adam step against float64 Adam on the
device's own gradients; a 20-step window and a small epoch within a stated drift; two fits bitwise equal; every counted event's
exported q against the float64 encoder (plain, history=, prefixes longer than max_len); the ranking bitwise the NumPy float64
ranking of the exported q in all four modes x plain / items= / exclude_seen / history=, with evaluate_gpu's sums recomputed from
the counts; and a learning check against Pop on sessions whose next item is fixed by an item three steps back."""
import numpy as np
import pandas as pd
import pytest

import narm_oracle as no
from gru4rec_b200 import _lib, baselines, evaluation

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _pieces(rs, n, NI, max_len):
    lens = np.r_[2, max_len, rs.randint(2, max_len + 1, n - 2)]
    return [list(rs.randint(0, NI, k)) for k in lens]


def _csr(pieces):
    off = np.r_[0, np.cumsum([len(p) for p in pieces])].astype(np.int64)
    return off, np.concatenate(pieces).astype(np.int32)


def _device(NI, d, H, max_len, bs, pieces, th):
    dev = _lib.Baselines('narm', NI, d)
    dev.narm_begin(H, max_len, bs, *_csr(pieces), th)
    return dev


@pytest.mark.parametrize('NI,d,H,nb,drop', [(1000, 16, 24, 37, (0.0, 0.0)), (1000, 16, 24, 37, (0.25, 0.5)), (2345, 50, 100, 45, (0.25, 0.5)),
                                            (37483, 50, 100, 33, (0.0, 0.0)), (37483, 50, 100, 33, (0.25, 0.5))])
def test_one_batch_loss_and_gradients_against_float64(NI, d, H, nb, drop):
    max_len = 12
    rs = np.random.RandomState(NI + nb)
    pieces = _pieces(rs, nb, NI, max_len)
    th = no.init(NI, d, H, rs)
    dev = _device(NI, d, H, max_len, nb, pieces, th)
    loss, g = dev.narm_grads(np.arange(nb), 77, 5, *drop)
    p = no.unpack(th, NI, d, H)
    l64, g64 = no.loss_and_grads(p, pieces, 77, 5, drop[0], drop[1], max_len)
    _, mag = no.loss_and_grads(p, pieces, 77, 5, drop[0], drop[1], max_len, mag=True)
    assert abs(loss - l64) <= 1e-5 * abs(l64), (loss, l64)
    worst = {}
    for name, gd in no.unpack(g, NI, d, H).items():
        bound = 1024 * U * mag[name] + 1e-30
        ratio = np.abs(gd - g64[name]) / bound
        worst[name] = float(ratio.max())
        assert (ratio <= 1.0).all(), (name, worst[name], np.unravel_index(ratio.argmax(), ratio.shape))
    print('NARM grads NI=%d d=%d H=%d batch=%d drop=%s: loss %.6f vs %.6f, worst |err| / bound per parameter %s'
          % (NI, d, H, nb, drop, loss, l64, {k: round(v, 4) for k, v in worst.items()}))


def test_one_adam_step_is_float64_adam_on_the_device_gradients():
    NI, d, H, nb, max_len = 1500, 32, 40, 29, 9
    rs = np.random.RandomState(1)
    pieces = _pieces(rs, nb, NI, max_len)
    th = no.init(NI, d, H, rs)
    dev = _device(NI, d, H, max_len, nb, pieces, th)
    _, g = dev.narm_grads(np.arange(nb), 3, 0, 0.25, 0.5)
    losses, _ = dev.narm_epoch(np.arange(nb), 3, 0.001, 0.25, 0.5)
    th1 = dev.narm_export()
    want, _, _ = no.adam(th.astype(np.float64), g.astype(np.float64), 0.0, 0.0, 1, 0.001)
    err = np.abs(th1 - want)
    assert (err <= 4 * U * np.abs(want) + 1e-6 * 0.001).all(), float(err.max())


def test_a_window_and_a_small_epoch_against_the_oracle():
    NI, d, H, max_len, bs = 300, 16, 24, 8, 10
    rs = np.random.RandomState(2)
    pieces = _pieces(rs, 200, NI, max_len)
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
