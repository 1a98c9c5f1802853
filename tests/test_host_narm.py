"""NARM (DESIGN §3s) without a GPU: the float64 oracle's backward against finite differences, the piece builder and the plan, the
package's host encoder and predict_next against the oracle, the class's fit, evaluation surface, pickles and run.py through a
CPU double of _lib.Baselines backed by the oracle, the refusals before any device work, and the ABI's exports."""
import os
import pickle
import sys

import numpy as np
import pandas as pd
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, 'oracle'), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import narm_oracle as no  # noqa: E402
from gru4rec_b200 import _lib, baselines, evaluation  # noqa: E402


def _params(n_items, d, H, seed=0, scale=3.0):
    rs = np.random.RandomState(seed)
    p = no.unpack(no.init(n_items, d, H, rs).astype(np.float64) * scale, n_items, d, H)
    p['Bh'] = rs.randn(3 * H) * 0.3
    return p


@pytest.mark.parametrize('drop', [(0.0, 0.0), (0.25, 0.5)])
def test_oracle_backward_matches_finite_differences(drop):
    NI, d, H = 7, 3, 4
    p = _params(NI, d, H)
    batch = [[1, 2, 3, 4], [5, 6], [0, 0, 2]]
    _, g = no.loss_and_grads(p, batch, 7, 3, drop[0], drop[1], 5)
    th, gf = no.pack(p), no.pack(g)
    for i in range(th.size):
        a, b = th.copy(), th.copy()
        a[i] += 1e-6
        b[i] -= 1e-6
        la = no.loss_and_grads(no.unpack(a, NI, d, H), batch, 7, 3, drop[0], drop[1], 5)[0]
        lb = no.loss_and_grads(no.unpack(b, NI, d, H), batch, 7, 3, drop[0], drop[1], 5)[0]
        fd = (la - lb) / 2e-6
        assert abs(fd - gf[i]) <= 1e-4 * abs(fd) + 1e-7, (i, fd, gf[i])


def test_magnitude_bound_dominates_the_gradient():
    NI, d, H = 9, 4, 5
    p = _params(NI, d, H, 1)
    batch = [[1, 2, 3, 4, 8], [5, 6], [0, 7, 2]]
    _, g = no.loss_and_grads(p, batch, 1, 0, 0.25, 0.5, 6)
    _, m = no.loss_and_grads(p, batch, 1, 0, 0.25, 0.5, 6, mag=True)
    assert (np.abs(no.pack(g)) <= no.pack(m) * (1 + 1e-12)).all()


@pytest.mark.parametrize('max_len', [2, 3, 5])
def test_every_pair_lands_in_exactly_one_piece(max_len):
    rs = np.random.RandomState(max_len)
    lens = [1, 2, max_len, max_len + 1, 2 * max_len + 3, 1, 7]
    sessions = [list(rs.randint(0, 20, n)) for n in lens]
    pieces = no.pieces(sessions, max_len)
    got = sorted((pc[t], pc[t + 1], k) for k, pc in enumerate(pieces) for t in range(len(pc) - 1))
    want_pairs = [(s[t], s[t + 1]) for s in sessions for t in range(len(s) - 1)]
    assert len(got) == len(want_pairs)
    assert sorted((a, b) for a, b, _ in got) == sorted(want_pairs)
    assert all(2 <= len(pc) <= max_len for pc in pieces)
    off = np.r_[0, np.cumsum(lens)]
    poff, pit = baselines.narm_pieces(off, np.concatenate(sessions), max_len)
    assert [list(pit[poff[k]:poff[k + 1]]) for k in range(len(poff) - 1)] == pieces


def test_plan_is_deterministic_and_the_package_draws_it():
    a = no.plan(11, 3, 4, 9, 5, 3)
    b = no.plan(11, 3, 4, 9, 5, 3)
    assert np.array_equal(a[0], b[0]) and all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))
    rs = np.random.RandomState(5)
    assert np.array_equal(baselines.narm_init(11, 3, 4, rs), a[0])
    assert np.array_equal(rs.permutation(9), a[1][0])
    assert not np.array_equal(no.plan(11, 3, 4, 9, 6, 1)[0], a[0])


def _model(NI=12, d=4, H=5, max_len=4, seed=3):
    m = baselines.NARM(embedding=d, hidden=H, max_len=max_len)
    m.n_items = NI
    m.itemidmap = pd.Series(data=np.arange(NI), index=np.arange(100, 100 + NI))
    m.params = no.pack(_params(NI, d, H, seed)).astype(np.float32)
    return m


def test_predict_next_equals_the_oracle_encoder():
    m = _model()
    p = no.unpack(m.params, m.n_items, m.embedding, m.hidden)
    ids = np.arange(100, 112)
    seq = [3, 5, 5, 0, 11, 2, 7]
    for t, x in enumerate(seq):
        got = m.predict_next('s', 100 + x, ids).values
        want = p['E'] @ no.encode(p, seq[:t + 1], m.max_len)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


class OracleNarm(object):
    """_lib.Baselines for kind 'narm' on the float64 oracle (parameters kept as float32, as the device keeps them)"""

    def __init__(self, kind, n_items, n_keep, device=0):
        assert kind == 'narm'
        self.n_items, self.n_keep = n_items, n_keep

    def narm_begin(self, hidden, max_len, batch_size, piece_offsets, items, params):
        self.H, self.L, self.bs = hidden, max_len, batch_size
        self.pieces = [list(items[piece_offsets[k]:piece_offsets[k + 1]]) for k in range(len(piece_offsets) - 1)]
        self.th = np.asarray(params, np.float32).copy()
        self.m = np.zeros(self.th.size)
        self.v = np.zeros(self.th.size)
        self.step = 0

    def narm_epoch(self, order, seed, lr, pe, pc):
        losses = []
        for b0 in range(0, len(order), self.bs):
            batch = [self.pieces[k] for k in order[b0:b0 + self.bs]]
            loss, g = no.loss_and_grads(no.unpack(self.th, self.n_items, self.n_keep, self.H), batch, seed, self.step, pe, pc, self.L)
            self.step += 1
            th, self.m, self.v = no.adam(self.th.astype(np.float64), no.pack(g), self.m, self.v, self.step, lr)
            self.th = th.astype(np.float32)
            losses.append(loss)
        return np.array(losses, np.float32), 0.0

    def narm_export(self):
        return self.th.copy()

    def narm_import(self, hidden, max_len, params):
        self.H, self.L, self.th = hidden, max_len, np.asarray(params, np.float32).copy()

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        p = no.unpack(self.th, self.n_items, self.n_keep, self.H)
        qs = no.encode_events(p, np.asarray(items), offsets, n_history, self.L).astype(np.float32)
        cnt, ti, ts = no.rank_events(p['E'], qs, items, offsets, n_history, ('standard', 'conservative', 'median', 'tiebreaking')[mode], cand,
                                     exclude_seen, k)
        rec, mrr = np.zeros(len(cut_off)), np.zeros(len(cut_off))
        for c, n in enumerate(cut_off):
            for gt, eq in cnt:
                if gt < 0:
                    continue
                r = (gt + eq) if mode == 1 else (gt + 0.5 * (eq - 1) + 1 if mode == 2 else gt + 1)
                if r <= n:
                    rec[c] += 1
                    mrr[c] += 1.0 / r
        return rec, mrr, len(cnt), cnt.astype(np.int32) if counts else None, ti, ts


@pytest.fixture
def double(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleNarm)


def _frame(n_sessions, n_items, seed, max_len=9):
    rs = np.random.RandomState(seed)
    rows = []
    for s in range(n_sessions):
        for t in range(rs.randint(1, max_len)):
            rows.append((s, 1000 + rs.randint(n_items), float(s * 100 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


@pytest.fixture
def fitted(double):
    train = _frame(40, 15, 0)
    m = baselines.NARM(embedding=4, hidden=5, n_epochs=2, batch_size=7, learning_rate=0.01, max_len=4, seed=1)
    m.fit(train)
    return m, train


def test_fit_prints_epochs_and_matches_the_oracle(double, capsys):
    train = _frame(40, 15, 0)
    m = baselines.NARM(embedding=4, hidden=5, n_epochs=2, batch_size=7, learning_rate=0.01, max_len=4, seed=1)
    capsys.readouterr()
    m.fit(train)
    lines = capsys.readouterr().out.split('\n')
    assert len(m.fit_stats) == 2 and all(np.isfinite(s[0]) for s in m.fit_stats)
    assert lines[:2] == ['%d %s' % (e, m.fit_stats[e][0]) for e in range(2)]
    assert all(s[0] == np.mean(s[2].astype(np.float64)) for s in m.fit_stats)
    poff, pit = m.pieces(train)
    pieces = [list(pit[poff[k]:poff[k + 1]]) for k in range(len(poff) - 1)]
    th0, orders = no.plan(m.n_items, 4, 5, len(pieces), 1, 2)
    th, losses = no.train(th0, (m.n_items, 4, 5), pieces, orders, 7, 0.01, 1, 0.25, 0.5, 4)
    np.testing.assert_allclose(m.params, th, rtol=1e-5, atol=1e-6)


def _test_frame(train, seed):
    te = _frame(12, 15, seed)
    return te[te.ItemId.isin(train.ItemId.unique())]


def test_evaluate_events_and_gpu_surface(fitted):
    m, train = fitted
    te = _test_frame(train, 5)
    r = evaluation.evaluate_events(m, te, cut_off=[1, 5], k=3)
    assert r['topk_items'].shape[1] == 3
    rec, mrr = evaluation.evaluate_gpu(m, te, cut_off=[1, 5])
    assert 0.0 <= rec[1] <= 1.0 and 0.0 <= mrr[1] <= 1.0
    items = train.ItemId.unique()[:6]
    evaluation.evaluate_events(m, te, cut_off=[2], items=items, exclude_seen=True)


def test_predict_next_of_a_fitted_model_ranks_as_the_evaluation(fitted):
    m, train = fitted
    ids = m.itemidmap.index.values
    te = _test_frame(train, 6)
    sid = te.SessionId.iloc[0]
    seq = te[te.SessionId == sid].ItemId.values
    p = m.params64()
    for t in range(len(seq)):
        got = m.predict_next(sid, seq[t], ids).values
        want = p['E'] @ no.encode(p, [m.itemidmap[x] for x in seq[:t + 1]], m.max_len)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_pickle_round_trip_without_the_handle(fitted, tmp_path):
    m, train = fitted
    m._device()
    b = pickle.loads(pickle.dumps(m))
    assert '_dev' not in b.__dict__ and np.array_equal(b.params, m.params)
    te = _test_frame(train, 7)
    r1 = evaluation.evaluate_events(m, te, cut_off=[5])
    r2 = evaluation.evaluate_events(b, te, cut_off=[5])
    pd.testing.assert_frame_equal(r1['events'], r2['events'])
    assert r1['recall'] == r2['recall'] and r1['mrr'] == r2['mrr']


@pytest.mark.parametrize('bad', [dict(embedding=0), dict(hidden=2000), dict(max_len=1), dict(dropout_emb=1.0), dict(dropout_ct=-0.1),
                                 dict(learning_rate=0.0), dict(batch_size=0), dict(embedding=2.5)])
def test_bad_arguments_are_refused_before_any_device_work(monkeypatch, bad):
    def no_device(*a, **k):
        raise AssertionError('device work')
    monkeypatch.setattr(_lib, 'Baselines', no_device)
    with pytest.raises(ValueError):
        baselines.NARM(**bad).fit(_frame(5, 4, 0))


def test_binding_refuses_wrong_parameter_counts():
    b = _lib.Baselines.__new__(_lib.Baselines)
    b.n_items, b.n_keep = 10, 4
    with pytest.raises(ValueError):
        b._narm_params(3, np.zeros(5, np.float32))
    assert b.narm_n_params(3) == 10 * 4 + 5 * 4 * 3 + 5 * 9 + 12


def test_exports_and_kind():
    for name in ('g4r_bl_narm_begin', 'g4r_bl_narm_epoch', 'g4r_bl_narm_grads', 'g4r_bl_narm_export', 'g4r_bl_narm_import',
                 'g4r_bl_narm_encode'):
        assert name in _lib.EXPORTS
    assert _lib.BASELINE_KINDS['narm'] == 12
    with open(os.path.join(ROOT, 'include', 'g4r.h')) as f:
        assert '#define G4R_BL_NARM 12' in f.read()


def test_run_py_baseline_narm(double, tmp_path, capsys):
    import run
    train, test = _frame(30, 10, 0), _frame(8, 10, 1)
    test = test[test.ItemId.isin(train.ItemId.unique())]
    tr, te = tmp_path / 'train.tsv', tmp_path / 'test.tsv'
    train.to_csv(tr, sep='\t', index=False)
    test.to_csv(te, sep='\t', index=False)
    run.main([str(tr), '--baseline', 'narm', '-ps', 'embedding=3,hidden=4,n_epochs=1,batch_size=5,max_len=3,dropout_ct=0.1', '-t', str(te),
              '-m', '5'])
    out = capsys.readouterr().out
    assert 'Creating NARM model' in out and 'Recall@5' in out
    with pytest.raises(SystemExit):
        run.main([str(tr), '--baseline', 'narm', '--rest_of_session', '-t', str(te)])
