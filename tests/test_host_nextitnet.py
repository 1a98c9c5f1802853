"""NextItNet (DESIGN §3w) without a GPU: the float64 oracle's backward against central differences (kernel sizes 1 to 3,
repeated items, a target that is also an input, one-input pieces), causality and the receptive field, the init layout, the
pieces, the package's host encoder and predict_next against the oracle, the class's fit, evaluation surface, pickles and run.py
(with its /-separated dilations) through a CPU double of _lib.Baselines backed by the oracle, the refusals before any device work,
the exports and a C99 caller of kind 19."""
import functools
import os
import pickle
import shutil
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, 'oracle'), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import nextitnet_cases as nic  # noqa: E402
import nextitnet_oracle as nio  # noqa: E402
from gru4rec_b200 import _lib, baselines, evaluation  # noqa: E402

# one-input pieces, repeated items, a target that is also an input
BATCH = [[1, 2, 1, 3, 3, 2, 4], [5, 6], [0, 0, 0], [2, 4, 2, 4, 6, 2], [3, 3, 3, 1]]


def _params(NI, d, dil, K, seed=0, scale=1.0):
    """the init with non-zero biases and gains away from 1, so that their gradients reach every term"""
    rs = np.random.RandomState(seed)
    p = nio.unpack(nio.init(NI, d, dil, K, rs).astype(np.float64), NI, d, dil, K)
    for name, v in p.items():
        if v.ndim == 1:
            p[name] = (1.0 if name[0] == 'g' else 0.0) + 0.3 * rs.randn(v.size)
    return {k: v * scale for k, v in p.items()}


@pytest.mark.parametrize('d,dil,K', [(1, (1,), 2), (3, (1, 2), 3), (2, (2, 1), 1)])
def test_oracle_backward_matches_central_differences(d, dil, K):
    NI = 7
    p = _params(NI, d, dil, K, d + K)
    _, g = nio.loss_and_grads(p, BATCH, dil, K)
    th, gf = nio.pack(p, dil, K), nio.pack(g, dil, K)
    assert np.abs(gf).max() > 1e-3

    def loss(t):
        return nio.loss_and_grads(nio.unpack(t, NI, d, dil, K), BATCH, dil, K)[0]

    for i in range(th.size):
        a, b = th.copy(), th.copy()
        a[i] += 1e-6
        b[i] -= 1e-6
        fd = (loss(a) - loss(b)) / 2e-6
        assert abs(fd - gf[i]) <= 1e-4 * abs(fd) + 1e-7, (i, fd, gf[i])


def test_magnitude_bound_dominates_the_gradient():
    dil, K = (1, 2), 3
    p = _params(9, 5, dil, K, 1, 2.0)
    _, g = nio.loss_and_grads(p, BATCH, dil, K)
    _, m = nio.loss_and_grads(p, BATCH, dil, K, mag=True)
    assert (np.abs(nio.pack(g, dil, K)) <= nio.pack(m, dil, K) * (1 + 1e-9) + 1e-300).all()


def test_taps_and_their_adjoint():
    rs = np.random.RandomState(0)
    for n, d, K, l in [(7, 3, 3, 2), (5, 2, 1, 4), (4, 2, 3, 9)]:
        x, y = rs.randn(n, d), rs.randn(n, K * d)
        col = nio.taps(x, K, l)
        np.testing.assert_allclose((col * y).sum(), (x * nio.taps_adjoint(y, K, l)).sum(), rtol=1e-12)
        np.testing.assert_array_equal(col[:, (K - 1) * d:], x)            # the last tap is the position itself
        np.testing.assert_array_equal(col, baselines._causal_taps(x, K, l))


def test_changing_an_input_leaves_every_earlier_q_unchanged():
    dil, K = (1, 2, 1), 3
    p = _params(20, 6, dil, K, 3)
    x = [3, 7, 1, 9, 12, 4, 4, 0, 18, 5]
    _, q = nio.piece_forward(p, x, dil, K)
    for t in range(len(x)):
        y = list(x)
        y[t] = (y[t] + 5) % 20
        _, q2 = nio.piece_forward(p, y, dil, K)
        np.testing.assert_array_equal(q2[:t], q[:t])
        assert np.abs(q2[t] - q[t]).max() > 1e-6


def test_an_input_past_the_receptive_field_leaves_q_unchanged():
    for dil, K in [((1, 2), 3), ((1,), 2), ((2, 1, 3), 2)]:
        R = nic.receptive_field(dil, K)
        p = _params(30, 5, dil, K, 4)
        rs = np.random.RandomState(R)
        x = list(rs.randint(0, 30, R + 4))
        q = nio.encode(p, x, dil, K, 512)
        y = list(x)
        y[len(x) - 2 - R] = (y[len(x) - 2 - R] + 1) % 30                    # further back than 1 + R: invisible
        np.testing.assert_array_equal(nio.encode(p, y, dil, K, 512), q)
        z = list(x)
        z[len(x) - 1 - R] = (z[len(x) - 1 - R] + 1) % 30                    # exactly R back: seen
        assert np.abs(nio.encode(p, z, dil, K, 512) - q).max() > 1e-9


def test_init_layout_and_n_params():
    NI, d, dil, K = 13, 6, (1, 2, 4), 3
    rs_a, rs_b = np.random.RandomState(5), np.random.RandomState(5)
    th = baselines.nextitnet_init(NI, d, dil, K, rs_a)
    n = 2 * NI * d + NI + len(dil) * (2 * K * d * d + 6 * d)
    assert th.dtype == np.float32 and th.size == n == nio.n_params(NI, d, dil, K)
    np.testing.assert_array_equal(th, nio.init(NI, d, dil, K, rs_b))
    assert np.array_equal(rs_a.permutation(20), rs_b.permutation(20))       # the epoch orders follow from the same state
    assert list(baselines.nextitnet_shapes(NI, d, dil, K)) == [name for name, _ in nio.shapes(NI, d, dil, K)]
    p = baselines.nextitnet_unpack(th, NI, d, dil, K)
    assert p['C1_0'].shape == (K * d, d) and p['W'].shape == (NI, d) and p['bW'].shape == (NI,)
    rs = np.random.RandomState(5)
    for name, shp in nio.shapes(NI, d, dil, K):
        if len(shp) == 2:
            s = np.sqrt(6.0 / (shp[0] + shp[1]))
            np.testing.assert_array_equal(p[name], rs.uniform(-s, s, size=shp).astype(np.float32))
        else:
            assert (p[name] == (1.0 if name[0] == 'g' else 0.0)).all(), name
    b = _lib.Baselines.__new__(_lib.Baselines)
    b.n_items, b.n_keep = NI, d
    assert b.nextitnet_n_params(len(dil), K) == th.size
    with pytest.raises(ValueError):
        b._nextitnet_params(dil, K, th[:-1])


@pytest.mark.parametrize('max_len', [1, 2, 5])
def test_pieces_cover_every_pair_once(max_len):
    rs = np.random.RandomState(max_len)
    lens = [1, 2, max_len, max_len + 1, max_len + 2, 2 * max_len + 3, 1, 7]
    sessions = [list(rs.randint(0, 20, n)) for n in lens]
    frame = pd.DataFrame([(s, 100 + it, float(t)) for s, seq in enumerate(sessions) for t, it in enumerate(seq)], columns=['SessionId', 'ItemId', 'Time'])
    m = baselines.NextItNet(max_len=max_len)
    poff, pitems = m.pieces(frame.sample(frac=1.0, random_state=0))        # rows in any order: events by time
    ids = m.itemidmap.index.values
    got = [[int(ids[i]) - 100 for i in pitems[poff[k]:poff[k + 1]]] for k in range(len(poff) - 1)]
    want = nio.pieces(sessions, max_len)
    assert sorted(got) == sorted([list(map(int, w)) for w in want])
    assert all(2 <= len(g) <= max_len + 1 for g in got)
    pairs = sorted((tuple(g[:j + 1]), g[j + 1]) for g in got for j in range(len(g) - 1))
    assert len(pairs) == sum(n - 1 for n in lens if n >= 2)


def _model(NI=12, d=8, dil=(1, 2), K=3, max_len=4, seed=3):
    m = baselines.NextItNet(embedding=d, dilations=dil, kernel_size=K, max_len=max_len)
    m.n_items = NI
    m.itemidmap = pd.Series(data=np.arange(NI), index=np.arange(100, 100 + NI))
    m.params = nio.pack(_params(NI, d, dil, K, seed), dil, K).astype(np.float32)
    return m


def test_predict_next_equals_the_oracle_encoder():
    m = _model()
    p = nio.unpack(m.params, m.n_items, m.embedding, m.dilations, m.kernel_size)
    ids = np.arange(100, 112)
    seq = [3, 5, 5, 0, 11, 3, 7]
    for t, x in enumerate(seq):
        got = m.predict_next('s', 100 + x, ids).values
        want = p['W'] @ nio.encode(p, seq[:t + 1], m.dilations, m.kernel_size, m.max_len) + p['bW']
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


class OracleNextItNet(object):
    """_lib.Baselines for kind 'nextitnet' on the float64 oracle (parameters kept as float32, as the device keeps them)"""

    def __init__(self, kind, n_items, n_keep, device=0):
        assert kind == 'nextitnet'
        self.n_items, self.n_keep = n_items, n_keep

    def nextitnet_begin(self, dilations, K, max_len, batch_size, piece_offsets, items, params):
        self.dil, self.K, self.L, self.bs = tuple(int(v) for v in dilations), int(K), max_len, batch_size
        self.pieces = [list(items[piece_offsets[k]:piece_offsets[k + 1]]) for k in range(len(piece_offsets) - 1)]
        self.th = np.asarray(params, np.float32).copy()
        self.m = np.zeros(self.th.size)
        self.v = np.zeros(self.th.size)
        self.t = 0

    def _p(self):
        return nio.unpack(self.th, self.n_items, self.n_keep, self.dil, self.K)

    def nextitnet_epoch(self, order, lr):
        losses = []
        for b0 in range(0, len(order), self.bs):
            loss, g = nio.loss_and_grads(self._p(), [self.pieces[k] for k in order[b0:b0 + self.bs]], self.dil, self.K)
            self.t += 1
            th, self.m, self.v = nio.adam(self.th.astype(np.float64), nio.pack(g, self.dil, self.K), self.m, self.v, self.t, lr)
            self.th = th.astype(np.float32)
            losses.append(loss)
        return np.array(losses, np.float32), 0.0

    def nextitnet_export(self):
        return self.th.copy()

    def nextitnet_import(self, dilations, K, max_len, params):
        self.dil, self.K, self.L = tuple(int(v) for v in dilations), int(K), max_len
        self.th = np.asarray(params, np.float32).copy()

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        p = self._p()
        qs = nio.encode_events(p, np.asarray(items), offsets, n_history, self.dil, self.K, self.L).astype(np.float32)
        cnt, ti, ts = nio.rank_events(p['W'], p['bW'], qs, items, offsets, n_history, ('standard', 'conservative', 'median', 'tiebreaking')[mode],
                                      cand, exclude_seen, k)
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
    monkeypatch.setattr(_lib, 'Baselines', OracleNextItNet)


def _frame(n_sessions, n_items, seed, max_len=9):
    rs = np.random.RandomState(seed)
    rows = []
    for s in range(n_sessions):
        for t in range(rs.randint(1, max_len)):
            rows.append((s, 1000 + rs.randint(n_items), float(s * 100 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


_KW = dict(embedding=4, dilations=(1, 2), kernel_size=2, n_epochs=3, batch_size=9, learning_rate=0.01, max_len=3, seed=1)


@pytest.fixture
def fitted(double):
    train = _frame(30, 15, 0)
    m = baselines.NextItNet(**_KW)
    m.fit(train)
    return m, train


def test_fit_prints_epochs_and_matches_the_oracle(double, capsys):
    train = _frame(30, 15, 0)
    m = baselines.NextItNet(**_KW)
    capsys.readouterr()
    m.fit(train)
    lines = capsys.readouterr().out.split('\n')
    assert len(m.fit_stats) == 3 and all(np.isfinite(s[0]) for s in m.fit_stats)
    assert lines[:3] == ['%d %s' % (e, m.fit_stats[e][0]) for e in range(3)]
    poff, pitems = m.pieces(train)
    pcs = [list(pitems[poff[k]:poff[k + 1]]) for k in range(len(poff) - 1)]
    th0, orders = nio.plan(m.n_items, 4, (1, 2), 2, len(pcs), 1, 3)
    th, _ = nio.train(th0, (m.n_items, 4, (1, 2), 2), pcs, orders, 9, 0.01)
    np.testing.assert_allclose(m.params, th, rtol=1e-5, atol=1e-6)
    assert m.fit_stats[-1][0] < m.fit_stats[0][0]


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
    evaluation.evaluate_events(m, te, cut_off=[2], items=train.ItemId.unique()[:6], exclude_seen=True)
    hist = _test_frame(train, 8)
    evaluation.evaluate_gpu(m, te, cut_off=[5], history=hist)


def test_predict_next_of_a_fitted_model_uses_the_last_max_len_inputs(fitted):
    m, train = fitted
    ids = m.itemidmap.index.values
    te = _test_frame(train, 6)
    sid = te.SessionId.value_counts().index[0]
    seq = te[te.SessionId == sid].ItemId.values
    assert len(seq) > m.max_len
    p = m.params64()
    for t in range(len(seq)):
        got = m.predict_next(sid, seq[t], ids).values
        want = p['W'] @ nio.encode(p, [m.itemidmap[x] for x in seq[:t + 1]], m.dilations, m.kernel_size, m.max_len) + p['bW']
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_pickle_round_trip_without_the_handle(fitted):
    m, train = fitted
    m._device()
    m.params64()
    b = pickle.loads(pickle.dumps(m))
    assert '_dev' not in b.__dict__ and '_p64' not in b.__dict__ and np.array_equal(b.params, m.params)
    te = _test_frame(train, 7)
    r1 = evaluation.evaluate_events(m, te, cut_off=[5])
    r2 = evaluation.evaluate_events(b, te, cut_off=[5])
    pd.testing.assert_frame_equal(r1['events'], r2['events'])
    assert r1['recall'] == r2['recall'] and r1['mrr'] == r2['mrr']


@pytest.mark.parametrize('bad', [dict(embedding=0), dict(embedding=1025), dict(embedding=2.5), dict(kernel_size=0), dict(kernel_size=9),
                                 dict(dilations=()), dict(dilations=(1,) * 17), dict(dilations=(0, 1)), dict(dilations=(1, 257)),
                                 dict(dilations=(1, 2.0)), dict(dilations=(1, True)), dict(dilations='12'), dict(dilations=3),
                                 dict(max_len=0), dict(max_len=513), dict(learning_rate=0.0), dict(learning_rate=-1.0),
                                 dict(learning_rate=float('inf')), dict(learning_rate=float('nan')), dict(batch_size=0), dict(n_epochs=-1)])
def test_bad_arguments_are_refused_before_any_device_work(monkeypatch, bad):
    def no_device(*a, **k):
        raise AssertionError('device work')
    monkeypatch.setattr(_lib, 'Baselines', no_device)
    with pytest.raises(ValueError):
        baselines.NextItNet(**bad).fit(_frame(5, 4, 0))


def test_a_training_set_without_a_pair_is_refused(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleNextItNet)
    frame = pd.DataFrame([(0, 1, 0.0), (1, 2, 1.0)], columns=['SessionId', 'ItemId', 'Time'])
    with pytest.raises(ValueError, match='at least 2 events'):
        baselines.NextItNet().fit(frame)


def test_exports_and_kind():
    for name in ('g4r_bl_nextitnet_begin', 'g4r_bl_nextitnet_epoch', 'g4r_bl_nextitnet_grads', 'g4r_bl_nextitnet_export',
                 'g4r_bl_nextitnet_import', 'g4r_bl_nextitnet_encode'):
        assert name in _lib.EXPORTS
    assert _lib.BASELINE_KINDS['nextitnet'] == 19
    with open(os.path.join(ROOT, 'include', 'g4r.h')) as f:
        assert '#define G4R_BL_NEXTITNET 19' in f.read()
    import baselines as shim
    assert shim.NextItNet is baselines.NextItNet


def test_run_py_baseline_nextitnet_with_a_dilation_list(double, tmp_path, capsys, monkeypatch):
    import run
    train, test = _frame(30, 10, 0), _frame(8, 10, 1)
    test = test[test.ItemId.isin(train.ItemId.unique())]
    tr, te = tmp_path / 'train.tsv', tmp_path / 'test.tsv'
    train.to_csv(tr, sep='\t', index=False)
    test.to_csv(te, sep='\t', index=False)
    made = []
    real = baselines.NextItNet.__init__

    @functools.wraps(real)                  # run.py reads the constructor's signature
    def spy(self, *a, **k):
        real(self, *a, **k)
        made.append(self)
    monkeypatch.setattr(baselines.NextItNet, '__init__', spy)
    run.main([str(tr), '--baseline', 'nextitnet', '-ps', 'embedding=4,dilations=1/2/4,kernel_size=2,n_epochs=2,batch_size=5,max_len=3',
              '-t', str(te), '-m', '5'])
    out = capsys.readouterr().out
    assert 'Creating NextItNet model' in out and 'Recall@5' in out and '\n1 ' in out
    assert made[-1].dilations == (1, 2, 4) and made[-1].kernel_size == 2 and made[-1].embedding == 4
    with pytest.raises(SystemExit):
        run.main([str(tr), '--baseline', 'nextitnet', '-ps', 'dilations=1/x', '-t', str(te)])
    assert 'list of integers' in capsys.readouterr().out
    with pytest.raises(SystemExit):
        run.main([str(tr), '--baseline', 'nextitnet', '--rest_of_session', '-t', str(te)])
    assert 'does not cover the baselines yet' in capsys.readouterr().out


SRC = r'''
#include <math.h>
#include <stdio.h>
#include <stddef.h>
#include "g4r.h"
int main(void) {
  g4r_baselines* h = NULL;
  g4r_baselines* nm = NULL;
  /* 10 items, d 4, dilations {1, 2}, kernel_size 3: n_params = 2 * 40 + 10 + 2 * (2 * 3 * 16 + 24) = 330; pieces {1,2,3,4}, {5,6} */
  float th[330], bad[330], g[330], q[12], loss = 0.f, ms = 0.f, ls[2];
  const int32_t dil[2] = {1, 2}, dil0[2] = {0, 2}, dil257[2] = {1, 257};
  int32_t dil17[17];
  const int64_t po[3] = {0, 4, 6}, po_bad[3] = {0, 5, 4}, so1[2] = {0, 4};
  const int32_t it[6] = {1, 2, 3, 4, 5, 6}, it_bad[6] = {1, 2, 3, 4, 5, 10}, order[2] = {0, 1}, order3[3] = {0, 1, 0}, oob[1] = {2};
  int rc, i;
  for (i = 0; i < 330; i++) { th[i] = 0.01f * (float)(i % 7); bad[i] = th[i]; }
  for (i = 0; i < 17; i++) dil17[i] = 1;
  bad[5] = NAN;
  if (g4r_bl_create(18, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 2;
  if (g4r_bl_create(20, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 3;
  if (g4r_bl_create(G4R_BL_NEXTITNET, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  if (g4r_bl_create(G4R_BL_NEXTITNET, 10, 0, 0, &h) != G4R_ERR_INVALID || h != NULL) return 5;
  rc = g4r_bl_create(G4R_BL_NEXTITNET, 10, 4, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 6;
  if (g4r_bl_nextitnet_export(h, th, 330) != G4R_ERR_STATE) return 7;
  if (g4r_bl_nextitnet_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 8;
  if (g4r_bl_nextitnet_epoch(h, order, 2, 0.001f, ls, &ms) != G4R_ERR_STATE) return 9;
  if (g4r_bl_nextitnet_grads(h, order, 2, &loss, g) != G4R_ERR_STATE) return 10;
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 0, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 11;     /* max_len 0 */
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 513, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 12;
  if (g4r_bl_nextitnet_begin(h, dil, 2, 0, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 13;     /* kernel_size */
  if (g4r_bl_nextitnet_begin(h, dil, 2, 9, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 14;
  if (g4r_bl_nextitnet_begin(h, dil0, 2, 3, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 15;    /* a dilation of 0 */
  if (g4r_bl_nextitnet_begin(h, dil257, 2, 3, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 16;
  if (g4r_bl_nextitnet_begin(h, dil17, 17, 3, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 17;  /* 17 blocks */
  if (g4r_bl_nextitnet_begin(h, dil, 0, 3, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 18;
  if (g4r_bl_nextitnet_begin(h, NULL, 2, 3, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 19;
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 3, 2, po, 2, it, 6, th, 329) != G4R_ERR_INVALID) return 20;     /* n_params */
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 3, 2, po, 2, it, 6, bad, 330) != G4R_ERR_INVALID) return 21;    /* not finite */
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 3, 2, po, 2, it_bad, 6, th, 330) != G4R_ERR_INDEX) return 22;
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 3, 2, po_bad, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 23;
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 2, 2, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 24;     /* a piece past max_len + 1 */
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 3, 0, po, 2, it, 6, th, 330) != G4R_ERR_INVALID) return 25;
  if (g4r_bl_nextitnet_export(h, th, 330) != G4R_ERR_STATE) return 26;                                     /* nothing was set */
  if (g4r_bl_nextitnet_begin(h, dil, 2, 3, 3, 2, po, 2, it, 6, th, 330) != G4R_OK) return 27;
  if (g4r_bl_nextitnet_epoch(h, oob, 1, 0.001f, ls, &ms) != G4R_ERR_INDEX) return 28;
  if (g4r_bl_nextitnet_epoch(h, order, 2, 0.f, ls, &ms) != G4R_ERR_INVALID) return 29;
  if (g4r_bl_nextitnet_epoch(h, order, 2, INFINITY, ls, &ms) != G4R_ERR_INVALID) return 30;
  if (g4r_bl_nextitnet_grads(h, order3, 3, &loss, g) != G4R_ERR_INVALID) return 31;                       /* n > batch_size */
  if (g4r_bl_nextitnet_grads(h, order, 2, &loss, g) != G4R_OK || !(loss > 0.f)) return 32;
  if (g4r_bl_nextitnet_epoch(h, order, 2, 0.001f, ls, &ms) != G4R_OK) return 33;
  if (g4r_bl_nextitnet_encode(h, it, 4, so1, 1, NULL, q, 1) != G4R_ERR_INVALID) return 34;                /* n_q must be 3 */
  if (g4r_bl_nextitnet_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_OK) return 35;
  if (g4r_bl_nextitnet_export(h, th, 330) != G4R_OK) return 36;
  /* the other kinds' calls refuse a NextItNet handle, and NextItNet's refuse a SASRec handle */
  if (g4r_bl_narm_import(h, 4, 3, th, 330) != G4R_ERR_STATE) return 37;
  if (g4r_bl_sasrec_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 38;
  if (g4r_bl_stamp_epoch(h, order, 2, 0.001f, ls, &ms) != G4R_ERR_STATE) return 39;
  if (g4r_bl_stamp_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 40;
  if (g4r_bl_srgnn_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 41;
  if (g4r_bl_sasrec_grads(h, order, 2, 0u, 0, 0.f, &loss, g) != G4R_ERR_STATE) return 42;
  if (g4r_bl_bpr_import(h, NULL, NULL) != G4R_ERR_STATE) return 43;
  if (g4r_bl_create(G4R_BL_SASREC, 10, 4, 0, &nm) != G4R_OK) return 44;
  if (g4r_bl_nextitnet_import(nm, dil, 2, 3, 3, th, 330) != G4R_ERR_STATE) return 45;
  if (g4r_bl_nextitnet_export(nm, th, 330) != G4R_ERR_STATE) return 46;
  if (g4r_bl_nextitnet_encode(nm, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 47;
  if (g4r_bl_nextitnet_begin(nm, dil, 2, 3, 3, 2, po, 2, it, 6, th, 330) != G4R_ERR_STATE) return 48;
  if (g4r_bl_nextitnet_epoch(nm, order, 2, 0.001f, ls, &ms) != G4R_ERR_STATE) return 49;
  if (g4r_bl_nextitnet_grads(nm, order, 2, &loss, g) != G4R_ERR_STATE) return 50;
  if (g4r_bl_destroy(nm) != G4R_OK) return 51;
  if (g4r_bl_nextitnet_import(h, dil, 2, 3, 3, bad, 330) != G4R_ERR_INVALID) return 52;
  if (g4r_bl_last_error(h)[0] == 0) return 53;
  if (g4r_bl_destroy(h) != G4R_OK) return 54;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_nextitnet_abi(tmp_path):
    gcc = shutil.which('gcc') or shutil.which('cc')
    if gcc is None:
        pytest.skip('no C compiler')
    inc, libdir = os.path.join(ROOT, 'include'), os.path.join(ROOT, 'gru4rec_b200')
    src = tmp_path / 'caller.c'
    src.write_text(SRC)
    exe = str(tmp_path / 'caller')
    cuda_lib = '/usr/local/cuda/lib64'
    r = subprocess.run([gcc, '-std=c99', '-Wall', '-Wextra', '-pedantic', '-Werror', '-I' + inc, str(src), '-L' + libdir, '-lg4r',
                        '-Wl,-rpath,' + libdir, '-L' + cuda_lib, '-Wl,-rpath,' + cuda_lib, '-o', exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert r.stdout.startswith('ok ')
