"""BERT4Rec (DESIGN §3x) without a GPU: the float64 oracle's backward against central differences, bidirectionality, the cloze
mask rule, the init layout, the package's host encoder and predict_next against the oracle, the class's fit, evaluation surface,
pickles and run.py through a CPU double of _lib.Baselines backed by the oracle, the refusals before any device work, the exports
and a C99 caller of kind 21."""
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

import bert4rec_oracle as bo  # noqa: E402
from gru4rec_b200 import _lib, baselines, evaluation  # noqa: E402


def _params(NI, d, nb, L, seed=0, scale=2.0):
    """the init at scale, with random gains and biases so that every gradient term is generic"""
    rs = np.random.RandomState(seed)
    p = bo.unpack(bo.init(NI, d, nb, L, rs).astype(np.float64) * scale, NI, d, nb, L)
    for k in p:
        if p[k].ndim == 1:
            p[k] = (1.0 if k[0] == 'g' else 0.0) + rs.randn(p[k].size) * 0.3
    return p


def _loss(p, batch, masked, heads, drop, L, bs):
    _, Q, Y = bo.batch_forward(p, batch, masked, heads, 7, 3, drop, L, bs)
    S = Q @ p['E'][:-1].T + p['bO']
    m = S.max(axis=1, keepdims=True)
    return float(np.mean(np.log(np.exp(S - m).sum(axis=1)) + m[:, 0] - S[np.arange(len(Y)), Y]))


BATCH = [[1, 2, 3, 4, 6], [5, 6], [0, 0, 2], [3, 1, 4, 1, 5]]
ONE_MASK = [[False] * 4 + [True], [False, True], [False, False, True], [False] * 4 + [True]]
MANY = [[True, False, True, False, True], [True, True], [False, True, False], [True, False, True, True, False]]


@pytest.mark.parametrize('heads,nb', [(1, 1), (4, 1), (1, 3), (4, 3)])
@pytest.mark.parametrize('drop', [0.0, 0.3])
@pytest.mark.parametrize('masked', [ONE_MASK, MANY], ids=['last-masked', 'several-masked'])
def test_oracle_backward_matches_central_differences(heads, nb, drop, masked):
    NI, d, L, bs = 7, 4, 5, 4
    p = _params(NI, d, nb, L, seed=heads + 10 * nb)
    _, g = bo.loss_and_grads(p, BATCH, masked, heads, 7, 3, drop, L, bs)
    th, gf = bo.pack(p), bo.pack(g)
    for i in range(th.size):
        a, b = th.copy(), th.copy()
        a[i] += 1e-6
        b[i] -= 1e-6
        fd = (_loss(bo.unpack(a, NI, d, nb, L), BATCH, masked, heads, drop, L, bs) -
              _loss(bo.unpack(b, NI, d, nb, L), BATCH, masked, heads, drop, L, bs)) / 2e-6
        assert abs(fd - gf[i]) <= 1e-4 * abs(fd) + 1e-7, (i, fd, gf[i])
    # the mask row is an input: its gradient is nonzero, and the output bias's sums to 0 (a softmax row's gradient does)
    assert np.abs(g['E'][NI]).max() > 1e-6 and abs(g['bO'].sum()) < 1e-12


def test_magnitude_bound_dominates_the_gradient():
    NI, d, nb, L = 9, 8, 2, 7
    p = _params(NI, d, nb, L, 1)
    batch = [[1, 2, 3, 4, 8, 0, 2], [5, 6], [0, 7, 2]]
    masked = [[True, False, False, True, False, False, True], [False, True], [True, True, False]]
    _, g = bo.loss_and_grads(p, batch, masked, 2, 1, 0, 0.25, L, 4)
    _, m = bo.loss_and_grads(p, batch, masked, 2, 1, 0, 0.25, L, 4, mag=True)
    assert (np.abs(bo.pack(g)) <= bo.pack(m) * (1 + 1e-9) + 1e-300).all()


def test_attention_is_bidirectional():
    NI, d, nb, L = 11, 8, 2, 9
    p = _params(NI, d, nb, L, 2)
    rs = np.random.RandomState(3)
    x = list(rs.randint(0, NI, L))
    none = [False] * L
    _, q = bo.piece_forward(p, x, none, 2)
    for k in range(1, L):
        y = list(x)
        y[k] = (y[k] + 1) % NI                                     # a later input changes every earlier position's q
        _, qy = bo.piece_forward(p, y, none, 2)
        assert (np.abs(q[:k] - qy[:k]).max(axis=1) > 1e-9).all(), k
    # a window's q (at the mask) depends on every input in it, and equals the package's host encoder
    w = x[:L - 1]
    q0 = bo.encode(p, w, 2, L)
    np.testing.assert_allclose(baselines.bert4rec_encode(p, w, 2), q0, rtol=1e-12, atol=1e-12)
    for k in range(L - 1):
        v = list(w)
        v[k] = (v[k] + 3) % NI
        assert np.abs(bo.encode(p, v, 2, L) - q0).max() > 1e-9, k


def test_the_mask_rule():
    rs = np.random.RandomState(0)
    lens = rs.randint(2, 30, 2000)
    off = np.r_[0, np.cumsum(lens)].astype(np.int64)
    for prob in (0.01, 0.2, 0.9):
        a, b, c = np.random.RandomState(4), np.random.RandomState(4), np.random.RandomState(5)
        mk = baselines.bert4rec_masks(off, prob, a)
        assert mk.dtype == np.uint8 and mk.size == off[-1] and set(np.unique(mk)) <= {0, 1}
        per = np.add.reduceat(mk.astype(np.int64), off[:-1])
        assert (per >= 1).all()                                              # at least one per piece
        want = bo.cloze(lens, prob, b)
        assert np.array_equal(mk, np.concatenate(want).astype(np.uint8))     # the oracle's rule, draw for draw
        assert not np.array_equal(mk, baselines.bert4rec_masks(off, prob, c))
        forced = (per == 1) & (mk[off[1:] - 1] == 1)
        rate = (mk.sum() - forced.sum()) / (off[-1] - forced.sum())          # the draws that are not forced
        assert abs(rate - prob) < 0.05 * max(prob, 0.1) + 0.01, (prob, rate)
    assert (np.add.reduceat(baselines.bert4rec_masks(off, 0.0, rs), off[:-1]) == 1).all()


def test_init_layout_and_n_params():
    NI, d, nb, L = 13, 6, 3, 7
    rs_a, rs_b = np.random.RandomState(5), np.random.RandomState(5)
    th = baselines.bert4rec_init(NI, d, nb, L, rs_a)
    assert th.dtype == np.float32 and th.size == (NI + 1) * d + L * d + 2 * d + nb * (12 * d * d + 13 * d) + d * d + 3 * d + NI == bo.n_params(NI, d, nb, L)
    np.testing.assert_array_equal(th, bo.init(NI, d, nb, L, rs_b))
    assert np.array_equal(rs_a.permutation(20), rs_b.permutation(20))       # the epoch orders follow from the same state
    assert list(baselines.bert4rec_shapes(NI, d, nb, L)) == [n for n, _ in bo.shapes(NI, d, nb, L)]
    p = baselines.bert4rec_unpack(th, NI, d, nb, L)
    assert p['E'].shape == (NI + 1, d) and p['W1_0'].shape == (d, 4 * d) and p['W2_2'].shape == (4 * d, d) and p['bO'].shape == (NI,)
    for name, v in p.items():
        if v.ndim == 2:
            s = np.sqrt(6.0 / sum(v.shape))
            assert np.abs(v).max() <= s and np.abs(v).max() > 0.5 * s, name
        else:
            assert (v == (1.0 if name[0] == 'g' else 0.0)).all(), name
    b = _lib.Baselines.__new__(_lib.Baselines)
    b.n_items, b.n_keep = NI, d
    assert b.bert4rec_n_params(nb, L) == th.size
    with pytest.raises(ValueError):
        b._bert4rec_params(nb, L, th[:-1])


@pytest.mark.parametrize('max_len', [2, 3, 6])
def test_pieces_hold_at_most_max_len_events(max_len):
    rs = np.random.RandomState(max_len)
    lens = [1, 2, max_len, max_len + 1, 2 * max_len + 3, 1, 7]
    sessions = [list(rs.randint(0, 20, n)) for n in lens]
    pieces = bo.pieces(sessions, max_len)
    assert all(2 <= len(pc) <= max_len for pc in pieces)
    assert sorted(set(x for pc in pieces for x in pc)) == sorted(set(x for s in sessions if len(s) > 1 for x in s))
    frame = pd.DataFrame([(s, 100 + it, float(t)) for s, seq in enumerate(sessions) for t, it in enumerate(seq)],
                         columns=['SessionId', 'ItemId', 'Time'])
    m = baselines.BERT4Rec(max_len=max_len)
    poff, pit = m.pieces(frame.sample(frac=1.0, random_state=0))
    ids = m.itemidmap.index.values
    assert sorted([int(ids[i]) - 100 for i in pit[poff[k]:poff[k + 1]]] for k in range(len(poff) - 1)) == sorted(pieces)


def _model(NI=12, d=8, nb=2, heads=2, max_len=4, seed=3):
    m = baselines.BERT4Rec(embedding=d, n_blocks=nb, n_heads=heads, max_len=max_len)
    m.n_items = NI
    m.itemidmap = pd.Series(data=np.arange(NI), index=np.arange(100, 100 + NI))
    m.params = bo.pack(_params(NI, d, nb, max_len, seed)).astype(np.float32)
    return m


def test_predict_next_equals_the_oracle_encoder():
    m = _model()
    p = bo.unpack(m.params, m.n_items, m.embedding, m.n_blocks, m.max_len)
    ids = np.arange(100, 112)
    seq = [3, 5, 5, 0, 11, 2, 7]
    for t, x in enumerate(seq):
        got = m.predict_next('s', 100 + x, ids).values
        want = p['E'][:-1] @ bo.piece_forward(p, seq[max(0, t + 2 - m.max_len):t + 1] + [0],
                                              [False] * (min(t + 1, m.max_len - 1)) + [True], m.n_heads)[1][-1] + p['bO']
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


class OracleBert4rec(object):
    """_lib.Baselines for kind 'bert4rec' on the float64 oracle (parameters kept as float32, as the device keeps them); it records
    every epoch's masks"""
    uploads = []

    def __init__(self, kind, n_items, n_keep, device=0):
        assert kind == 'bert4rec'
        self.n_items, self.n_keep = n_items, n_keep

    def bert4rec_begin(self, n_blocks, n_heads, max_len, batch_size, piece_offsets, items, params):
        self.nb, self.heads, self.L, self.bs = n_blocks, n_heads, max_len, batch_size
        self.off = np.asarray(piece_offsets)
        self.pieces = [list(items[piece_offsets[k]:piece_offsets[k + 1]]) for k in range(len(piece_offsets) - 1)]
        self.th = np.asarray(params, np.float32).copy()
        self.m = np.zeros(self.th.size)
        self.v = np.zeros(self.th.size)
        self.step = 0

    def _p(self):
        return bo.unpack(self.th, self.n_items, self.n_keep, self.nb, self.L)

    def bert4rec_epoch(self, order, masks, seed, lr, dropout):
        OracleBert4rec.uploads.append(np.array(masks))
        masked = [list(np.asarray(masks[self.off[k]:self.off[k + 1]]) != 0) for k in range(len(self.pieces))]
        losses = []
        for b0 in range(0, len(order), self.bs):
            ks = order[b0:b0 + self.bs]
            loss, g = bo.loss_and_grads(self._p(), [self.pieces[k] for k in ks], [masked[k] for k in ks], self.heads, seed, self.step, dropout,
                                        self.L, self.bs)
            self.step += 1
            th, self.m, self.v = bo.adam(self.th.astype(np.float64), bo.pack(g), self.m, self.v, self.step, lr)
            self.th = th.astype(np.float32)
            losses.append(loss)
        return np.array(losses, np.float32), 0.0

    def bert4rec_export(self):
        return self.th.copy()

    def bert4rec_import(self, n_blocks, n_heads, max_len, params):
        self.nb, self.heads, self.L, self.th = n_blocks, n_heads, max_len, np.asarray(params, np.float32).copy()

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        p = self._p()
        qs = bo.encode_events(p, np.asarray(items), offsets, n_history, self.heads, self.L).astype(np.float32)
        cnt, ti, ts = bo.rank_events(p['E'][:-1], p['bO'], qs, items, offsets, n_history, ('standard', 'conservative', 'median', 'tiebreaking')[mode],
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
    OracleBert4rec.uploads = []
    monkeypatch.setattr(_lib, 'Baselines', OracleBert4rec)


def _frame(n_sessions, n_items, seed, max_len=9):
    rs = np.random.RandomState(seed)
    rows = []
    for s in range(n_sessions):
        for t in range(rs.randint(1, max_len)):
            rows.append((s, 1000 + rs.randint(n_items), float(s * 100 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


_KW = dict(embedding=4, n_blocks=2, n_heads=2, n_epochs=2, batch_size=7, learning_rate=0.01, dropout=0.2, mask_prob=0.3, max_len=4, seed=1)


@pytest.fixture
def fitted(double):
    train = _frame(40, 15, 0)
    m = baselines.BERT4Rec(**_KW)
    m.fit(train)
    return m, train


def test_fit_prints_epochs_uploads_the_mask_rule_and_matches_the_oracle(double, capsys):
    train = _frame(40, 15, 0)
    m = baselines.BERT4Rec(**_KW)
    capsys.readouterr()
    m.fit(train)
    lines = capsys.readouterr().out.split('\n')
    assert len(m.fit_stats) == 2 and all(np.isfinite(s[0]) for s in m.fit_stats)
    assert lines[:2] == ['%d %s' % (e, m.fit_stats[e][0]) for e in range(2)]
    poff, pit = m.pieces(train)
    pieces = [list(pit[poff[k]:poff[k + 1]]) for k in range(len(poff) - 1)]
    th0, epochs = bo.plan(m.n_items, 4, 2, 4, [len(pc) for pc in pieces], 1, 2, 0.3)
    # the masks fit uploads are the oracle's rule drawn after each epoch's permutation
    assert len(OracleBert4rec.uploads) == 2
    for up, (_, masked) in zip(OracleBert4rec.uploads, epochs):
        assert np.array_equal(up, np.concatenate(masked).astype(np.uint8))
    th, _ = bo.train(th0, (m.n_items, 4, 2, 4), 2, pieces, epochs, 7, 0.01, 1, 0.2)
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
    evaluation.evaluate_events(m, te, cut_off=[2], items=train.ItemId.unique()[:6], exclude_seen=True)


def test_predict_next_of_a_fitted_model_uses_the_last_max_len_minus_one_inputs(fitted):
    m, train = fitted
    ids = m.itemidmap.index.values
    te = _test_frame(train, 6)
    sid = te.SessionId.value_counts().index[0]
    seq = te[te.SessionId == sid].ItemId.values
    assert len(seq) > m.max_len
    p = m.params64()
    for t in range(len(seq)):
        got = m.predict_next(sid, seq[t], ids).values
        want = p['E'][:-1] @ bo.encode(p, [m.itemidmap[x] for x in seq[:t + 1]], m.n_heads, m.max_len) + p['bO']
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_pickle_round_trip_without_the_handle(fitted):
    m, train = fitted
    m._device()
    b = pickle.loads(pickle.dumps(m))
    assert '_dev' not in b.__dict__ and '_p64' not in b.__dict__ and np.array_equal(b.params, m.params)
    te = _test_frame(train, 7)
    r1 = evaluation.evaluate_events(m, te, cut_off=[5])
    r2 = evaluation.evaluate_events(b, te, cut_off=[5])
    pd.testing.assert_frame_equal(r1['events'], r2['events'])
    assert r1['recall'] == r2['recall'] and r1['mrr'] == r2['mrr']


@pytest.mark.parametrize('bad', [dict(embedding=0), dict(embedding=1025), dict(embedding=2.5), dict(n_heads=3), dict(n_heads=0),
                                 dict(n_blocks=0), dict(n_blocks=9), dict(max_len=1), dict(max_len=513), dict(dropout=1.0),
                                 dict(dropout=-0.1), dict(mask_prob=-0.1), dict(mask_prob=1.5), dict(learning_rate=0.0),
                                 dict(learning_rate=float('inf')), dict(batch_size=0), dict(n_epochs=-1),
                                 dict(embedding=1024, n_blocks=8, max_len=512, batch_size=1024)])
def test_bad_arguments_are_refused_before_any_device_work(monkeypatch, bad):
    def no_device(*a, **k):
        raise AssertionError('device work')
    monkeypatch.setattr(_lib, 'Baselines', no_device)
    with pytest.raises(ValueError):
        baselines.BERT4Rec(**bad).fit(_frame(5, 4, 0))


def test_exports_and_kind():
    for name in ('g4r_bl_bert4rec_begin', 'g4r_bl_bert4rec_epoch', 'g4r_bl_bert4rec_grads', 'g4r_bl_bert4rec_export', 'g4r_bl_bert4rec_import',
                 'g4r_bl_bert4rec_encode'):
        assert name in _lib.EXPORTS
    assert _lib.BASELINE_KINDS['bert4rec'] == 21
    with open(os.path.join(ROOT, 'include', 'g4r.h')) as f:
        src = f.read()
    assert '#define G4R_BL_BERT4REC 21' in src
    assert 'n_params = (n_items + 1) d + max_len d + 2 d + n_blocks (12 d^2 + 13 d) + d^2 + 3 d + n_items' in src
    import baselines as shim
    assert shim.BERT4Rec is baselines.BERT4Rec


def test_run_py_baseline_bert4rec(double, tmp_path, capsys):
    import run
    train, test = _frame(30, 10, 0), _frame(8, 10, 1)
    test = test[test.ItemId.isin(train.ItemId.unique())]
    tr, te = tmp_path / 'train.tsv', tmp_path / 'test.tsv'
    train.to_csv(tr, sep='\t', index=False)
    test.to_csv(te, sep='\t', index=False)
    run.main([str(tr), '--baseline', 'bert4rec', '-ps', 'embedding=4,n_blocks=1,n_heads=2,mask_prob=0.2,n_epochs=2,batch_size=5,max_len=3',
              '-t', str(te), '-m', '5'])
    out = capsys.readouterr().out
    assert 'Creating BERT4Rec model' in out and 'Recall@5' in out and '\n1 ' in out
    with pytest.raises(SystemExit):
        run.main([str(tr), '--baseline', 'bert4rec', '--rest_of_session', '-t', str(te)])


SRC = r'''
#include <math.h>
#include <stdio.h>
#include <stddef.h>
#include "g4r.h"
int main(void) {
  g4r_baselines* h = NULL;
  g4r_baselines* sa = NULL;
  /* 10 items, d 4: one block, two heads, max_len 3; n_params = 44 + 12 + 8 + (192 + 52) + 16 + 12 + 10 = 346 */
  float th[346], bad[346], g[346], q[8], loss = 0.f, ms = 0.f, ls[2];
  const int64_t po[3] = {0, 3, 5}, po_long[2] = {0, 5}, so[2] = {0, 4};
  const int32_t it[5] = {1, 2, 3, 4, 5}, it_bad[5] = {1, 2, 3, 4, 10}, order[2] = {0, 1}, order3[3] = {0, 1, 0}, oob[1] = {2};
  const uint8_t mk[5] = {0, 1, 0, 1, 1}, mk_none[5] = {0, 0, 0, 1, 1}, mk_two[5] = {0, 2, 0, 1, 1};
  int rc, i;
  for (i = 0; i < 346; i++) { th[i] = 0.01f * (float)(i % 7); bad[i] = th[i]; }
  bad[5] = INFINITY;
  if (g4r_bl_create(20, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 2;
  if (g4r_bl_create(22, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 3;
  if (g4r_bl_create(G4R_BL_BERT4REC, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  rc = g4r_bl_create(G4R_BL_BERT4REC, 10, 4, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 5;
  /* nothing to export or evaluate before begin / import; no epoch before begin */
  if (g4r_bl_bert4rec_export(h, th, 346) != G4R_ERR_STATE) return 6;
  if (g4r_bl_bert4rec_encode(h, it, 4, so, 1, NULL, q, 2) != G4R_ERR_STATE) return 7;
  if (g4r_bl_bert4rec_epoch(h, order, 2, mk, 5, 1, 0.001f, 0.f, ls, &ms) != G4R_ERR_STATE) return 8;
  /* shapes, counts, pieces and values */
  if (g4r_bl_bert4rec_begin(h, 0, 2, 3, 2, po, 2, it, 5, th, 346) != G4R_ERR_INVALID) return 9;
  if (g4r_bl_bert4rec_begin(h, 9, 2, 3, 2, po, 2, it, 5, th, 346) != G4R_ERR_INVALID) return 10;
  if (g4r_bl_bert4rec_begin(h, 1, 3, 3, 2, po, 2, it, 5, th, 346) != G4R_ERR_INVALID) return 11;
  if (g4r_bl_bert4rec_begin(h, 1, 2, 1, 2, po, 2, it, 5, th, 346) != G4R_ERR_INVALID) return 12;
  if (g4r_bl_bert4rec_begin(h, 1, 2, 513, 2, po, 2, it, 5, th, 346) != G4R_ERR_INVALID) return 13;
  if (g4r_bl_bert4rec_begin(h, 1, 2, 3, 2, po, 2, it, 5, th, 345) != G4R_ERR_INVALID) return 14;
  if (g4r_bl_bert4rec_begin(h, 1, 2, 3, 2, po, 2, it, 5, bad, 346) != G4R_ERR_INVALID) return 15;
  if (g4r_bl_bert4rec_begin(h, 1, 2, 3, 2, po, 2, it_bad, 5, th, 346) != G4R_ERR_INDEX) return 16;
  if (g4r_bl_bert4rec_begin(h, 1, 2, 3, 2, po_long, 1, it, 5, th, 346) != G4R_ERR_INVALID) return 17;   /* 5 events > max_len */
  if (g4r_bl_bert4rec_begin(h, 1, 2, 3, 0, po, 2, it, 5, th, 346) != G4R_ERR_INVALID) return 18;
  if (g4r_bl_bert4rec_export(h, th, 346) != G4R_ERR_STATE) return 19;                                   /* nothing was set */
  if (g4r_bl_bert4rec_begin(h, 1, 2, 3, 2, po, 2, it, 5, th, 346) != G4R_OK) return 20;
  if (g4r_bl_bert4rec_epoch(h, oob, 1, mk, 5, 1, 0.001f, 0.f, ls, &ms) != G4R_ERR_INDEX) return 21;
  if (g4r_bl_bert4rec_epoch(h, order, 2, mk, 5, 1, 0.f, 0.f, ls, &ms) != G4R_ERR_INVALID) return 22;
  if (g4r_bl_bert4rec_epoch(h, order, 2, mk, 5, 1, 0.001f, 1.f, ls, &ms) != G4R_ERR_INVALID) return 23;
  if (g4r_bl_bert4rec_epoch(h, order, 2, mk_none, 5, 1, 0.001f, 0.f, ls, &ms) != G4R_ERR_INVALID) return 24;  /* piece 0 unmasked */
  if (g4r_bl_bert4rec_epoch(h, order, 2, mk_two, 5, 1, 0.001f, 0.f, ls, &ms) != G4R_ERR_INVALID) return 25;   /* a byte of 2 */
  if (g4r_bl_bert4rec_epoch(h, order, 2, mk, 4, 1, 0.001f, 0.f, ls, &ms) != G4R_ERR_INVALID) return 26;       /* n_masks */
  if (g4r_bl_bert4rec_grads(h, order3, 3, mk, 5, 1, 0, 0.f, &loss, g) != G4R_ERR_INVALID) return 27;         /* n > batch_size */
  if (g4r_bl_bert4rec_grads(h, order, 2, mk, 5, 1, 0, 0.1f, &loss, g) != G4R_OK || !(loss > 0.f)) return 28;
  if (g4r_bl_bert4rec_epoch(h, order, 2, mk, 5, 1, 0.001f, 0.1f, ls, &ms) != G4R_OK) return 29;
  if (g4r_bl_bert4rec_encode(h, it, 4, so, 1, NULL, q, 1) != G4R_ERR_INVALID) return 30;               /* n_q must be 3 */
  /* the other kinds' calls refuse a BERT4Rec handle, and BERT4Rec's refuse a SASRec handle */
  if (g4r_bl_sasrec_import(h, 1, 2, 3, th, 196) != G4R_ERR_STATE) return 31;
  if (g4r_bl_nextitnet_encode(h, it, 4, so, 1, NULL, q, 2) != G4R_ERR_STATE) return 32;
  if (g4r_bl_bpr_import(h, NULL, NULL) != G4R_ERR_STATE) return 33;
  if (g4r_bl_create(G4R_BL_SASREC, 10, 4, 0, &sa) != G4R_OK) return 34;
  if (g4r_bl_bert4rec_import(sa, 1, 2, 3, th, 346) != G4R_ERR_STATE) return 35;
  if (g4r_bl_bert4rec_epoch(sa, order, 2, mk, 5, 1, 0.001f, 0.f, ls, &ms) != G4R_ERR_STATE) return 36;
  if (g4r_bl_destroy(sa) != G4R_OK) return 37;
  if (g4r_bl_bert4rec_import(h, 1, 2, 3, bad, 346) != G4R_ERR_INVALID) return 38;
  if (g4r_bl_last_error(h)[0] == 0) return 39;
  if (g4r_bl_destroy(h) != G4R_OK) return 40;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_bert4rec_abi(tmp_path):
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
