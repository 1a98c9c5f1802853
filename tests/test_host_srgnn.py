"""SR-GNN (DESIGN §3u) without a GPU: the float64 oracle's backward against central differences (step 1 and 3, prefixes with
repeated items, self-loops and a single node), the graph construction, the samples, the init layout, the package's host encoder
and predict_next against the oracle, the class's fit, evaluation surface, pickles and run.py through a CPU double of
_lib.Baselines backed by the oracle, the refusals before any device work, the exports and a C99 caller of kind 15."""
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

import srgnn_oracle as so  # noqa: E402
from gru4rec_b200 import _lib, baselines, evaluation  # noqa: E402

BATCH = [([1, 2, 1, 3, 3, 2], 4), ([5], 6), ([0, 0], 1), ([2, 4, 2, 4, 6], 0), ([3, 3, 3], 3)]


def _params(NI, d, seed=0, scale=3.0):
    return so.unpack(so.init(NI, d, np.random.RandomState(seed)).astype(np.float64) * scale, NI, d)


def _loss(p, batch, step):
    return so.loss_and_grads(p, batch, step)[0]


@pytest.mark.parametrize('step', [1, 3])
def test_oracle_backward_matches_central_differences(step):
    NI, d = 7, 3
    p = _params(NI, d, step)
    _, g = so.loss_and_grads(p, BATCH, step)
    th, gf = so.pack(p), so.pack(g)
    for i in range(th.size):
        a, b = th.copy(), th.copy()
        a[i] += 1e-6
        b[i] -= 1e-6
        fd = (_loss(so.unpack(a, NI, d), BATCH, step) - _loss(so.unpack(b, NI, d), BATCH, step)) / 2e-6
        assert abs(fd - gf[i]) <= 1e-4 * abs(fd) + 1e-7, (i, fd, gf[i])


def test_magnitude_bound_dominates_the_gradient():
    p = _params(9, 5, 1)
    _, g = so.loss_and_grads(p, BATCH, 2)
    _, m = so.loss_and_grads(p, BATCH, 2, mag=True)
    assert (np.abs(so.pack(g)) <= so.pack(m) * (1 + 1e-9) + 1e-300).all()


def test_graph_nodes_alias_and_normalisation():
    x = [5, 2, 5, 5, 7, 2, 5, 2]
    for nodes, alias, a_in, a_out in (so.graph(x), baselines.srgnn_graph(x)):
        assert list(nodes) == [2, 5, 7] and list(alias) == [1, 0, 1, 1, 2, 0, 1, 0]
        # edges (repeats once): 5->2, 2->5, 5->5 (a self-loop), 5->7, 7->2
        want_in = np.array([[0, 1 / 2, 1 / 2], [1 / 2, 1 / 2, 0], [0, 1, 0]])       # A_in[v][u] = 1 / indeg(v)
        want_out = np.array([[0, 1, 0], [1 / 3, 1 / 3, 1 / 3], [1, 0, 0]])          # A_out[u][v] = 1 / outdeg(u)
        np.testing.assert_array_equal(a_in, want_in)
        np.testing.assert_array_equal(a_out, want_out)
    nodes, alias, a_in, a_out = baselines.srgnn_graph([4])
    assert list(nodes) == [4] and list(alias) == [0] and not a_in.any() and not a_out.any()    # a single node: zero rows
    nodes, alias, a_in, a_out = baselines.srgnn_graph([3, 1])
    np.testing.assert_array_equal(a_in, [[0, 1], [0, 0]])                                   # node 1 (item 3) has no in-edge


def test_a_repeated_edge_counts_once():
    for graph in (so.graph, baselines.srgnn_graph):
        a, b = graph([1, 2, 1, 2, 3]), graph([1, 2, 1, 2, 1, 2, 3])
        np.testing.assert_array_equal(a[2], b[2])
        np.testing.assert_array_equal(a[3], b[3])
        np.testing.assert_array_equal(a[3], [[0, 1, 0], [1 / 2, 0, 1 / 2], [0, 0, 0]])


@pytest.mark.parametrize('max_len', [1, 2, 5])
def test_samples_cover_every_pair_once_within_a_window_of_max_len(max_len):
    rs = np.random.RandomState(max_len)
    lens = [1, 2, max_len, max_len + 1, max_len + 2, 2 * max_len + 3, 1, 7]
    sessions = [list(rs.randint(0, 20, n)) for n in lens]
    smp = so.samples(sessions, max_len)
    assert sorted((tuple(x), y) for x, y in smp) == sorted((tuple(s[max(0, j - max_len):j]), s[j]) for s in sessions for j in range(1, len(s)))
    assert len(smp) == sum(n - 1 for n in lens) and all(1 <= len(x) <= max_len for x, _ in smp)
    frame = pd.DataFrame([(s, 100 + it, float(t)) for s, seq in enumerate(sessions) for t, it in enumerate(seq)], columns=['SessionId', 'ItemId', 'Time'])
    m = baselines.SRGNN(max_len=max_len)
    off, items = m.sessions(frame.sample(frac=1.0, random_state=0))        # rows in any order: events by time
    ids = m.itemidmap.index.values
    got = sorted([int(ids[i]) - 100 for i in items[off[k]:off[k + 1]]] for k in range(len(off) - 1))
    assert got == sorted(sessions)


def test_init_layout_and_n_params():
    NI, d = 13, 6
    rs_a, rs_b = np.random.RandomState(5), np.random.RandomState(5)
    th = baselines.srgnn_init(NI, d, rs_a)
    assert th.dtype == np.float32 and th.size == NI * d + 15 * d * d + 14 * d == so.n_params(NI, d)
    np.testing.assert_array_equal(th, so.init(NI, d, rs_b))
    assert np.array_equal(rs_a.permutation(20), rs_b.permutation(20))       # the epoch orders follow from the same state
    assert list(baselines.srgnn_shapes(NI, d)) == [n for n, _ in so.shapes(NI, d)]
    assert tuple(baselines.srgnn_shapes(NI, d)) == baselines.SRGNN_PARAMS
    s = 1.0 / np.sqrt(d)
    assert np.abs(th).max() <= s and np.abs(th).max() > 0.9 * s
    b = _lib.Baselines.__new__(_lib.Baselines)
    b.n_items, b.n_keep = NI, d
    assert b.srgnn_n_params() == th.size
    with pytest.raises(ValueError):
        b._srgnn_params(th[:-1])


def _model(NI=12, d=8, step=2, max_len=4, seed=3):
    m = baselines.SRGNN(embedding=d, step=step, max_len=max_len)
    m.n_items = NI
    m.itemidmap = pd.Series(data=np.arange(NI), index=np.arange(100, 100 + NI))
    m.params = so.pack(_params(NI, d, seed, 1.0)).astype(np.float32)
    return m


def test_predict_next_equals_the_oracle_encoder():
    m = _model()
    p = so.unpack(m.params, m.n_items, m.embedding)
    ids = np.arange(100, 112)
    seq = [3, 5, 5, 0, 11, 3, 7]
    for t, x in enumerate(seq):
        got = m.predict_next('s', 100 + x, ids).values
        want = p['E'] @ so.encode(p, seq[:t + 1], m.step, m.max_len)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


class OracleSrgnn(object):
    """_lib.Baselines for kind 'srgnn' on the float64 oracle (parameters kept as float32, as the device keeps them)"""

    def __init__(self, kind, n_items, n_keep, device=0):
        assert kind == 'srgnn'
        self.n_items, self.n_keep = n_items, n_keep

    def srgnn_begin(self, step, max_len, batch_size, session_offsets, items, params):
        self.step, self.L, self.bs = step, max_len, batch_size
        sessions = [list(items[session_offsets[k]:session_offsets[k + 1]]) for k in range(len(session_offsets) - 1)]
        self.samples = so.samples(sessions, max_len)
        self.th = np.asarray(params, np.float32).copy()
        self.m = np.zeros(self.th.size)
        self.v = np.zeros(self.th.size)
        self.t = 0

    def _p(self):
        return so.unpack(self.th, self.n_items, self.n_keep)

    def srgnn_epoch(self, order, lr, l2):
        losses = []
        for b0 in range(0, len(order), self.bs):
            loss, g = so.loss_and_grads(self._p(), [self.samples[k] for k in order[b0:b0 + self.bs]], self.step)
            self.t += 1
            th = self.th.astype(np.float64)
            th, self.m, self.v = so.adam(th, so.pack(g) + l2 * th, self.m, self.v, self.t, lr)
            self.th = th.astype(np.float32)
            losses.append(loss)
        return np.array(losses, np.float32), 0.0

    def srgnn_export(self):
        return self.th.copy()

    def srgnn_import(self, step, max_len, params):
        self.step, self.L, self.th = step, max_len, np.asarray(params, np.float32).copy()

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        p = self._p()
        qs = so.encode_events(p, np.asarray(items), offsets, n_history, self.step, self.L).astype(np.float32)
        cnt, ti, ts = so.rank_events(p['E'], qs, items, offsets, n_history, ('standard', 'conservative', 'median', 'tiebreaking')[mode], cand,
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
    monkeypatch.setattr(_lib, 'Baselines', OracleSrgnn)


def _frame(n_sessions, n_items, seed, max_len=9):
    rs = np.random.RandomState(seed)
    rows = []
    for s in range(n_sessions):
        for t in range(rs.randint(1, max_len)):
            rows.append((s, 1000 + rs.randint(n_items), float(s * 100 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


_KW = dict(embedding=4, step=2, n_epochs=3, batch_size=9, learning_rate=0.01, lr_decay=0.5, lr_decay_step=2, l2=1e-3, max_len=3, seed=1)


@pytest.fixture
def fitted(double):
    train = _frame(30, 15, 0)
    m = baselines.SRGNN(**_KW)
    m.fit(train)
    return m, train


def test_fit_prints_epochs_and_matches_the_oracle(double, capsys):
    train = _frame(30, 15, 0)
    m = baselines.SRGNN(**_KW)
    capsys.readouterr()
    m.fit(train)
    lines = capsys.readouterr().out.split('\n')
    assert len(m.fit_stats) == 3 and all(np.isfinite(s[0]) for s in m.fit_stats)
    assert lines[:3] == ['%d %s' % (e, m.fit_stats[e][0]) for e in range(3)]
    assert m.learning_rates() == [float(np.float32(0.01)), float(np.float32(0.01)), float(np.float32(0.005))]
    off, items = m.sessions(train)
    smp = so.samples([list(items[off[k]:off[k + 1]]) for k in range(len(off) - 1)], 3)
    th0, orders = so.plan(m.n_items, 4, len(smp), 1, 3)
    th, _ = so.train(th0, m.n_items, 4, 2, smp, orders, 9, m.learning_rates(), 1e-3)
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
        want = p['E'] @ so.encode(p, [m.itemidmap[x] for x in seq[:t + 1]], m.step, m.max_len)
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


@pytest.mark.parametrize('bad', [dict(embedding=0), dict(embedding=1025), dict(embedding=2.5), dict(step=0), dict(step=9), dict(max_len=0),
                                 dict(max_len=513), dict(learning_rate=0.0), dict(learning_rate=float('inf')), dict(lr_decay=0.0),
                                 dict(lr_decay_step=0), dict(l2=-1e-5), dict(l2=float('nan')), dict(batch_size=0), dict(n_epochs=-1),
                                 dict(embedding=1024, step=8, max_len=512, batch_size=200), dict(lr_decay=1e-30, n_epochs=8, lr_decay_step=1)])
def test_bad_arguments_are_refused_before_any_device_work(monkeypatch, bad):
    def no_device(*a, **k):
        raise AssertionError('device work')
    monkeypatch.setattr(_lib, 'Baselines', no_device)
    with pytest.raises(ValueError):
        baselines.SRGNN(**bad).fit(_frame(5, 4, 0))


def test_exports_and_kind():
    for name in ('g4r_bl_srgnn_begin', 'g4r_bl_srgnn_epoch', 'g4r_bl_srgnn_grads', 'g4r_bl_srgnn_export', 'g4r_bl_srgnn_import',
                 'g4r_bl_srgnn_encode'):
        assert name in _lib.EXPORTS
    assert _lib.BASELINE_KINDS['srgnn'] == 15
    with open(os.path.join(ROOT, 'include', 'g4r.h')) as f:
        assert '#define G4R_BL_SRGNN 15' in f.read()
    import baselines as shim
    assert shim.SRGNN is baselines.SRGNN


def test_run_py_baseline_srgnn(double, tmp_path, capsys):
    import run
    train, test = _frame(30, 10, 0), _frame(8, 10, 1)
    test = test[test.ItemId.isin(train.ItemId.unique())]
    tr, te = tmp_path / 'train.tsv', tmp_path / 'test.tsv'
    train.to_csv(tr, sep='\t', index=False)
    test.to_csv(te, sep='\t', index=False)
    run.main([str(tr), '--baseline', 'srgnn', '-ps', 'embedding=4,step=2,n_epochs=2,batch_size=5,max_len=3,l2=0.001', '-t', str(te), '-m', '5'])
    out = capsys.readouterr().out
    assert 'Creating SRGNN model' in out and 'Recall@5' in out and '\n1 ' in out
    with pytest.raises(SystemExit):
        run.main([str(tr), '--baseline', 'srgnn', '--rest_of_session', '-t', str(te)])


SRC = r'''
#include <math.h>
#include <stdio.h>
#include <stddef.h>
#include "g4r.h"
int main(void) {
  g4r_baselines* h = NULL;
  g4r_baselines* nm = NULL;
  /* 10 items, d 4: n_params = 40 + 15 * 16 + 14 * 4 = 336; sessions {1,2,3,4} and {5,6}: samples 0 .. 3 */
  float th[336], bad[336], g[336], q[12], loss = 0.f, ms = 0.f, ls[2];
  const int64_t so[3] = {0, 4, 6}, so_bad[3] = {0, 5, 4}, so1[2] = {0, 4};
  const int32_t it[6] = {1, 2, 3, 4, 5, 6}, it_bad[6] = {1, 2, 3, 4, 5, 10}, order[2] = {0, 3}, order3[3] = {0, 1, 2}, oob[1] = {4};
  int rc, i;
  for (i = 0; i < 336; i++) { th[i] = 0.01f * (float)(i % 7); bad[i] = th[i]; }
  bad[5] = NAN;
  if (g4r_bl_create(14, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 2;
  if (g4r_bl_create(16, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 3;
  if (g4r_bl_create(G4R_BL_SRGNN, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  rc = g4r_bl_create(G4R_BL_SRGNN, 10, 4, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 5;
  if (g4r_bl_srgnn_export(h, th, 336) != G4R_ERR_STATE) return 6;
  if (g4r_bl_srgnn_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 7;
  if (g4r_bl_srgnn_epoch(h, order, 2, 0.001f, 0.f, ls, &ms) != G4R_ERR_STATE) return 8;
  if (g4r_bl_srgnn_begin(h, 0, 3, 2, so, 2, it, 6, th, 336) != G4R_ERR_INVALID) return 9;
  if (g4r_bl_srgnn_begin(h, 9, 3, 2, so, 2, it, 6, th, 336) != G4R_ERR_INVALID) return 10;
  if (g4r_bl_srgnn_begin(h, 1, 0, 2, so, 2, it, 6, th, 336) != G4R_ERR_INVALID) return 11;
  if (g4r_bl_srgnn_begin(h, 1, 513, 2, so, 2, it, 6, th, 336) != G4R_ERR_INVALID) return 12;
  if (g4r_bl_srgnn_begin(h, 1, 3, 2, so, 2, it, 6, th, 335) != G4R_ERR_INVALID) return 13;
  if (g4r_bl_srgnn_begin(h, 1, 3, 2, so, 2, it, 6, bad, 336) != G4R_ERR_INVALID) return 14;
  if (g4r_bl_srgnn_begin(h, 1, 3, 2, so, 2, it_bad, 6, th, 336) != G4R_ERR_INDEX) return 15;
  if (g4r_bl_srgnn_begin(h, 1, 3, 2, so_bad, 2, it, 6, th, 336) != G4R_ERR_INVALID) return 16;
  if (g4r_bl_srgnn_begin(h, 1, 3, 0, so, 2, it, 6, th, 336) != G4R_ERR_INVALID) return 17;
  if (g4r_bl_srgnn_begin(h, 8, 512, 100000, so, 2, it, 6, th, 336) != G4R_ERR_INVALID) return 18;   /* flat indices past 2^31 */
  if (g4r_bl_srgnn_export(h, th, 336) != G4R_ERR_STATE) return 19;                                   /* nothing was set */
  if (g4r_bl_srgnn_begin(h, 2, 3, 2, so, 2, it, 6, th, 336) != G4R_OK) return 20;
  if (g4r_bl_srgnn_epoch(h, oob, 1, 0.001f, 0.f, ls, &ms) != G4R_ERR_INDEX) return 21;
  if (g4r_bl_srgnn_epoch(h, order, 2, 0.f, 0.f, ls, &ms) != G4R_ERR_INVALID) return 22;
  if (g4r_bl_srgnn_epoch(h, order, 2, 0.001f, -1.f, ls, &ms) != G4R_ERR_INVALID) return 23;
  if (g4r_bl_srgnn_grads(h, order3, 3, &loss, g) != G4R_ERR_INVALID) return 24;                     /* n > batch_size */
  if (g4r_bl_srgnn_grads(h, order, 2, &loss, g) != G4R_OK || !(loss > 0.f)) return 25;
  if (g4r_bl_srgnn_epoch(h, order, 2, 0.001f, 1e-5f, ls, &ms) != G4R_OK) return 26;
  if (g4r_bl_srgnn_encode(h, it, 4, so1, 1, NULL, q, 1) != G4R_ERR_INVALID) return 27;              /* n_q must be 3 */
  if (g4r_bl_srgnn_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_OK) return 28;
  /* the other kinds' calls refuse an SR-GNN handle, and SR-GNN's refuse a NARM handle */
  if (g4r_bl_narm_import(h, 4, 3, th, 336) != G4R_ERR_STATE) return 29;
  if (g4r_bl_sasrec_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 30;
  if (g4r_bl_narm_epoch(h, order, 2, 1, 0.001f, 0.f, 0.f, ls, &ms) != G4R_ERR_STATE) return 31;
  if (g4r_bl_bpr_import(h, NULL, NULL) != G4R_ERR_STATE) return 32;
  if (g4r_bl_create(G4R_BL_NARM, 10, 4, 0, &nm) != G4R_OK) return 33;
  if (g4r_bl_srgnn_import(nm, 1, 3, th, 336) != G4R_ERR_STATE) return 34;
  if (g4r_bl_srgnn_export(nm, th, 336) != G4R_ERR_STATE) return 35;
  if (g4r_bl_srgnn_encode(nm, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 36;
  if (g4r_bl_srgnn_begin(nm, 1, 3, 2, so, 2, it, 6, th, 336) != G4R_ERR_STATE) return 37;
  if (g4r_bl_destroy(nm) != G4R_OK) return 38;
  if (g4r_bl_srgnn_import(h, 1, 3, bad, 336) != G4R_ERR_INVALID) return 39;
  if (g4r_bl_last_error(h)[0] == 0) return 40;
  if (g4r_bl_destroy(h) != G4R_OK) return 41;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_srgnn_abi(tmp_path):
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
