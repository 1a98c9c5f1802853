"""STAMP (DESIGN §3v) without a GPU: the float64 oracle's backward against central differences (n = 1, repeated items, a target
that is also an input), the samples, the init layout, the package's host encoder and predict_next against the oracle, the class's
fit, evaluation surface, pickles and run.py through a CPU double of _lib.Baselines backed by the oracle, the refusals before any
device work, the exports and a C99 caller of kind 17."""
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

import stamp_oracle as sto  # noqa: E402
from gru4rec_b200 import _lib, baselines, evaluation  # noqa: E402

# n = 1, repeated items, a target that is also an input, a prefix of one item repeated
BATCH = [([1, 2, 1, 3, 3, 2], 4), ([5], 6), ([0, 0], 0), ([2, 4, 2, 4, 6], 2), ([3, 3, 3], 3)]


def _params(NI, d, seed=0, scale=1.0):
    rs = np.random.RandomState(seed)
    th = sto.init(NI, d, 0.7, rs).astype(np.float64)
    p = sto.unpack(th, NI, d)
    for name in sto.BIASES:                      # non-zero biases, so that their gradients reach every term
        p[name] = rs.normal(0.0, 0.3, size=p[name].shape)
    return {k: v * scale for k, v in p.items()}


def _loss(p, batch):
    return sto.loss_and_grads(p, batch)[0]


@pytest.mark.parametrize('d', [1, 3])
def test_oracle_backward_matches_central_differences(d):
    NI = 7
    p = _params(NI, d, d)
    _, g = sto.loss_and_grads(p, BATCH)
    th, gf = sto.pack(p), sto.pack(g)
    assert np.abs(gf).max() > 1e-3
    for i in range(th.size):
        a, b = th.copy(), th.copy()
        a[i] += 1e-6
        b[i] -= 1e-6
        fd = (_loss(sto.unpack(a, NI, d), BATCH) - _loss(sto.unpack(b, NI, d), BATCH)) / 2e-6
        assert abs(fd - gf[i]) <= 1e-4 * abs(fd) + 1e-7, (i, fd, gf[i])


def test_magnitude_bound_dominates_the_gradient():
    p = _params(9, 5, 1, 2.0)
    _, g = sto.loss_and_grads(p, BATCH)
    _, m = sto.loss_and_grads(p, BATCH, mag=True)
    assert (np.abs(sto.pack(g)) <= sto.pack(m) * (1 + 1e-9) + 1e-300).all()


def test_one_input_takes_it_as_mean_and_last_click():
    p = _params(6, 4, 2)
    c, q = sto.forward(p, [3])
    np.testing.assert_array_equal(c['ms'], p['E'][3])
    np.testing.assert_array_equal(c['mt'], p['E'][3])
    np.testing.assert_allclose(q, baselines.stamp_encode(p, [3]), rtol=1e-13, atol=1e-15)


def test_attention_is_not_normalised_and_follows_the_definition():
    p = _params(8, 3, 4)
    x = [2, 5, 2, 7]
    X = p['E'][x]
    ms, mt = X.mean(axis=0), X[-1]
    a = np.array([p['w0'] @ (1.0 / (1.0 + np.exp(-(xi @ p['W1'] + mt @ p['W2'] + ms @ p['W3'] + p['b_a'])))) for xi in X])
    q = np.tanh((a @ X) @ p['Ws'] + p['bs']) * np.tanh(mt @ p['Wt'] + p['bt'])
    c, q0 = sto.forward(p, x)
    np.testing.assert_allclose(c['a'], a, rtol=1e-13)
    assert abs(a.sum() - 1.0) > 1e-3
    np.testing.assert_allclose(q0, q, rtol=1e-12)
    np.testing.assert_allclose(baselines.stamp_encode(p, x), q, rtol=1e-12)


@pytest.mark.parametrize('max_len', [1, 2, 5])
def test_samples_cover_every_pair_once_within_a_window_of_max_len(max_len):
    rs = np.random.RandomState(max_len)
    lens = [1, 2, max_len, max_len + 1, max_len + 2, 2 * max_len + 3, 1, 7]
    sessions = [list(rs.randint(0, 20, n)) for n in lens]
    smp = sto.samples(sessions, max_len)
    assert sorted((tuple(x), y) for x, y in smp) == sorted((tuple(s[max(0, j - max_len):j]), s[j]) for s in sessions for j in range(1, len(s)))
    assert len(smp) == sum(n - 1 for n in lens) and all(1 <= len(x) <= max_len for x, _ in smp)
    frame = pd.DataFrame([(s, 100 + it, float(t)) for s, seq in enumerate(sessions) for t, it in enumerate(seq)], columns=['SessionId', 'ItemId', 'Time'])
    m = baselines.STAMP(max_len=max_len)
    off, items = m.sessions(frame.sample(frac=1.0, random_state=0))        # rows in any order: events by time
    ids = m.itemidmap.index.values
    got = sorted([int(ids[i]) - 100 for i in items[off[k]:off[k + 1]]] for k in range(len(off) - 1))
    assert got == sorted(sessions)


def test_init_layout_and_n_params():
    NI, d = 13, 6
    rs_a, rs_b = np.random.RandomState(5), np.random.RandomState(5)
    th = baselines.stamp_init(NI, d, 0.05, rs_a)
    assert th.dtype == np.float32 and th.size == NI * d + 5 * d * d + 4 * d == sto.n_params(NI, d)
    np.testing.assert_array_equal(th, sto.init(NI, d, 0.05, rs_b))
    assert np.array_equal(rs_a.permutation(20), rs_b.permutation(20))       # the epoch orders follow from the same state
    assert list(baselines.stamp_shapes(NI, d)) == [n for n, _ in sto.shapes(NI, d)]
    assert tuple(baselines.stamp_shapes(NI, d)) == baselines.STAMP_PARAMS
    p = baselines.stamp_unpack(th, NI, d)
    for name in baselines.STAMP_PARAMS:
        if name in baselines.STAMP_BIASES:
            assert not p[name].any(), name
        else:
            assert p[name].std() > 0.02 and abs(p[name].mean()) < 0.03, name
    # the draws run in layout order with no draw for a bias: E first, then W1, W2, W3, w0, Ws, Wt
    rs = np.random.RandomState(5)
    np.testing.assert_array_equal(p['E'], rs.normal(0.0, 0.05, size=(NI, d)).astype(np.float32))
    for name in ('W1', 'W2', 'W3', 'w0', 'Ws', 'Wt'):
        np.testing.assert_array_equal(p[name], rs.normal(0.0, 0.05, size=p[name].shape).astype(np.float32))
    b = _lib.Baselines.__new__(_lib.Baselines)
    b.n_items, b.n_keep = NI, d
    assert b.stamp_n_params() == th.size
    with pytest.raises(ValueError):
        b._stamp_params(th[:-1])


def _model(NI=12, d=8, max_len=4, seed=3):
    m = baselines.STAMP(embedding=d, max_len=max_len)
    m.n_items = NI
    m.itemidmap = pd.Series(data=np.arange(NI), index=np.arange(100, 100 + NI))
    m.params = sto.pack(_params(NI, d, seed)).astype(np.float32)
    return m


def test_predict_next_equals_the_oracle_encoder():
    m = _model()
    p = sto.unpack(m.params, m.n_items, m.embedding)
    ids = np.arange(100, 112)
    seq = [3, 5, 5, 0, 11, 3, 7]
    for t, x in enumerate(seq):
        got = m.predict_next('s', 100 + x, ids).values
        want = p['E'] @ sto.encode(p, seq[:t + 1], m.max_len)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


class OracleStamp(object):
    """_lib.Baselines for kind 'stamp' on the float64 oracle (parameters kept as float32, as the device keeps them)"""

    def __init__(self, kind, n_items, n_keep, device=0):
        assert kind == 'stamp'
        self.n_items, self.n_keep = n_items, n_keep

    def stamp_begin(self, max_len, batch_size, session_offsets, items, params):
        self.L, self.bs = max_len, batch_size
        sessions = [list(items[session_offsets[k]:session_offsets[k + 1]]) for k in range(len(session_offsets) - 1)]
        self.samples = sto.samples(sessions, max_len)
        self.th = np.asarray(params, np.float32).copy()
        self.m = np.zeros(self.th.size)
        self.v = np.zeros(self.th.size)
        self.t = 0

    def _p(self):
        return sto.unpack(self.th, self.n_items, self.n_keep)

    def stamp_epoch(self, order, lr):
        losses = []
        for b0 in range(0, len(order), self.bs):
            loss, g = sto.loss_and_grads(self._p(), [self.samples[k] for k in order[b0:b0 + self.bs]])
            self.t += 1
            th, self.m, self.v = sto.adam(self.th.astype(np.float64), sto.pack(g), self.m, self.v, self.t, lr)
            self.th = th.astype(np.float32)
            losses.append(loss)
        return np.array(losses, np.float32), 0.0

    def stamp_export(self):
        return self.th.copy()

    def stamp_import(self, max_len, params):
        self.L, self.th = max_len, np.asarray(params, np.float32).copy()

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        p = self._p()
        qs = sto.encode_events(p, np.asarray(items), offsets, n_history, self.L).astype(np.float32)
        cnt, ti, ts = sto.rank_events(p['E'], qs, items, offsets, n_history, ('standard', 'conservative', 'median', 'tiebreaking')[mode], cand,
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
    monkeypatch.setattr(_lib, 'Baselines', OracleStamp)


def _frame(n_sessions, n_items, seed, max_len=9):
    rs = np.random.RandomState(seed)
    rows = []
    for s in range(n_sessions):
        for t in range(rs.randint(1, max_len)):
            rows.append((s, 1000 + rs.randint(n_items), float(s * 100 + t)))
    return pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])


_KW = dict(embedding=4, n_epochs=3, batch_size=9, learning_rate=0.01, init_std=0.3, max_len=3, seed=1)


@pytest.fixture
def fitted(double):
    train = _frame(30, 15, 0)
    m = baselines.STAMP(**_KW)
    m.fit(train)
    return m, train


def test_fit_prints_epochs_and_matches_the_oracle(double, capsys):
    train = _frame(30, 15, 0)
    m = baselines.STAMP(**_KW)
    capsys.readouterr()
    m.fit(train)
    lines = capsys.readouterr().out.split('\n')
    assert len(m.fit_stats) == 3 and all(np.isfinite(s[0]) for s in m.fit_stats)
    assert lines[:3] == ['%d %s' % (e, m.fit_stats[e][0]) for e in range(3)]
    off, items = m.sessions(train)
    smp = sto.samples([list(items[off[k]:off[k + 1]]) for k in range(len(off) - 1)], 3)
    th0, orders = sto.plan(m.n_items, 4, 0.3, len(smp), 1, 3)
    th, _ = sto.train(th0, m.n_items, 4, smp, orders, 9, 0.01)
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
        want = p['E'] @ sto.encode(p, [m.itemidmap[x] for x in seq[:t + 1]], m.max_len)
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


@pytest.mark.parametrize('bad', [dict(embedding=0), dict(embedding=1025), dict(embedding=2.5), dict(max_len=0), dict(max_len=513),
                                 dict(learning_rate=0.0), dict(learning_rate=float('inf')), dict(init_std=0.0), dict(init_std=float('nan')),
                                 dict(batch_size=0), dict(n_epochs=-1), dict(embedding=1024, max_len=512, batch_size=2048)])
def test_bad_arguments_are_refused_before_any_device_work(monkeypatch, bad):
    def no_device(*a, **k):
        raise AssertionError('device work')
    monkeypatch.setattr(_lib, 'Baselines', no_device)
    with pytest.raises(ValueError):
        baselines.STAMP(**bad).fit(_frame(5, 4, 0))


def test_a_training_set_without_a_pair_is_refused(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleStamp)
    frame = pd.DataFrame([(0, 1, 0.0), (1, 2, 1.0)], columns=['SessionId', 'ItemId', 'Time'])
    with pytest.raises(ValueError, match='at least 2 events'):
        baselines.STAMP().fit(frame)


def test_exports_and_kind():
    for name in ('g4r_bl_stamp_begin', 'g4r_bl_stamp_epoch', 'g4r_bl_stamp_grads', 'g4r_bl_stamp_export', 'g4r_bl_stamp_import',
                 'g4r_bl_stamp_encode'):
        assert name in _lib.EXPORTS
    assert _lib.BASELINE_KINDS['stamp'] == 17
    with open(os.path.join(ROOT, 'include', 'g4r.h')) as f:
        assert '#define G4R_BL_STAMP 17' in f.read()
    import baselines as shim
    assert shim.STAMP is baselines.STAMP


def test_run_py_baseline_stamp(double, tmp_path, capsys):
    import run
    train, test = _frame(30, 10, 0), _frame(8, 10, 1)
    test = test[test.ItemId.isin(train.ItemId.unique())]
    tr, te = tmp_path / 'train.tsv', tmp_path / 'test.tsv'
    train.to_csv(tr, sep='\t', index=False)
    test.to_csv(te, sep='\t', index=False)
    run.main([str(tr), '--baseline', 'stamp', '-ps', 'embedding=4,n_epochs=2,batch_size=5,max_len=3,init_std=0.2', '-t', str(te), '-m', '5'])
    out = capsys.readouterr().out
    assert 'Creating STAMP model' in out and 'Recall@5' in out and '\n1 ' in out
    with pytest.raises(SystemExit):
        run.main([str(tr), '--baseline', 'stamp', '--rest_of_session', '-t', str(te)])


SRC = r'''
#include <math.h>
#include <stdio.h>
#include <stddef.h>
#include "g4r.h"
int main(void) {
  g4r_baselines* h = NULL;
  g4r_baselines* nm = NULL;
  /* 10 items, d 4: n_params = 40 + 5 * 16 + 4 * 4 = 136; sessions {1,2,3,4} and {5,6}: samples 0 .. 3 */
  float th[136], bad[136], g[136], q[12], loss = 0.f, ms = 0.f, ls[2];
  const int64_t so[3] = {0, 4, 6}, so_bad[3] = {0, 5, 4}, so1[2] = {0, 4};
  const int32_t it[6] = {1, 2, 3, 4, 5, 6}, it_bad[6] = {1, 2, 3, 4, 5, 10}, order[2] = {0, 3}, order3[3] = {0, 1, 2}, oob[1] = {4};
  int rc, i;
  for (i = 0; i < 136; i++) { th[i] = 0.01f * (float)(i % 7); bad[i] = th[i]; }
  bad[5] = NAN;
  if (g4r_bl_create(14, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 2;
  if (g4r_bl_create(16, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 3;
  if (g4r_bl_create(18, 10, 4, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  if (g4r_bl_create(G4R_BL_STAMP, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 5;
  rc = g4r_bl_create(G4R_BL_STAMP, 10, 4, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 6;
  if (g4r_bl_stamp_export(h, th, 136) != G4R_ERR_STATE) return 7;
  if (g4r_bl_stamp_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 8;
  if (g4r_bl_stamp_epoch(h, order, 2, 0.001f, ls, &ms) != G4R_ERR_STATE) return 9;
  if (g4r_bl_stamp_begin(h, 0, 2, so, 2, it, 6, th, 136) != G4R_ERR_INVALID) return 10;
  if (g4r_bl_stamp_begin(h, 513, 2, so, 2, it, 6, th, 136) != G4R_ERR_INVALID) return 11;
  if (g4r_bl_stamp_begin(h, 3, 2, so, 2, it, 6, th, 135) != G4R_ERR_INVALID) return 12;
  if (g4r_bl_stamp_begin(h, 3, 2, so, 2, it, 6, bad, 136) != G4R_ERR_INVALID) return 13;
  if (g4r_bl_stamp_begin(h, 3, 2, so, 2, it_bad, 6, th, 136) != G4R_ERR_INDEX) return 14;
  if (g4r_bl_stamp_begin(h, 3, 2, so_bad, 2, it, 6, th, 136) != G4R_ERR_INVALID) return 15;
  if (g4r_bl_stamp_begin(h, 3, 0, so, 2, it, 6, th, 136) != G4R_ERR_INVALID) return 16;
  if (g4r_bl_stamp_begin(h, 512, 600000, so, 2, it, 6, th, 136) != G4R_ERR_INVALID) return 17;   /* flat indices past 2^31 */
  if (g4r_bl_stamp_export(h, th, 136) != G4R_ERR_STATE) return 18;                                /* nothing was set */
  if (g4r_bl_stamp_begin(h, 3, 2, so, 2, it, 6, th, 136) != G4R_OK) return 19;
  if (g4r_bl_stamp_epoch(h, oob, 1, 0.001f, ls, &ms) != G4R_ERR_INDEX) return 20;
  if (g4r_bl_stamp_epoch(h, order, 2, 0.f, ls, &ms) != G4R_ERR_INVALID) return 21;
  if (g4r_bl_stamp_grads(h, order3, 3, &loss, g) != G4R_ERR_INVALID) return 22;                  /* n > batch_size */
  if (g4r_bl_stamp_grads(h, order, 2, &loss, g) != G4R_OK || !(loss > 0.f)) return 23;
  if (g4r_bl_stamp_epoch(h, order, 2, 0.001f, ls, &ms) != G4R_OK) return 24;
  if (g4r_bl_stamp_encode(h, it, 4, so1, 1, NULL, q, 1) != G4R_ERR_INVALID) return 25;           /* n_q must be 3 */
  if (g4r_bl_stamp_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_OK) return 26;
  /* the other kinds' calls refuse a STAMP handle, and STAMP's refuse a NARM handle */
  if (g4r_bl_narm_import(h, 4, 3, th, 136) != G4R_ERR_STATE) return 27;
  if (g4r_bl_srgnn_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 28;
  if (g4r_bl_srgnn_epoch(h, order, 2, 0.001f, 0.f, ls, &ms) != G4R_ERR_STATE) return 29;
  if (g4r_bl_sasrec_encode(h, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 30;
  if (g4r_bl_bpr_import(h, NULL, NULL) != G4R_ERR_STATE) return 31;
  if (g4r_bl_create(G4R_BL_NARM, 10, 4, 0, &nm) != G4R_OK) return 32;
  if (g4r_bl_stamp_import(nm, 3, th, 136) != G4R_ERR_STATE) return 33;
  if (g4r_bl_stamp_export(nm, th, 136) != G4R_ERR_STATE) return 34;
  if (g4r_bl_stamp_encode(nm, it, 4, so1, 1, NULL, q, 3) != G4R_ERR_STATE) return 35;
  if (g4r_bl_stamp_begin(nm, 3, 2, so, 2, it, 6, th, 136) != G4R_ERR_STATE) return 36;
  if (g4r_bl_destroy(nm) != G4R_OK) return 37;
  if (g4r_bl_stamp_import(h, 3, bad, 136) != G4R_ERR_INVALID) return 38;
  if (g4r_bl_last_error(h)[0] == 0) return 39;
  if (g4r_bl_destroy(h) != G4R_OK) return 40;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_stamp_abi(tmp_path):
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
