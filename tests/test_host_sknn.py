"""CPU tests of session-based kNN (DESIGN §3o): oracle/sknn_oracle.py against hand-computed values, baselines.SessionKNN's fit and
predict_next against the oracle on messy data, and the Python surface -- evaluate_gpu / evaluate_events, pickles, run.py
--baseline sknn -- on a CPU double of _lib.Baselines backed by the oracle.  Parameter refusals, the binding's checks and the C ABI
from a C99 caller at the end.  The device path is tested in test_gpu_sknn.py."""
import contextlib
import io
import os
import pickle
import shutil
import subprocess

import numpy as np
import pandas as pd
import pytest

import baselines_oracle as bo
import sknn_oracle as sko
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
from test_host_baselines import OracleBaselines

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class OracleSknn(OracleBaselines):
    """_lib.Baselines('sknn', ...) on the host: the oracle's index and ranking behind the binding's methods"""

    def sknn_fit(self, session_offsets, items, recency, sample_size, similarity):
        off = np.asarray(session_offsets)
        sess = np.repeat(np.arange(len(off) - 1), np.diff(off))
        self.index = sko.Index(sess, np.asarray(items), -np.repeat(np.asarray(recency), np.diff(off)), self.n_items)
        self.sample, self.sim = sample_size, similarity

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        name = [m for m, v in bo.MODES.items() if v == mode][0]
        cnt, ti, ts = sko.rank_events(self.index, self.n_keep, self.sample, self.sim, items, offsets, n_history, name, cand, exclude_seen, k)
        rec, mrr = bo.sums(cnt, name, cut_off)
        return np.array(rec), np.array(mrr), len(cnt), cnt.astype(np.int32) if counts else None, ti, ts


@pytest.fixture
def double(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleSknn)


def _index(rows, n_items):
    """rows: (session, item index, time)"""
    s, i, t = zip(*rows)
    return sko.Index(np.array(s), np.array(i), np.array(t, dtype=np.float64), n_items)


# A = {0, 1} T 11; B = {1, 2} T 20; C = {0, 2, 3} T 20 (after B in the data); D = {3} T 5.  Recency: B, C, A, D.
TINY = [('A', 0, 10), ('A', 1, 11), ('B', 1, 20), ('B', 2, 19), ('C', 0, 20), ('C', 2, 3), ('C', 3, 4), ('D', 3, 5)]


def test_oracle_recency_and_sample_truncation_among_equal_times():
    ix = _index(TINY, 4)
    assert list(ix.rank) == [2, 0, 1, 3]                                  # sessions A, B, C, D by first appearance
    r, v = sko.neighbours(ix, [1, 0], 5, 1, 'cosine')                     # B and C tie on T: B appeared first
    assert list(r) == [0]
    r, v = sko.neighbours(ix, [1, 0], 5, 2, 'cosine')
    assert list(r) == [0, 1]


def test_oracle_cosine_by_hand():
    ix = _index(TINY, 4)
    r, v = sko.neighbours(ix, [0, 1, 0], 2, 3, 'cosine')                 # I(c) = {0, 1}; candidates B, C, A
    assert list(r) == [2, 0] and list(v) == [2 / np.sqrt(4.0), 1 / np.sqrt(4.0)]
    s = sko.scores(ix, [0, 1, 0], 2, 3, 'cosine')
    assert list(s) == [1.0, 1.5, 0.5, 0.0]


def test_oracle_vector_by_hand_last_occurrence_weighs():
    ix = _index(TINY, 4)
    # c = (0, 1, 0): item 1 last at 2 (2/3), item 0 last at 3 (1, not 1/3); A shares both: 2/3 + 1 in position order
    r, v = sko.neighbours(ix, [0, 1, 0], 2, 3, 'vector')
    assert list(r) == [2, 1] and list(v) == [2 / 3 + 1.0, 1.0]
    s = sko.scores(ix, [0, 1, 0], 2, 3, 'vector')
    assert list(s) == [(2 / 3 + 1.0) + 1.0, 2 / 3 + 1.0, 1.0, 1.0]


def test_oracle_neighbour_ties_go_to_the_more_recent():
    ix = _index(TINY, 4)
    r, v = sko.neighbours(ix, [1], 1, 4, 'cosine')                        # A and B both 1 / sqrt(2): B is more recent
    assert list(r) == [0] and v[0] == 1 / np.sqrt(2.0)
    assert list(sko.scores(ix, [1], 1, 4, 'cosine')) == [0.0, v[0], v[0], 0.0]


def test_oracle_sums_in_neighbour_order():
    # c = (0, 1, 2): s1 = {0, 1, 2} (1.0), s2 = {0, 1, 2, 3} (3 / sqrt(12)), s3 = {0, 1} (2 / sqrt(6)); item 0 is in all three
    rows = [('s3', 0, 1), ('s3', 1, 1), ('s1', 0, 3), ('s1', 1, 3), ('s1', 2, 3), ('s2', 0, 2), ('s2', 1, 2), ('s2', 2, 2), ('s2', 3, 2)]
    ix = _index(rows, 4)
    a, b, c = 1.0, 3 / np.sqrt(12.0), 2 / np.sqrt(6.0)
    assert (a + b) + c != (c + b) + a
    r, v = sko.neighbours(ix, [0, 1, 2], 3, 10, 'cosine')
    assert list(v) == [a, b, c]
    assert sko.scores(ix, [0, 1, 2], 3, 10, 'cosine')[0] == (a + b) + c


def _messy_train(seed=3, n_items=50, n_events=1500):
    rs = np.random.RandomState(seed)
    df = make_sessions(n_items=n_items, n_events=n_events, seed=seed, item_as_str=True)
    rep = np.flatnonzero(rs.rand(len(df)) < 0.2)
    rep = rep[(rep > 0) & (df.SessionId.values[rep] == df.SessionId.values[np.maximum(rep - 1, 0)])]
    df.loc[rep, 'ItemId'] = df.ItemId.values[rep - 1]                    # repeated items
    df['Time'] = np.floor(df.Time.values / 300.0)                          # many equal session times
    df['SessionId'] = 's' + (df.SessionId * 7919 % 10007).astype(str)      # string ids, not in time order
    return df.sample(frac=1.0, random_state=seed).reset_index(drop=True)   # unsorted rows


@pytest.mark.parametrize('similarity', ['cosine', 'vector'])
def test_fit_and_predict_next_equal_the_oracle(double, similarity):
    import baselines
    tr = _messy_train()
    m = baselines.SessionKNN(k=7, sample_size=40, similarity=similarity)
    m.fit(tr)
    ix = sko.Index(tr.SessionId.values, m.itemidmap[tr.ItemId.values].values, tr.Time.values, m.n_items)
    off, items, rank = ix.csr()
    np.testing.assert_array_equal(m.session_offsets, off)
    np.testing.assert_array_equal(m.session_items, items)
    np.testing.assert_array_equal(m.recency, rank)
    assert m.n_sessions == len(rank) and list(m.itemidmap.index) == list(pd.unique(tr.ItemId.values))
    ids = m.itemidmap.index.values
    rs = np.random.RandomState(1)
    for sid in ('t1', 't2'):
        prefix = []
        for x in ids[rs.randint(0, len(ids), 6)].tolist() + [ids[0], ids[0]]:
            prefix.append(m.itemidmap[x])
            got = m.predict_next(sid, x, ids)
            want = sko.scores(ix, prefix, 7, 40, similarity)
            assert list(got.index) == list(ids)
            np.testing.assert_array_equal(got.values, want)
    assert m.current_session == 't2'


@pytest.fixture(scope='module')
def fitted():
    import baselines
    mp_ = pytest.MonkeyPatch()
    mp_.setattr(_lib, 'Baselines', OracleSknn)
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    models = {s: baselines.SessionKNN(k=6, sample_size=30, similarity=s) for s in ('cosine', 'vector')}
    for m in models.values():
        m.fit(train.copy())
    mp_.undo()
    return models, train


def _test_frame(seed):
    rs = np.random.RandomState(seed)
    te = make_sessions(n_items=60, n_events=300, seed=seed + 1)
    te['SessionId'] += 10000
    te.loc[rs.rand(len(te)) < 0.05, 'ItemId'] = 999999                     # unknown: dropped
    rep = np.flatnonzero(rs.rand(len(te)) < 0.2)
    rep = rep[(rep > 0) & (te.SessionId.values[rep] == te.SessionId.values[np.maximum(rep - 1, 0)])]
    te.loc[rep, 'ItemId'] = te.ItemId.values[rep - 1]
    return te.sample(frac=1.0, random_state=seed).reset_index(drop=True)


def _sorted(model, te):
    df = pd.merge(te, pd.DataFrame({'ItemIdx': model.itemidmap.values, 'ItemId': model.itemidmap.index}), on='ItemId', how='inner')
    df = df.sort_values(['SessionId', 'Time', 'ItemId']).reset_index(drop=True)
    off = np.zeros(df.SessionId.nunique() + 1, np.int64)
    off[1:] = df.groupby('SessionId', sort=True).size().cumsum()
    return df, off


def _oracle(m, train):
    return sko.Index(train.SessionId.values, m.itemidmap[train.ItemId.values].values, train.Time.values, m.n_items)


@pytest.mark.parametrize('similarity', ['cosine', 'vector'])
@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_evaluate_events_frame_ranks_and_sums(double, fitted, similarity, mode):
    import evaluation
    models, train = fitted
    m = models[similarity]
    te = _test_frame(seed=11)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(m, te.copy(), cut_off=[1, 5, 20], mode=mode, k=4)
        rec, mrr = evaluation.evaluate_gpu(m, te.copy(), cut_off=[1, 5, 20], mode=mode)
    df, off = _sorted(m, te)
    ev = res['events']
    assert len(ev) == len(df) - (len(off) - 1)
    cnt, ti, ts = sko.rank_events(_oracle(m, train), 6, 30, similarity, df.ItemIdx.values, off, None, mode, None, False, 4)
    np.testing.assert_array_equal(ev['rank'].values, bo.ranks(cnt, mode))
    np.testing.assert_array_equal(res['topk_items'], m.itemidmap.index.values[ti])
    np.testing.assert_array_equal(res['topk_scores'], ts)
    assert res['recall'] == rec and res['mrr'] == mrr


@pytest.mark.parametrize('similarity', ['cosine', 'vector'])
def test_items_exclude_seen_history_and_lists(double, fitted, similarity):
    import evaluation
    models, train = fitted
    m = models[similarity]
    ix = _oracle(m, train)
    te = _test_frame(seed=5)
    ids = m.itemidmap.index.values
    cand = list(ids[::3]) + [ids[0], ids[0]]                               # duplicates count
    df, off = _sorted(m, te)
    with contextlib.redirect_stdout(io.StringIO()):
        a = evaluation.evaluate_events(m, te.copy(), items=cand, cut_off=[3, 10], mode='conservative', k=3)
        b = evaluation.evaluate_events(m, te.copy(), cut_off=[5], exclude_seen=True, k=5)
    cnt, ti, ts = sko.rank_events(ix, 6, 30, similarity, df.ItemIdx.values, off, None, 'conservative', m.itemidmap[cand].values, k=3)
    np.testing.assert_array_equal(a['events']['rank'].values, bo.ranks(cnt, 'conservative'))
    np.testing.assert_array_equal(a['topk_scores'], ts)
    cnt, ti, ts = sko.rank_events(ix, 6, 30, similarity, df.ItemIdx.values, off, None, 'standard', None, True, k=5)
    np.testing.assert_array_equal(b['events']['rank'].values, bo.ranks(cnt, 'standard'))
    np.testing.assert_array_equal(b['topk_items'], m.itemidmap.index.values[ti])
    assert np.isinf(b['events']['rank'].values).any()
    pos, size = df.groupby('SessionId').cumcount(), df.groupby('SessionId').SessionId.transform('size')
    hist = df[pos < size // 2][['SessionId', 'ItemId', 'Time']]
    rest = df.drop(hist.index)[['SessionId', 'ItemId', 'Time']]
    with contextlib.redirect_stdout(io.StringIO()):
        h = evaluation.evaluate_events(m, rest.copy(), cut_off=[5], history=hist.copy())
    sids = np.sort(rest.SessionId.unique())
    both = pd.concat([df[df.index.isin(hist.index)], df[~df.index.isin(hist.index)]]).sort_values('SessionId', kind='stable')
    both = both[both.SessionId.isin(sids)]
    nh = hist.groupby('SessionId').size().reindex(sids, fill_value=0).values
    boff = np.r_[0, np.cumsum(both.groupby('SessionId').size().values)]
    cnt = sko.rank_events(ix, 6, 30, similarity, both.ItemIdx.values, boff, nh)[0]
    np.testing.assert_array_equal(h['events']['rank'].values, bo.ranks(cnt, 'standard'))


def test_pickle_round_trip_without_the_handle(double, fitted):
    import evaluation
    models, train = fitted
    m = models['vector']
    te = _test_frame(seed=9)
    with contextlib.redirect_stdout(io.StringIO()):
        want = evaluation.evaluate_gpu(m, te.copy(), cut_off=[5, 20])
    m.predict_next('x', m.itemidmap.index[0], m.itemidmap.index.values)     # builds the host postings
    assert '_dev' in m.__dict__ and '_post' in m.__dict__
    m2 = pickle.loads(pickle.dumps(m))
    assert '_dev' not in m2.__dict__ and '_post' not in m2.__dict__
    for name in ('session_offsets', 'session_items', 'recency', 'n_sessions', 'k', 'sample_size', 'similarity', 'n_items'):
        assert np.array_equal(getattr(m2, name), getattr(m, name))
    with contextlib.redirect_stdout(io.StringIO()):
        assert evaluation.evaluate_gpu(m2, te.copy(), cut_off=[5, 20]) == want


def test_run_py_baseline_sknn(double, tmp_path, capsys):
    import run
    import baselines
    import evaluation
    df = make_sessions(n_items=40, n_events=800, seed=4)
    tr, te = df[df.SessionId < 200], df[df.SessionId >= 200]
    tr.to_csv(tmp_path / 'tr.tsv', sep='\t', index=False); te.to_csv(tmp_path / 'te.tsv', sep='\t', index=False)
    run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'sknn', '-ps', 'k=10,sample_size=50,similarity=vector', '-t', str(tmp_path / 'te.tsv'),
              '-m', '5', '20'])
    out = capsys.readouterr().out
    assert 'Creating SessionKNN model' in out and 'Total training time' in out
    args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv')])
    m = baselines.SessionKNN(k=10, sample_size=50, similarity='vector')
    m.fit(run.load_data(str(tmp_path / 'tr.tsv'), args))
    with contextlib.redirect_stdout(io.StringIO()):
        rec, mrr = evaluation.evaluate_gpu(m, run.load_data(str(tmp_path / 'te.tsv'), args), batch_size=512, cut_off=[5, 20])
    for q, c in enumerate((5, 20)):
        assert 'Recall@{}: {:.6f} MRR@{}: {:.6f}'.format(c, rec[q], c, mrr[q]) in out
    args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv'), '--baseline', 'sknn', '-ps', 'k=4,sample_size=9,similarity=cosine'])
    with contextlib.redirect_stdout(io.StringIO()):
        m = run._train_baseline(args)
    assert (m.k, m.sample_size, m.similarity) == (4, 9, 'cosine') and type(m.k) is int and type(m.sample_size) is int
    assert 'sknn' in run.build_parser().format_help()


@pytest.mark.parametrize('params', [dict(similarity='jaccard'), dict(sample_size=0), dict(sample_size=8193), dict(k=0),
                                    dict(k=501), dict(k=1025, sample_size=2000), dict(k=5, sample_size=4)])
def test_fit_refuses_bad_parameters(double, params):
    import baselines
    m = baselines.SessionKNN(**params)
    with pytest.raises(ValueError):
        m.fit(make_sessions(n_items=20, n_events=100, seed=1))
    assert '_dev' not in m.__dict__


def test_binding_refuses_bad_arguments_before_the_library():
    dev = object.__new__(_lib.Baselines)
    dev.n_items, dev.n_keep, dev.h = 5, 3, None
    with pytest.raises(ValueError):
        dev.sknn_fit([0, 1, 2], [0, 1], [0], 10, 'cosine')               # a rank per session
    with pytest.raises(ValueError):
        dev.sknn_fit([0, 1, 2], [0, 1], [0, 1], 10, 'jaccard')
    assert _lib.BASELINE_KINDS['sknn'] == 5


SRC = r'''
#include <stdio.h>
#include "g4r.h"

int main(void) {
  int64_t o[3] = {0, 2, 3}, bad_o[3] = {0, 3, 2};
  int32_t it[3] = {0, 1, 1}, desc[3] = {1, 0, 1}, big[3] = {0, 1, 10}, rk[2] = {1, 0}, dup[2] = {0, 0}, far[2] = {0, 2};
  int32_t c[1] = {5};
  double r[1], m[1];
  int64_t n = 0;
  g4r_baselines* h = NULL;
  int rc;
  if (G4R_BL_SKNN != 5) return 1;
  if (g4r_bl_sknn_fit(NULL, o, 2, it, 3, rk, 10, 0) != G4R_ERR_INVALID) return 2;
  if (g4r_bl_create(G4R_BL_SKNN, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 3;
  if (g4r_bl_create(G4R_BL_SKNN, 10, 0, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  if (g4r_bl_create(4, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 5;
  rc = g4r_bl_create(G4R_BL_SKNN, 10, 2, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 6;
  if (g4r_bl_evaluate(h, it, 3, o, 2, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_STATE) return 7;
  if (g4r_bl_sknn_fit(h, NULL, 2, it, 3, rk, 10, 0) != G4R_ERR_INVALID) return 8;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, NULL, 10, 0) != G4R_ERR_INVALID) return 9;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, rk, 0, 0) != G4R_ERR_INVALID) return 10;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, rk, 8193, 0) != G4R_ERR_INVALID) return 11;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, rk, 1, 0) != G4R_ERR_INVALID) return 12;        /* k = 2 > sample_size */
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, rk, 10, 2) != G4R_ERR_INVALID) return 13;
  if (g4r_bl_sknn_fit(h, bad_o, 2, it, 3, rk, 10, 0) != G4R_ERR_INVALID) return 14;
  if (g4r_bl_sknn_fit(h, o, 2, big, 3, rk, 10, 0) != G4R_ERR_INDEX) return 15;
  if (g4r_bl_sknn_fit(h, o, 2, desc, 3, rk, 10, 0) != G4R_ERR_INVALID) return 16;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, dup, 10, 0) != G4R_ERR_INVALID) return 17;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, far, 10, 0) != G4R_ERR_INDEX) return 18;
  if (g4r_bl_last_error(h)[0] == 0) return 19;
  if (g4r_bl_set_pop(h, r, 10) != G4R_ERR_STATE) return 20;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, rk, 10, 1) != G4R_OK) return 21;
  if (g4r_bl_evaluate(h, it, 3, o, 2, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_OK || n != 1) return 22;
  if (g4r_bl_destroy(h) != G4R_OK) return 23;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_sknn_abi(tmp_path):
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
