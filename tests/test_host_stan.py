"""CPU tests of STAN-style session kNN (DESIGN §3p): tests/stan_oracle.py against hand-computed values (each decay alone, a repeated
prefix item, r(n) among several shared items, underflow to exact zeros) and against oracle/sknn_oracle.py's cosine with every
decay off, baselines.STAN's fit and predict_next against the oracle on messy data, and the Python surface -- evaluate_gpu /
evaluate_events, pickles, run.py --baseline stan -- on a CPU double of _lib.Baselines backed by the oracle.  Parameter refusals,
the binding's checks and the C ABI from a C99 caller at the end.  The device path is tested in test_gpu_stan.py."""
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
import stan_oracle as sto
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions
from test_host_baselines import OracleBaselines

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float('inf')


class OracleStan(OracleBaselines):
    """_lib.Baselines('stan', ...) on the host: the oracle's index and ranking behind the binding's methods"""

    def stan_fit(self, session_offsets, items, positions, recency, w2, w3, sample_size):
        self.arrays = (session_offsets, items, positions, recency, w2, w3)
        self.sample = sample_size

    def stan_set_w1(self, w1):
        self.n_w1 = len(w1)
        self.index = sto.Index.from_arrays(*self.arrays, w1=np.asarray(w1), n_items=self.n_items)

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        name = [m for m, v in bo.MODES.items() if v == mode][0]
        cnt, ti, ts = sto.rank_events(self.index, self.n_keep, self.sample, items, offsets, n_history, name, cand, exclude_seen, k)
        rec, mrr = bo.sums(cnt, name, cut_off)
        return np.array(rec), np.array(mrr), len(cnt), cnt.astype(np.int32) if counts else None, ti, ts


@pytest.fixture
def double(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleStan)


def _index(rows, n_items, **lam):
    """rows: (session, item index, time)"""
    s, i, t = zip(*rows)
    return sto.Index(np.array(s), np.array(i), np.array(t, dtype=np.float64), n_items, **lam)


# A = {0, 1} T 11; B = {1, 2} T 20; C = {0, 2, 3} T 20 (after B in the data); D = {3} T 5.  Recency: B, C, A, D.
# Positions by time: A 0@1 1@2; B 2@1 1@2; C 2@1 3@2 0@3; D 3@1.
TINY = [('A', 0, 10), ('A', 1, 11), ('B', 1, 20), ('B', 2, 19), ('C', 0, 20), ('C', 2, 3), ('C', 3, 4), ('D', 3, 5)]


def test_oracle_positions_and_tables():
    ix = _index(TINY, 4, lambda_spw=1.0, lambda_snh=10.0, lambda_inh=2.0)
    assert list(ix.rank) == [2, 0, 1, 3]
    assert ix.q == [{2: 1, 1: 2}, {2: 1, 3: 2, 0: 3}, {0: 1, 1: 2}, {3: 1}]      # by rank: B, C, A, D
    assert list(ix.w2) == [1.0, 1.0, np.exp(-(9.0 / 10.0)), np.exp(-(15.0 / 10.0))]
    assert list(ix.w3) == [1.0, np.exp(-0.5), np.exp(-1.0)]
    assert list(ix.w1(3)) == [1.0, np.exp(-1.0), np.exp(-2.0)]


def test_oracle_session_decay_alone():
    ix = _index(TINY, 4, lambda_snh=10.0)
    r, v, q = sto.neighbours(ix, [1], 2, 4)                                # B and A share item 1; A is 9 time units older
    b, a = 1.0 / np.sqrt(2.0), (1.0 / np.sqrt(2.0)) * np.exp(-(9.0 / 10.0))
    assert list(r) == [0, 2] and list(v) == [b, a]
    assert list(sto.scores(ix, [1], 2, 4)) == [a, b + a, b, 0.0]


def test_oracle_prefix_decay_alone_last_occurrence_weighs():
    ix = _index(TINY, 4, lambda_spw=1.0)
    # c = (0, 1, 0): item 1 last at 2 (d = 1), item 0 last at 3 (d = 0, not 2); A shares both, summed in position order
    r, v, q = sto.neighbours(ix, [0, 1, 0], 2, 3)
    sa = (np.exp(-1.0) + 1.0) / np.sqrt(4.0)
    sc = 1.0 / np.sqrt(6.0)
    assert list(r) == [2, 1] and list(v) == [sa, sc]
    assert list(sto.scores(ix, [0, 1, 0], 2, 3)) == [sa + sc, sa, sc, sc]


def test_oracle_item_decay_alone_r_among_several_shared_items():
    ix = _index(TINY, 4, lambda_inh=1.0)
    sc = 2.0 / np.sqrt(6.0)
    # c = (2, 0): C shares both; r(C) = 0 (the larger p) at q = 3; C holds 2@1 3@2 0@3
    r, v, q = sto.neighbours(ix, [2, 0], 1, 4)
    assert list(r) == [1] and list(v) == [sc] and list(q) == [3]
    assert list(sto.scores(ix, [2, 0], 1, 4)) == [sc, 0.0, sc * np.exp(-2.0), sc * np.exp(-1.0)]
    # c = (0, 2): r(C) = 2 at q = 1
    r, v, q = sto.neighbours(ix, [0, 2], 1, 4)
    assert list(q) == [1]
    assert list(sto.scores(ix, [0, 2], 1, 4)) == [sc * np.exp(-2.0), 0.0, sc, sc * np.exp(-1.0)]


def test_oracle_underflow_to_exact_zeros_lists_and_counts():
    ix = _index(TINY, 4, lambda_snh=1e-300, lambda_inh=1e-300)
    r, v, q = sto.neighbours(ix, [1], 2, 4)                                # A's W2 underflows: still a neighbour, sim 0
    assert list(r) == [0, 2] and list(v) == [1.0 / np.sqrt(2.0), 0.0]
    s = sto.scores(ix, [1], 2, 4)                                          # B: 1 at r (W3[0] = 1), 2 at distance 1 -> 0
    assert list(s) == [0.0, 1.0 / np.sqrt(2.0), 0.0, 0.0]
    # session (1, 0): the target 0 scores 0 (scored by A and by B's underflow) and ties the three zero-score items
    cnt, ti, ts = sto.rank_events(ix, 2, 4, [1, 0], [0, 2], mode='conservative', k=4)
    assert cnt.tolist() == [[1, 3]]
    assert ti.tolist() == [[1, 0, 2, 3]] and ts[0, 0] == 1.0 / np.sqrt(2.0) and list(ts[0, 1:]) == [0.0, 0.0, 0.0]


def _random_index(seed, n_items=40, n_events=900, **lam):
    items, off, _, _ = make_session_arrays(n_items, n_events, seed=seed, max_len=9)
    rs = np.random.RandomState(seed)
    sess = np.repeat(np.arange(len(off) - 1), np.diff(off))
    times = rs.randint(0, 30, len(sess))                                   # ties inside and across sessions
    return items, sess, times


def test_oracle_with_every_decay_off_is_sknn_cosine():
    items, sess, times = _random_index(4)
    ix = sto.Index(sess, items, times, 40)
    ck = sko.Index(sess, items, times, 40)
    rs = np.random.RandomState(0)
    for t in (1, 2, 5, 9):
        for _ in range(6):
            prefix = rs.randint(0, 40, t)
            r1, v1, _ = sto.neighbours(ix, prefix, 8, 25)
            r2, v2 = sko.neighbours(ck, prefix, 8, 25, 'cosine')
            assert r1.tolist() == r2.tolist() and v1.tobytes() == v2.tobytes()
            assert sto.scores(ix, prefix, 8, 25).tobytes() == sko.scores(ck, prefix, 8, 25, 'cosine').tobytes()


def _messy_train(seed=3, n_items=50, n_events=1500):
    rs = np.random.RandomState(seed)
    df = make_sessions(n_items=n_items, n_events=n_events, seed=seed, item_as_str=True)
    rep = np.flatnonzero(rs.rand(len(df)) < 0.2)
    rep = rep[(rep > 0) & (df.SessionId.values[rep] == df.SessionId.values[np.maximum(rep - 1, 0)])]
    df.loc[rep, 'ItemId'] = df.ItemId.values[rep - 1]                    # repeated items
    df['Time'] = np.floor(df.Time.values / 300.0)                          # many equal times, inside sessions too
    df['SessionId'] = 's' + (df.SessionId * 7919 % 10007).astype(str)      # string ids, not in time order
    return df.sample(frac=1.0, random_state=seed).reset_index(drop=True)   # unsorted rows


LAM = dict(lambda_spw=1.02, lambda_snh=40.0, lambda_inh=2.05)


@pytest.mark.parametrize('int_time', [False, True])
def test_fit_and_predict_next_equal_the_oracle(double, int_time):
    import baselines
    tr = _messy_train()
    if int_time:
        tr['Time'] = tr.Time.astype(np.int64)
    m = baselines.STAN(k=7, sample_size=40, **LAM)
    m.fit(tr)
    ix = sto.Index(tr.SessionId.values, m.itemidmap[tr.ItemId.values].values, tr.Time.values, m.n_items, **LAM)
    off, items, rank = ix.csr()
    np.testing.assert_array_equal(m.session_offsets, off)
    np.testing.assert_array_equal(m.session_items, items)
    np.testing.assert_array_equal(m.recency, rank)
    for s in range(m.n_sessions):
        assert dict(zip(items[off[s]:off[s + 1]].tolist(), m.positions[off[s]:off[s + 1]].tolist())) == ix.q[rank[s]]
    assert m.w2.tobytes() == ix.w2[m.recency].tobytes() and m.w3.tobytes() == ix.w3.tobytes()
    assert m.n_sessions == len(rank) and list(m.itemidmap.index) == list(pd.unique(tr.ItemId.values))
    ids = m.itemidmap.index.values
    rs = np.random.RandomState(1)
    for sid in ('t1', 't2'):
        prefix = []
        for x in ids[rs.randint(0, len(ids), 6)].tolist() + [ids[0], ids[0]]:
            prefix.append(m.itemidmap[x])
            got = m.predict_next(sid, x, ids)
            want = sto.scores(ix, prefix, 7, 40)
            assert list(got.index) == list(ids)
            np.testing.assert_array_equal(got.values, want)
    assert m.current_session == 't2'


def test_host_scores_with_every_decay_off_equal_sessionknn_cosine(double, monkeypatch):
    import baselines
    tr = _messy_train(seed=5)
    a = baselines.STAN(k=6, sample_size=30, lambda_spw=INF, lambda_snh=INF, lambda_inh=INF)
    a.fit(tr)
    monkeypatch.setattr(_lib, 'Baselines', OracleBaselines)
    b = baselines.SessionKNN(k=6, sample_size=30, similarity='cosine')
    monkeypatch.setattr(b, '_device', lambda: None)
    b.fit(tr)
    for prefix in ([0], [3, 1, 3], list(range(12))):
        assert a.score_prefix(prefix).tobytes() == b.score_prefix(prefix).tobytes()


@pytest.fixture(scope='module')
def fitted():
    import baselines
    mp_ = pytest.MonkeyPatch()
    mp_.setattr(_lib, 'Baselines', OracleStan)
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    m = baselines.STAN(k=6, sample_size=30, lambda_spw=1.5, lambda_snh=3600.0, lambda_inh=1.5)
    m.fit(train.copy())
    mp_.undo()
    return m, train


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
    return sto.Index(train.SessionId.values, m.itemidmap[train.ItemId.values].values, train.Time.values, m.n_items,
                     lambda_spw=m.lambda_spw, lambda_snh=m.lambda_snh, lambda_inh=m.lambda_inh)


@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_evaluate_events_frame_ranks_and_sums(double, fitted, mode):
    import evaluation
    m, train = fitted
    te = _test_frame(seed=11)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(m, te.copy(), cut_off=[1, 5, 20], mode=mode, k=4)
        rec, mrr = evaluation.evaluate_gpu(m, te.copy(), cut_off=[1, 5, 20], mode=mode)
    df, off = _sorted(m, te)
    ev = res['events']
    assert len(ev) == len(df) - (len(off) - 1)
    cnt, ti, ts = sto.rank_events(_oracle(m, train), 6, 30, df.ItemIdx.values, off, None, mode, None, False, 4)
    np.testing.assert_array_equal(ev['rank'].values, bo.ranks(cnt, mode))
    np.testing.assert_array_equal(res['topk_items'], m.itemidmap.index.values[ti])
    np.testing.assert_array_equal(res['topk_scores'], ts)
    assert res['recall'] == rec and res['mrr'] == mrr


def test_items_exclude_seen_history_and_the_w1_table(double, fitted):
    import evaluation
    m, train = fitted
    ix = _oracle(m, train)
    te = _test_frame(seed=5)
    ids = m.itemidmap.index.values
    cand = list(ids[::3]) + [ids[0], ids[0]]                               # duplicates count
    df, off = _sorted(m, te)
    with contextlib.redirect_stdout(io.StringIO()):
        a = evaluation.evaluate_events(m, te.copy(), items=cand, cut_off=[3, 10], mode='conservative', k=3)
        b = evaluation.evaluate_events(m, te.copy(), cut_off=[5], exclude_seen=True, k=5)
    cnt, ti, ts = sto.rank_events(ix, 6, 30, df.ItemIdx.values, off, None, 'conservative', m.itemidmap[cand].values, k=3)
    np.testing.assert_array_equal(a['events']['rank'].values, bo.ranks(cnt, 'conservative'))
    np.testing.assert_array_equal(a['topk_scores'], ts)
    cnt, ti, ts = sto.rank_events(ix, 6, 30, df.ItemIdx.values, off, None, 'standard', None, True, k=5)
    np.testing.assert_array_equal(b['events']['rank'].values, bo.ranks(cnt, 'standard'))
    np.testing.assert_array_equal(b['topk_items'], m.itemidmap.index.values[ti])
    assert np.isinf(b['events']['rank'].values).any()
    # history: a session longer than any training session, so W1 has to grow to the frame's longest session
    rs = np.random.RandomState(2)
    long_s = pd.DataFrame({'SessionId': 77777, 'ItemId': ids[rs.randint(0, len(ids), 60)], 'Time': np.arange(60) + 10 ** 6})
    df = pd.concat([df, long_s.assign(ItemIdx=m.itemidmap[long_s.ItemId].values)], ignore_index=True)
    assert 60 > len(m.w3) and m._device().n_w1 < 60
    pos, size = df.groupby('SessionId').cumcount(), df.groupby('SessionId').SessionId.transform('size')
    hist = df[pos < size // 2][['SessionId', 'ItemId', 'Time']]
    rest = df.drop(hist.index)[['SessionId', 'ItemId', 'Time']]
    with contextlib.redirect_stdout(io.StringIO()):
        h = evaluation.evaluate_events(m, rest.copy(), cut_off=[5], history=hist.copy())
    assert m._device().n_w1 >= 60
    sids = np.sort(rest.SessionId.unique())
    both = pd.concat([df[df.index.isin(hist.index)], df[~df.index.isin(hist.index)]]).sort_values('SessionId', kind='stable')
    both = both[both.SessionId.isin(sids)]
    nh = hist.groupby('SessionId').size().reindex(sids, fill_value=0).values
    boff = np.r_[0, np.cumsum(both.groupby('SessionId').size().values)]
    cnt = sto.rank_events(ix, 6, 30, both.ItemIdx.values, boff, nh)[0]
    np.testing.assert_array_equal(h['events']['rank'].values, bo.ranks(cnt, 'standard'))


def test_pickle_round_trip_without_the_handle(double, fitted):
    import evaluation
    m, train = fitted
    te = _test_frame(seed=9)
    with contextlib.redirect_stdout(io.StringIO()):
        want = evaluation.evaluate_gpu(m, te.copy(), cut_off=[5, 20])
    m.predict_next('x', m.itemidmap.index[0], m.itemidmap.index.values)     # builds the host postings
    assert '_dev' in m.__dict__ and '_post' in m.__dict__
    m2 = pickle.loads(pickle.dumps(m))
    assert '_dev' not in m2.__dict__ and '_post' not in m2.__dict__
    for name in ('session_offsets', 'session_items', 'positions', 'recency', 'w2', 'w3', 'n_sessions', 'k', 'sample_size', 'lambda_spw',
                 'lambda_snh', 'lambda_inh', 'n_items'):
        assert np.array_equal(getattr(m2, name), getattr(m, name))
    with contextlib.redirect_stdout(io.StringIO()):
        assert evaluation.evaluate_gpu(m2, te.copy(), cut_off=[5, 20]) == want


def test_run_py_baseline_stan(double, tmp_path, capsys):
    import run
    import baselines
    import evaluation
    df = make_sessions(n_items=40, n_events=800, seed=4)
    tr, te = df[df.SessionId < 200], df[df.SessionId >= 200]
    tr.to_csv(tmp_path / 'tr.tsv', sep='\t', index=False); te.to_csv(tmp_path / 'te.tsv', sep='\t', index=False)
    run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'stan', '-ps', 'k=10,sample_size=50,lambda_spw=1.02,lambda_snh=inf,lambda_inh=2.05',
              '-t', str(tmp_path / 'te.tsv'), '-m', '5', '20'])
    out = capsys.readouterr().out
    assert 'Creating STAN model' in out and 'Total training time' in out
    args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv')])
    m = baselines.STAN(k=10, sample_size=50, lambda_spw=1.02, lambda_snh=INF, lambda_inh=2.05)
    m.fit(run.load_data(str(tmp_path / 'tr.tsv'), args))
    with contextlib.redirect_stdout(io.StringIO()):
        rec, mrr = evaluation.evaluate_gpu(m, run.load_data(str(tmp_path / 'te.tsv'), args), batch_size=512, cut_off=[5, 20])
    for q, c in enumerate((5, 20)):
        assert 'Recall@{}: {:.6f} MRR@{}: {:.6f}'.format(c, rec[q], c, mrr[q]) in out
    args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv'), '--baseline', 'stan', '-ps', 'k=4,sample_size=9,lambda_snh=inf'])
    with contextlib.redirect_stdout(io.StringIO()):
        m = run._train_baseline(args)
    assert (m.k, m.sample_size, m.lambda_snh, m.lambda_spw) == (4, 9, INF, 1.02) and type(m.k) is int and type(m.lambda_snh) is float
    assert 'stan' in run.build_parser().format_help()


@pytest.mark.parametrize('params', [dict(sample_size=0), dict(sample_size=8193), dict(k=0), dict(k=501), dict(k=1025, sample_size=2000),
                                    dict(k=5, sample_size=4), dict(lambda_spw=0.0), dict(lambda_snh=-1.0), dict(lambda_inh=float('nan')),
                                    dict(lambda_spw=-INF)])
def test_fit_refuses_bad_parameters(double, params):
    import baselines
    m = baselines.STAN(**params)
    with pytest.raises(ValueError):
        m.fit(make_sessions(n_items=20, n_events=100, seed=1))
    assert '_dev' not in m.__dict__


def test_fit_refuses_a_non_numeric_time_column(double):
    import baselines
    df = make_sessions(n_items=20, n_events=100, seed=1)
    df['Time'] = pd.to_datetime(df.Time, unit='s')
    with pytest.raises(ValueError):
        baselines.STAN().fit(df)
    df['Time'] = df.Time.astype(str)
    m = baselines.STAN()
    with pytest.raises(ValueError):
        m.fit(df)
    assert '_dev' not in m.__dict__


def test_binding_refuses_bad_arguments_before_the_library():
    dev = object.__new__(_lib.Baselines)
    dev.n_items, dev.n_keep, dev.h = 5, 3, None
    ok = dict(session_offsets=[0, 1, 2], items=[0, 1], positions=[1, 1], recency=[0, 1], w2=[1.0, 0.5], w3=[1.0], sample_size=10)
    for bad in (dict(positions=[1]), dict(recency=[0]), dict(w2=[1.0]), dict(w3=[]), dict(w3=[[1.0]]), dict(session_offsets=[0])):
        with pytest.raises(ValueError):
            dev.stan_fit(**dict(ok, **bad))
    for bad in ([], [[1.0]]):
        with pytest.raises(ValueError):
            dev.stan_set_w1(bad)
    assert _lib.BASELINE_KINDS['stan'] == 6 and _lib.BASELINE_KINDS['sknn'] == 5


SRC = r'''
#include <math.h>
#include <stdio.h>
#include "g4r.h"

int main(void) {
  int64_t o[3] = {0, 2, 3}, bad_o[3] = {0, 3, 2};
  int32_t it[3] = {0, 1, 1}, desc[3] = {1, 0, 1}, big[3] = {0, 1, 10}, rk[2] = {1, 0}, dup[2] = {0, 0}, far[2] = {0, 2};
  int32_t pos[3] = {1, 2, 1}, pos0[3] = {0, 2, 1}, pos_far[3] = {1, 3, 1}, pos_same[3] = {2, 2, 1};
  int32_t ev[4] = {0, 1, 0, 1}, c[1] = {5};
  int64_t eo[2] = {0, 4}, eo3[3] = {0, 3, 4};
  double w2[2] = {1.0, 0.5}, w2_bad[2] = {1.0, 1.5}, w3[2] = {1.0, 0.25}, w3_nan[2] = {1.0, NAN}, w1[3] = {1.0, 0.5, 0.25};
  double w1_neg[3] = {1.0, -0.5, 0.25};
  double r[1], m[1], sc[2];
  int32_t ti[2], cnt[6];
  int64_t n = 0;
  g4r_baselines* h = NULL;
  int rc;
  if (G4R_BL_STAN != 6 || G4R_BL_SKNN != 5) return 1;
  if (g4r_bl_stan_fit(NULL, o, 2, it, 3, pos, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 2;
  if (g4r_bl_stan_set_w1(NULL, w1, 3) != G4R_ERR_INVALID) return 3;
  if (g4r_bl_create(G4R_BL_STAN, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  if (g4r_bl_create(G4R_BL_STAN, 10, 0, 0, &h) != G4R_ERR_INVALID || h != NULL) return 5;
  if (g4r_bl_create(4, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 6;
  if (g4r_bl_create(7, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 7;
  rc = g4r_bl_create(G4R_BL_STAN, 10, 2, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 8;
  if (g4r_bl_evaluate(h, it, 3, o, 2, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_STATE) return 9;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, rk, 10, 0) != G4R_ERR_STATE) return 10;
  if (g4r_bl_stan_fit(h, NULL, 2, it, 3, pos, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 11;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, NULL, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 12;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, NULL, w2, w3, 2, 10) != G4R_ERR_INVALID) return 13;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, NULL, w3, 2, 10) != G4R_ERR_INVALID) return 14;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, NULL, 2, 10) != G4R_ERR_INVALID) return 15;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3, 0, 10) != G4R_ERR_INVALID) return 16;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3, 2, 0) != G4R_ERR_INVALID) return 17;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3, 2, 8193) != G4R_ERR_INVALID) return 18;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3, 2, 1) != G4R_ERR_INVALID) return 19;   /* k = 2 > sample_size */
  if (g4r_bl_stan_fit(h, bad_o, 2, it, 3, pos, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 20;
  if (g4r_bl_stan_fit(h, o, 2, big, 3, pos, rk, w2, w3, 2, 10) != G4R_ERR_INDEX) return 21;
  if (g4r_bl_stan_fit(h, o, 2, desc, 3, pos, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 22;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos0, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 23;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos_far, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 24;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos_same, rk, w2, w3, 2, 10) != G4R_ERR_INVALID) return 25;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2_bad, w3, 2, 10) != G4R_ERR_INVALID) return 26;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3_nan, 2, 10) != G4R_ERR_INVALID) return 27;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, dup, w2, w3, 2, 10) != G4R_ERR_INVALID) return 28;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, far, w2, w3, 2, 10) != G4R_ERR_INDEX) return 29;
  if (g4r_bl_stan_set_w1(h, NULL, 3) != G4R_ERR_INVALID) return 30;
  if (g4r_bl_stan_set_w1(h, w1, 0) != G4R_ERR_INVALID) return 31;
  if (g4r_bl_stan_set_w1(h, w1_neg, 3) != G4R_ERR_INVALID) return 32;
  if (g4r_bl_last_error(h)[0] == 0) return 33;
  if (g4r_bl_set_pop(h, r, 10) != G4R_ERR_STATE) return 34;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3, 2, 10) != G4R_OK) return 35;
  /* no W1 table yet: every counted event's prefix is longer than it */
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_INVALID) return 36;
  if (g4r_bl_stan_set_w1(h, w1, 2) != G4R_OK) return 37;
  /* a 4-event session has a prefix of 3 > 2; sessions of 3 and 1 events need only 2 */
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_INVALID) return 38;
  if (g4r_bl_evaluate(h, ev, 4, eo3, 2, NULL, 0, c, 1, NULL, 0, 0, 1, r, m, &n, cnt, ti, sc) != G4R_OK || n != 2) return 39;
  if (g4r_bl_stan_set_w1(h, w1, 3) != G4R_OK) return 40;
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_OK || n != 3) return 41;
  if (g4r_bl_destroy(h) != G4R_OK) return 42;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_stan_abi(tmp_path):
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
