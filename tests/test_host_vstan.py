"""CPU tests of VSTAN-style session kNN (DESIGN §3r): tests/vstan_oracle.py against hand-computed values ('vector' alone, W4 alone
with r(n) among several shared items, F alone with df counted in sessions, underflow to exact zeros) and against
tests/stan_oracle.py with every addition off, baselines.VSTAN's fit and predict_next against the oracle on messy data, and the
Python surface -- evaluate_gpu / evaluate_events, pickles, run.py --baseline vstan -- on a CPU double of _lib.Baselines backed by
the oracle.  Parameter refusals, the binding's checks and the C ABI from a C99 caller at the end.  The device path is tested in
test_gpu_vstan.py."""
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
import stan_oracle as sto
import vstan_oracle as vso
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions
from test_host_baselines import OracleBaselines

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float('inf')


class OracleVstan(OracleBaselines):
    """_lib.Baselines('vstan', ...) on the host: the oracle's index and ranking behind the binding's methods"""

    def stan_fit(self, session_offsets, items, positions, recency, w2, w3, sample_size):
        self.arrays = (session_offsets, items, positions, recency, w2, w3)
        self.sample = sample_size
        self.settings = None

    def stan_set_w1(self, w1):
        self.n_w1, self.w1 = len(w1), np.asarray(w1)

    def vstan_set(self, similarity, f, w4):
        self.n_w4, self.settings = len(w4), (similarity, np.asarray(f), np.asarray(w4))

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        assert self.settings is not None
        L = int(np.diff(offsets).max(initial=1)) - 1
        assert self.n_w1 >= L and self.n_w4 >= L
        index = vso.Index.from_arrays(*self.arrays, w1=self.w1, n_items=self.n_items, similarity=self.settings[0], f=self.settings[1],
                                      w4=self.settings[2])
        name = [m for m, v in bo.MODES.items() if v == mode][0]
        cnt, ti, ts = vso.rank_events(index, self.n_keep, self.sample, items, offsets, n_history, name, cand, exclude_seen, k)
        rec, mrr = bo.sums(cnt, name, cut_off)
        return np.array(rec), np.array(mrr), len(cnt), cnt.astype(np.int32) if counts else None, ti, ts


@pytest.fixture
def double(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleVstan)


def _index(rows, n_items, **kw):
    """rows: (session, item index, time)"""
    s, i, t = zip(*rows)
    return vso.Index(np.array(s), np.array(i), np.array(t, dtype=np.float64), n_items, **kw)


# A = {0, 1} T 11; B = {1, 2} T 20; C = {0, 2, 3} T 20 (after B in the data); D = {3} T 5.  Recency: B, C, A, D.
# Positions by time: A 0@1 1@2; B 2@1 1@2; C 2@1 3@2 0@3; D 3@1.
TINY = [('A', 0, 10), ('A', 1, 11), ('B', 1, 20), ('B', 2, 19), ('C', 0, 20), ('C', 2, 3), ('C', 3, 4), ('D', 3, 5)]


def test_oracle_vector_similarity_alone():
    ix = _index(TINY, 4, similarity='vector', lambda_spw=1.0)
    # c = (0, 1, 0): item 1 last at 2 (W1[1]), item 0 last at 3 (W1[0]); B shares 1, C shares 0, A both, summed in position order
    r, v, q, dr, g = vso.neighbours(ix, [0, 1, 0], 2, 3)
    a = np.exp(-1.0) + 1.0
    assert list(r) == [2, 1] and list(v) == [a, 1.0] and list(g) == [a, 1.0] and list(dr) == [0, 0]
    assert list(vso.scores(ix, [0, 1, 0], 2, 3)) == [a + 1.0, a, 1.0, 1.0]
    assert list(vso.scores(ix, [0, 1, 0], 3, 3)) == [a + 1.0, a + np.exp(-1.0), 1.0 + np.exp(-1.0), 1.0]   # B (e^-1) third


def test_oracle_neighbour_weight_alone_r_among_several_shared_items():
    ix = _index(TINY, 4, lambda_ipw=1.0)
    # c = (2, 0, 1): B shares 2 and 1 (r = 1, d = 0), A shares 0 and 1 (r = 1, d = 0), C shares 2 and 0 (r = 0 at p 2, d = 1)
    r, v, q, dr, g = vso.neighbours(ix, [2, 0, 1], 3, 4)
    sb, sc = 2.0 / np.sqrt(6.0), 2.0 / np.sqrt(9.0)
    assert list(r) == [0, 2, 1] and list(v) == [sb, sb, sc] and list(dr) == [0, 0, 1]
    gc = sc * np.exp(-1.0)
    assert list(g) == [sb, sb, gc]
    assert list(vso.scores(ix, [2, 0, 1], 3, 4)) == [sb + gc, sb + sb, sb + gc, gc]
    # c = (0, 2, 1, 1): C shares 0 and 2, r = 2 at p 2 of t = 4: d = 2
    r, v, q, dr, g = vso.neighbours(ix, [0, 2, 1, 1], 3, 4)
    assert dict(zip(r.tolist(), dr.tolist())) == {0: 0, 1: 2, 2: 0}
    assert g[list(r).index(1)] == v[list(r).index(1)] * np.exp(-2.0)


def test_oracle_idf_alone_counts_sessions_not_events():
    # A holds 0 twice and E holds 1 twice: df = (2, 3, 2, 2) over 5 sessions.  Recency: B, C, A, D, E.
    rows = TINY + [('A', 0, 12), ('E', 1, 1), ('E', 1, 2)]
    ix = _index(rows, 4, lambda_idf=0.5)
    f = [1.0 + 0.5 * np.log(5 / 2), 1.0 + 0.5 * np.log(5 / 3), 1.0 + 0.5 * np.log(5 / 2), 1.0 + 0.5 * np.log(5 / 2)]
    assert list(ix.f) == f
    s = 1.0 / np.sqrt(2.0)                                                 # c = (1): E (sim 1), B and A (1 / sqrt 2), in that order
    r, v, q, dr, g = vso.neighbours(ix, [1], 3, 5)
    assert list(r) == [4, 0, 2] and list(v) == [1.0, s, s]
    assert list(vso.scores(ix, [1], 3, 5)) == [s * f[0], (1.0 + s + s) * f[1], s * f[2], 0.0]


def test_oracle_underflow_to_exact_zeros_lists_and_counts():
    ix = _index(TINY, 4, lambda_ipw=1e-300, lambda_idf=1.0)
    # c = (1, 0): A shares both (r = 0, d = 0, sim 1), B shares 1 only (d = 1: g = 0), C shares 0 (sim 1 / sqrt 6)
    r, v, q, dr, g = vso.neighbours(ix, [1, 0], 2, 4)
    assert list(r) == [2, 0] and list(v) == [1.0, 0.5] and list(g) == [1.0, 0.0]
    s = vso.scores(ix, [1, 0], 2, 4)
    assert list(s) == [ix.f[0], ix.f[1], 0.0, 0.0]                         # 2 is scored (by B) and scores 0
    # session (1, 0, 2): the target 2 scores 0 and ties the zero-score items 2 and 3
    cnt, ti, ts = vso.rank_events(ix, 2, 4, [1, 0, 2], [0, 3], mode='conservative', k=4, only=[1])
    assert cnt.tolist() == [[2, 2]]
    assert ix.f[0] == ix.f[1]                                              # df 2 of 4 sessions each: a tie, by index
    assert ti.tolist() == [[0, 1, 2, 3]] and list(ts[0]) == [ix.f[0], ix.f[1], 0.0, 0.0]


def _random_index(seed, n_items=40, n_events=900):
    items, off, _, _ = make_session_arrays(n_items, n_events, seed=seed, max_len=9)
    rs = np.random.RandomState(seed)
    sess = np.repeat(np.arange(len(off) - 1), np.diff(off))
    times = rs.randint(0, 30, len(sess))                                   # ties inside and across sessions
    return items, sess, times


def test_oracle_with_every_addition_off_is_stan():
    items, sess, times = _random_index(4)
    lam = dict(lambda_spw=1.02, lambda_snh=10.0, lambda_inh=2.05)
    ix = vso.Index(sess, items, times, 40, 'cosine', lambda_ipw=INF, lambda_idf=0.0, **lam)
    st = sto.Index(sess, items, times, 40, **lam)
    rs = np.random.RandomState(0)
    for t in (1, 2, 5, 9):
        for _ in range(6):
            prefix = rs.randint(0, 40, t)
            r1, v1, q1, _, g1 = vso.neighbours(ix, prefix, 8, 25)
            r2, v2, q2 = sto.neighbours(st, prefix, 8, 25)
            assert r1.tolist() == r2.tolist() and v1.tobytes() == v2.tobytes() and g1.tobytes() == v2.tobytes() and q1.tolist() == q2.tolist()
            assert vso.scores(ix, prefix, 8, 25).tobytes() == sto.scores(st, prefix, 8, 25).tobytes()
    only = np.arange(0, 60, 7)
    a = vso.rank_events(ix, 8, 25, items[:200], np.r_[0, 50, 120, 200], mode='median', exclude_seen=True, k=5, only=only)
    b = sto.rank_events(st, 8, 25, items[:200], np.r_[0, 50, 120, 200], mode='median', exclude_seen=True, k=5, only=only)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


def _messy_train(seed=3, n_items=50, n_events=1500):
    rs = np.random.RandomState(seed)
    df = make_sessions(n_items=n_items, n_events=n_events, seed=seed, item_as_str=True)
    rep = np.flatnonzero(rs.rand(len(df)) < 0.2)
    rep = rep[(rep > 0) & (df.SessionId.values[rep] == df.SessionId.values[np.maximum(rep - 1, 0)])]
    df.loc[rep, 'ItemId'] = df.ItemId.values[rep - 1]                    # repeated items
    df['Time'] = np.floor(df.Time.values / 300.0)                          # many equal times, inside sessions too
    df['SessionId'] = 's' + (df.SessionId * 7919 % 10007).astype(str)      # string ids, not in time order
    return df.sample(frac=1.0, random_state=seed).reset_index(drop=True)   # unsorted rows


LAM = dict(lambda_spw=1.02, lambda_snh=40.0, lambda_inh=2.05, lambda_ipw=1.3, lambda_idf=0.6)


@pytest.mark.parametrize('similarity,int_time', [('cosine', False), ('vector', False), ('vector', True)])
def test_fit_and_predict_next_equal_the_oracle(double, similarity, int_time):
    import baselines
    tr = _messy_train()
    if int_time:
        tr['Time'] = tr.Time.astype(np.int64)
    m = baselines.VSTAN(k=7, sample_size=40, similarity=similarity, **LAM)
    m.fit(tr)
    ix = vso.Index(tr.SessionId.values, m.itemidmap[tr.ItemId.values].values, tr.Time.values, m.n_items, similarity, **LAM)
    off, items, rank = ix.csr()
    np.testing.assert_array_equal(m.session_offsets, off)
    np.testing.assert_array_equal(m.session_items, items)
    np.testing.assert_array_equal(m.recency, rank)
    assert m.w2.tobytes() == ix.w2[m.recency].tobytes() and m.w3.tobytes() == ix.w3.tobytes() and m.f.tobytes() == ix.f.tobytes()
    assert m._w4(9).tobytes() == ix.w4(9).tobytes() and (m.f > 1.0).all()
    ids = m.itemidmap.index.values
    rs = np.random.RandomState(1)
    for sid in ('t1', 't2'):
        prefix = []
        for x in ids[rs.randint(0, len(ids), 6)].tolist() + [ids[0], ids[0]]:
            prefix.append(m.itemidmap[x])
            got = m.predict_next(sid, x, ids)
            assert list(got.index) == list(ids)
            np.testing.assert_array_equal(got.values, vso.scores(ix, prefix, 7, 40))
    assert m.current_session == 't2'


def test_host_scores_with_every_addition_off_equal_stan(double):
    import baselines
    tr = _messy_train(seed=5)
    lam = dict(lambda_spw=1.02, lambda_snh=40.0, lambda_inh=2.05)
    a = baselines.VSTAN(k=6, sample_size=30, similarity='cosine', lambda_ipw=INF, lambda_idf=0.0, **lam)
    a.fit(tr)
    b = baselines.STAN(k=6, sample_size=30, **lam)
    b._device = lambda: None
    b.fit(tr)
    assert (a.f == 1.0).all()
    for prefix in ([0], [3, 1, 3], list(range(12))):
        assert a.score_prefix(prefix).tobytes() == b.score_prefix(prefix).tobytes()


@pytest.fixture(scope='module')
def fitted():
    import baselines
    mp_ = pytest.MonkeyPatch()
    mp_.setattr(_lib, 'Baselines', OracleVstan)
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    m = baselines.VSTAN(k=6, sample_size=30, similarity='vector', lambda_spw=1.5, lambda_snh=3600.0, lambda_inh=1.5, lambda_ipw=1.2,
                        lambda_idf=0.8)
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
    return vso.Index(train.SessionId.values, m.itemidmap[train.ItemId.values].values, train.Time.values, m.n_items, m.similarity,
                     lambda_spw=m.lambda_spw, lambda_snh=m.lambda_snh, lambda_inh=m.lambda_inh, lambda_ipw=m.lambda_ipw,
                     lambda_idf=m.lambda_idf)


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
    cnt, ti, ts = vso.rank_events(_oracle(m, train), 6, 30, df.ItemIdx.values, off, None, mode, None, False, 4)
    np.testing.assert_array_equal(ev['rank'].values, bo.ranks(cnt, mode))
    np.testing.assert_array_equal(res['topk_items'], m.itemidmap.index.values[ti])
    np.testing.assert_array_equal(res['topk_scores'], ts)
    assert res['recall'] == rec and res['mrr'] == mrr


def test_items_exclude_seen_history_and_the_w1_w4_tables(double, fitted):
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
    cnt, ti, ts = vso.rank_events(ix, 6, 30, df.ItemIdx.values, off, None, 'conservative', m.itemidmap[cand].values, k=3)
    np.testing.assert_array_equal(a['events']['rank'].values, bo.ranks(cnt, 'conservative'))
    np.testing.assert_array_equal(a['topk_scores'], ts)
    cnt, ti, ts = vso.rank_events(ix, 6, 30, df.ItemIdx.values, off, None, 'standard', None, True, k=5)
    np.testing.assert_array_equal(b['events']['rank'].values, bo.ranks(cnt, 'standard'))
    np.testing.assert_array_equal(b['topk_items'], m.itemidmap.index.values[ti])
    assert np.isinf(b['events']['rank'].values).any()
    # history: a session longer than any training session, so W1 and W4 have to grow to the frame's longest session
    rs = np.random.RandomState(2)
    long_s = pd.DataFrame({'SessionId': 77777, 'ItemId': ids[rs.randint(0, len(ids), 60)], 'Time': np.arange(60) + 10 ** 6})
    df = pd.concat([df, long_s.assign(ItemIdx=m.itemidmap[long_s.ItemId].values)], ignore_index=True)
    assert 60 > len(m.w3) and m._device().n_w1 < 60 and m._device().n_w4 < 60
    pos, size = df.groupby('SessionId').cumcount(), df.groupby('SessionId').SessionId.transform('size')
    hist = df[pos < size // 2][['SessionId', 'ItemId', 'Time']]
    rest = df.drop(hist.index)[['SessionId', 'ItemId', 'Time']]
    with contextlib.redirect_stdout(io.StringIO()):
        h = evaluation.evaluate_events(m, rest.copy(), cut_off=[5], history=hist.copy())
    assert m._device().n_w1 >= 60 and m._device().n_w4 >= 60
    sids = np.sort(rest.SessionId.unique())
    both = pd.concat([df[df.index.isin(hist.index)], df[~df.index.isin(hist.index)]]).sort_values('SessionId', kind='stable')
    both = both[both.SessionId.isin(sids)]
    nh = hist.groupby('SessionId').size().reindex(sids, fill_value=0).values
    boff = np.r_[0, np.cumsum(both.groupby('SessionId').size().values)]
    cnt = vso.rank_events(ix, 6, 30, both.ItemIdx.values, boff, nh)[0]
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
    for name in ('session_offsets', 'session_items', 'positions', 'recency', 'w2', 'w3', 'f', 'n_sessions', 'k', 'sample_size', 'similarity',
                 'lambda_spw', 'lambda_snh', 'lambda_inh', 'lambda_ipw', 'lambda_idf', 'n_items'):
        assert np.array_equal(getattr(m2, name), getattr(m, name))
    with contextlib.redirect_stdout(io.StringIO()):
        assert evaluation.evaluate_gpu(m2, te.copy(), cut_off=[5, 20]) == want
    assert m2._device().settings[0] == 'vector'                            # re-uploaded from the pickle, no refit


def test_run_py_baseline_vstan(double, tmp_path, capsys):
    import run
    import baselines
    import evaluation
    df = make_sessions(n_items=40, n_events=800, seed=4)
    tr, te = df[df.SessionId < 200], df[df.SessionId >= 200]
    tr.to_csv(tmp_path / 'tr.tsv', sep='\t', index=False); te.to_csv(tmp_path / 'te.tsv', sep='\t', index=False)
    run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'vstan', '-ps', 'k=10,sample_size=50,similarity=vector,lambda_ipw=inf,lambda_idf=0',
              '-t', str(tmp_path / 'te.tsv'), '-m', '5', '20'])
    out = capsys.readouterr().out
    assert 'Creating VSTAN model' in out and 'Total training time' in out
    args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv')])
    m = baselines.VSTAN(k=10, sample_size=50, similarity='vector', lambda_ipw=INF, lambda_idf=0.0)
    m.fit(run.load_data(str(tmp_path / 'tr.tsv'), args))
    with contextlib.redirect_stdout(io.StringIO()):
        rec, mrr = evaluation.evaluate_gpu(m, run.load_data(str(tmp_path / 'te.tsv'), args), batch_size=512, cut_off=[5, 20])
    for q, c in enumerate((5, 20)):
        assert 'Recall@{}: {:.6f} MRR@{}: {:.6f}'.format(c, rec[q], c, mrr[q]) in out
    args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv'), '--baseline', 'vstan', '-ps', 'k=4,sample_size=9,similarity=vector,lambda_idf=0'])
    with contextlib.redirect_stdout(io.StringIO()):
        m = run._train_baseline(args)
    assert (m.k, m.sample_size, m.similarity, m.lambda_idf, m.lambda_ipw) == (4, 9, 'vector', 0.0, 1.02) and type(m.lambda_idf) is float
    assert 'vstan' in run.build_parser().format_help()


@pytest.mark.parametrize('params', [dict(similarity='dot'), dict(sample_size=0), dict(sample_size=8193), dict(k=0), dict(k=501),
                                    dict(k=1025, sample_size=2000), dict(lambda_spw=0.0), dict(lambda_snh=-1.0),
                                    dict(lambda_inh=float('nan')), dict(lambda_ipw=0.0), dict(lambda_ipw=-1.0),
                                    dict(lambda_ipw=float('nan')), dict(lambda_idf=-0.5), dict(lambda_idf=float('nan')),
                                    dict(lambda_idf=INF)])
def test_fit_refuses_bad_parameters(double, params):
    import baselines
    m = baselines.VSTAN(**params)
    with pytest.raises(ValueError):
        m.fit(make_sessions(n_items=20, n_events=100, seed=1))
    assert '_dev' not in m.__dict__


def test_fit_refuses_a_non_numeric_or_boolean_time_column(double):
    import baselines
    df = make_sessions(n_items=20, n_events=100, seed=1)
    for col in (pd.to_datetime(df.Time, unit='s'), df.Time.astype(str), df.Time > df.Time.median()):
        m = baselines.VSTAN()
        with pytest.raises(ValueError):
            m.fit(df.assign(Time=col))
        assert '_dev' not in m.__dict__


def test_binding_refuses_bad_arguments_before_the_library():
    dev = object.__new__(_lib.Baselines)
    dev.n_items, dev.n_keep, dev.h = 3, 2, None
    ok = dict(similarity='vector', f=[1.0, 2.0, 1.5], w4=[1.0, 0.5])
    for bad in (dict(similarity='dot'), dict(similarity=1), dict(f=[1.0, 2.0]), dict(f=[1.0, -1.0, 1.0]), dict(f=[1.0, INF, 1.0]),
                dict(f=[1.0, np.nan, 1.0]), dict(w4=[]), dict(w4=[[1.0]]), dict(w4=[1.0, 1.5]), dict(w4=[1.0, -0.1]), dict(w4=[np.nan])):
        with pytest.raises(ValueError):
            dev.vstan_set(**dict(ok, **bad))
    assert _lib.BASELINE_KINDS['vstan'] == 11 and _lib.BASELINE_KINDS['stan'] == 6
    assert 'g4r_bl_vstan_set' in _lib.EXPORTS


SRC = r'''
#include <math.h>
#include <stdio.h>
#include "g4r.h"

int main(void) {
  int64_t o[3] = {0, 2, 3};
  int32_t it[3] = {0, 1, 1}, rk[2] = {1, 0}, pos[3] = {1, 2, 1};
  int32_t ev[4] = {0, 1, 0, 1}, c[1] = {5};
  int64_t eo[2] = {0, 4}, eo3[3] = {0, 3, 4};
  double w2[2] = {1.0, 0.5}, w3[2] = {1.0, 0.25}, w1[3] = {1.0, 0.5, 0.25};
  double f[10] = {1, 2, 1, 1, 1, 1, 1, 1, 1, 1}, f_neg[10] = {1, -2, 1, 1, 1, 1, 1, 1, 1, 1}, f_inf[10] = {1, INFINITY, 1, 1, 1, 1, 1, 1, 1, 1};
  double w4[3] = {1.0, 0.5, 0.25}, w4_big[3] = {1.0, 1.5, 0.25}, w4_nan[3] = {1.0, NAN, 0.25};
  double r[1], m[1], sc[2];
  int32_t ti[2], cnt[6];
  int64_t n = 0;
  g4r_baselines* h = NULL;
  g4r_baselines* st = NULL;
  int rc;
  if (G4R_BL_VSTAN != 11 || G4R_BL_STAN != 6) return 1;
  if (g4r_bl_vstan_set(NULL, 0, f, 10, w4, 3) != G4R_ERR_INVALID) return 2;
  if (g4r_bl_create(G4R_BL_VSTAN, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 3;
  if (g4r_bl_create(G4R_BL_VSTAN, 10, 0, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  if (g4r_bl_create(4, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 5;
  if (g4r_bl_create(7, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 6;
  if (g4r_bl_create(10, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 7;
  rc = g4r_bl_create(G4R_BL_VSTAN, 10, 2, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 8;
  if (g4r_bl_evaluate(h, it, 3, o, 2, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_STATE) return 9;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, rk, 10, 0) != G4R_ERR_STATE) return 10;
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3, 2, 10) != G4R_OK) return 11;
  if (g4r_bl_stan_set_w1(h, w1, 3) != G4R_OK) return 12;
  /* fitted with W1, but not set since the fit */
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_STATE) return 13;
  if (g4r_bl_vstan_set(h, 2, f, 10, w4, 3) != G4R_ERR_INVALID) return 14;
  if (g4r_bl_vstan_set(h, -1, f, 10, w4, 3) != G4R_ERR_INVALID) return 15;
  if (g4r_bl_vstan_set(h, 1, NULL, 10, w4, 3) != G4R_ERR_INVALID) return 16;
  if (g4r_bl_vstan_set(h, 1, f, 9, w4, 3) != G4R_ERR_INVALID) return 17;
  if (g4r_bl_vstan_set(h, 1, f_neg, 10, w4, 3) != G4R_ERR_INVALID) return 18;
  if (g4r_bl_vstan_set(h, 1, f_inf, 10, w4, 3) != G4R_ERR_INVALID) return 19;
  if (g4r_bl_vstan_set(h, 1, f, 10, NULL, 3) != G4R_ERR_INVALID) return 20;
  if (g4r_bl_vstan_set(h, 1, f, 10, w4, 0) != G4R_ERR_INVALID) return 21;
  if (g4r_bl_vstan_set(h, 1, f, 10, w4_big, 3) != G4R_ERR_INVALID) return 22;
  if (g4r_bl_vstan_set(h, 1, f, 10, w4_nan, 3) != G4R_ERR_INVALID) return 23;
  if (g4r_bl_last_error(h)[0] == 0) return 24;
  /* the refused calls set nothing */
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_STATE) return 25;
  if (g4r_bl_vstan_set(h, 1, f, 10, w4, 2) != G4R_OK) return 26;
  /* a 4-event session has a prefix of 3 > n_w4 = 2; sessions of 3 and 1 events need only 2 */
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_INVALID) return 27;
  if (g4r_bl_evaluate(h, ev, 4, eo3, 2, NULL, 0, c, 1, NULL, 0, 0, 1, r, m, &n, cnt, ti, sc) != G4R_OK || n != 2) return 28;
  if (g4r_bl_vstan_set(h, 0, f, 10, w4, 3) != G4R_OK) return 29;
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_OK || n != 3) return 30;
  /* a fit clears the settings */
  if (g4r_bl_stan_fit(h, o, 2, it, 3, pos, rk, w2, w3, 2, 10) != G4R_OK) return 31;
  if (g4r_bl_evaluate(h, ev, 4, eo, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_STATE) return 32;
  /* a STAN handle takes no VSTAN settings */
  if (g4r_bl_create(G4R_BL_STAN, 10, 2, 0, &st) != G4R_OK) return 33;
  if (g4r_bl_vstan_set(st, 0, f, 10, w4, 3) != G4R_ERR_STATE) return 34;
  if (g4r_bl_destroy(st) != G4R_OK) return 35;
  if (g4r_bl_destroy(h) != G4R_OK) return 36;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_vstan_abi(tmp_path):
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
