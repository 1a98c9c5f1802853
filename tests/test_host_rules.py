"""CPU tests of the rule-based baselines (DESIGN §3q): tests/rules_oracle.py against hand-computed weights ('div' weights, the
steps cut-off, i = j pairs dropped while repeats elsewhere count, time ties by row order, AR's occ * occ against ItemKNN's cnt,
SR(1, 'same') against transition counts), baselines.SR / AR's fit and predict_next against the oracle on messy data, and the
Python surface -- evaluate_gpu / evaluate_events, pickles, run.py --baseline sr / ar -- on a CPU double of _lib.Baselines backed by
the oracle.  The binding's refusals and the C ABI from a C99 caller at the end.  The device path is tested in test_gpu_rules.py."""
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
import rules_oracle as ro
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_session_arrays, make_sessions
from test_host_baselines import OracleBaselines

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class OracleRules(OracleBaselines):
    """_lib.Baselines('sr' / 'ar', ...) on the host: the oracle's rows behind the binding's methods; ranked as ItemKNN rows"""

    def rules_fit(self, offsets, items, steps=None, weighting=None):
        self.fit_args = (np.array(offsets), np.array(items), steps, weighting)
        self.rows = ro.dense(ro.rows(offsets, items, self.n_items, self.n_keep, steps, weighting), self.n_items, self.n_keep)
        return 0, 0, 0.0

    def model(self):
        idx, sim, ln = self.rows
        return self.n_items, {i: (idx[i, :ln[i]].astype(np.int64), sim[i, :ln[i]]) for i in range(self.n_items)}

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        name = [m for m, v in bo.MODES.items() if v == mode][0]
        cnt, ti, ts = bo.rank_events('itemknn', self.model(), self.n_items, items, offsets, n_history, name, cand, exclude_seen, k)
        rec, mrr = bo.sums(cnt, name, cut_off)
        return np.array(rec), np.array(mrr), len(cnt), cnt.astype(np.int32) if counts else None, ti, ts


@pytest.fixture
def double(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleRules)


def _W(sessions, n_items, steps=None, weighting=None):
    off = np.r_[0, np.cumsum([len(s) for s in sessions])]
    return ro.counts(off, np.concatenate([np.asarray(s, np.int64) for s in sessions]), n_items, steps, weighting)


# ---- the oracle by hand --------------------------------------------------------------------------------------------------
def test_div_weights():
    assert [ro.scale(s, 'div') for s in (1, 2, 3, 4, 10, 20)] == [1, 2, 6, 12, 2520, 232792560]
    assert ro.scale(10, 'same') == 1 and ro.scale(None, None) == 1
    W = _W([[0, 1, 2]], 3, 2, 'div')                                      # L = 2: d = 1 adds 2, d = 2 adds 1
    assert W == [{1: 2, 2: 1}, {2: 2}, {}]
    r = ro.rows([0, 3], [0, 1, 2], 3, 20, 2, 'div')
    assert r[0][0].tolist() == [1, 2] and r[0][1].tolist() == [1.0, 0.5] and r[2][0].tolist() == []
    r = ro.rows([0, 4], [0, 1, 2, 3], 4, 20, 3, 'div')                   # L = 6: 1, 1/2, 1/3 exactly as W / 6
    assert r[0][1].tolist() == [1.0, 0.5, 2.0 / 6.0] and r[0][1][2] == float(2) / 6.0
    assert _W([[0, 1, 2]], 3, 2, 'same') == [{1: 1, 2: 1}, {2: 1}, {}]


def test_steps_cut_off():
    s = [[0, 1, 2, 3, 4]]
    assert 3 not in _W(s, 5, 2, 'same')[0] and _W(s, 5, 3, 'same')[0] == {1: 1, 2: 1, 3: 1}
    assert _W(s, 5, 20, 'div')[0] == {1: 232792560, 2: 232792560 // 2, 3: 232792560 // 3, 4: 232792560 // 4}
    assert _W([[0, 1], [2, 0]], 3, 20, 'same') == [{1: 1}, {}, {0: 1}]   # nothing crosses a session boundary


def test_self_pairs_dropped_repeats_elsewhere_count():
    # (0 0 1), steps 2, 'div' (L = 2): 0 -> 0 dropped; 0@1 -> 1@3 (d = 2) adds 1, 0@2 -> 1@3 (d = 1) adds 2
    assert _W([[0, 0, 1]], 2, 2, 'div') == [{1: 3}, {}]
    r = ro.rows([0, 3], [0, 0, 1], 2, 5, 2, 'div')
    assert r[0][1].tolist() == [1.5] and len(r[1][0]) == 0
    # the repeat blocks nothing: (0 1 0 1) steps 3 'same' gives 0 -> 1 three times (d 1, 3 and 1), 1 -> 0 once
    assert _W([[0, 1, 0, 1]], 2, 3, 'same') == [{1: 3}, {0: 1}]
    assert _W([[0, 1, 0, 1]], 2, None, None) == [{1: 4}, {0: 4}]


def test_time_ties_by_row_order():
    off, items = ro.sequences(['a', 'b', 'a', 'a', 'b'], [5, 7, 6, 4, 8], [3.0, 1.0, 1.0, 1.0, 0.0])
    # a: rows 0 (t 3), 2 (t 1), 3 (t 1) -> 6, 4, 5; b: rows 1 (t 1), 4 (t 0) -> 8, 7
    assert off.tolist() == [0, 3, 5] and items.tolist() == [6, 4, 5, 8, 7]


def test_ar_is_occ_times_occ_not_itemknn_cnt():
    assert _W([[0, 0, 1]], 2) == [{1: 2}, {0: 2}]
    knn = bo.cooccurrence(np.array([0, 3]), np.array([0, 0, 1]), 2).toarray()
    assert knn.tolist() == [[0, 2], [1, 0]]                                # ItemKNN: occ(1) * [0 in s] = 1
    items, off, _, _ = make_session_arrays(30, 600, seed=2, max_len=9)
    items = items.copy()
    rep = np.flatnonzero(np.random.RandomState(0).rand(len(items)) < 0.3)
    items[rep[rep > 0]] = items[rep[rep > 0] - 1]
    sess = np.repeat(np.arange(len(off) - 1), np.diff(off))
    occ = np.zeros((len(off) - 1, 30), np.int64)
    np.add.at(occ, (sess, items), 1)
    want = occ.T @ occ
    np.fill_diagonal(want, 0)
    got = np.zeros((30, 30), np.int64)
    for i, row in enumerate(_W([items[off[s]:off[s + 1]] for s in range(len(off) - 1)], 30)):
        for j, c in row.items():
            got[i, j] = c
    np.testing.assert_array_equal(got, want)
    assert (want != bo.cooccurrence(off, items, 30).toarray()).any()


def test_sr_1_same_is_transition_counts():
    items, off, _, _ = make_session_arrays(25, 700, seed=6, max_len=10)
    items = items.copy()
    items[5::7] = items[4::7][:len(items[5::7])]                          # self-transitions
    T = np.zeros((25, 25), np.int64)
    for s in range(len(off) - 1):
        x = items[off[s]:off[s + 1]]
        np.add.at(T, (x[:-1], x[1:]), 1)
    np.fill_diagonal(T, 0)
    r = ro.rows(off, items, 25, 1024, 1, 'same')
    for i in range(25):
        j = np.flatnonzero(T[i])
        o = np.lexsort((j, -T[i, j]))
        assert r[i][0].tolist() == j[o].tolist() and r[i][1].tolist() == T[i, j[o]].astype(float).tolist()


# ---- the classes on the double ---------------------------------------------------------------------------------------------
def _messy_train(seed=3, n_items=50, n_events=1500):
    rs = np.random.RandomState(seed)
    df = make_sessions(n_items=n_items, n_events=n_events, seed=seed, item_as_str=True)
    rep = np.flatnonzero(rs.rand(len(df)) < 0.2)
    rep = rep[(rep > 0) & (df.SessionId.values[rep] == df.SessionId.values[np.maximum(rep - 1, 0)])]
    df.loc[rep, 'ItemId'] = df.ItemId.values[rep - 1]                    # repeated items
    df['Time'] = np.floor(df.Time.values / 300.0)                          # many equal times, inside sessions too
    df['SessionId'] = 's' + (df.SessionId * 7919 % 10007).astype(str)      # string ids, not in time order
    return df.sample(frac=1.0, random_state=seed).reset_index(drop=True)   # unsorted rows


def _model(kind, **kw):
    import baselines
    return baselines.SR(**kw) if kind == 'sr' else baselines.AR(**kw)


@pytest.mark.parametrize('kind, kw', [('sr', dict(steps=10, weighting='div', pruning=7)), ('sr', dict(steps=3, weighting='same', pruning=5)),
                                      ('ar', dict(pruning=6))])
def test_fit_and_predict_next_equal_the_oracle(double, kind, kw):
    tr = _messy_train()
    before = tr.copy()
    m = _model(kind, **kw)
    m.fit(tr)
    pd.testing.assert_frame_equal(tr, before)                              # fit leaves the caller's frame alone
    assert list(m.itemidmap.index) == list(pd.unique(tr.ItemId.values)) and m.error_during_train is False
    off, items = ro.sequences(tr.SessionId.values, m.itemidmap[tr.ItemId.values].values, tr.Time.values)
    dev = m._device()
    np.testing.assert_array_equal(dev.fit_args[0], off)
    np.testing.assert_array_equal(dev.fit_args[1], items)
    assert dev.fit_args[2:] == ((kw['steps'], kw['weighting']) if kind == 'sr' else (None, None))
    want = ro.rows(off, items, m.n_items, kw['pruning'], kw.get('steps'), kw.get('weighting'))
    for a, b in zip(m.rows, ro.dense(want, m.n_items, kw['pruning'])):
        assert a.tobytes() == b.tobytes()
    assert m.fit_stats == (0, 0, 0.0)
    ids = m.itemidmap.index.values
    for x in ids[::7]:
        got = m.predict_next('t', x, ids)
        i = m.itemidmap[x]
        s = np.zeros(m.n_items)
        s[want[i][0]] = want[i][1]
        assert list(got.index) == list(ids) and got.values.tobytes() == s.tobytes()
    with pytest.raises(KeyError):
        m.predict_next('t', 'no such item', ids)


@pytest.mark.parametrize('kw', [dict(steps=0), dict(steps=21), dict(steps=2.0), dict(steps=True), dict(weighting='log'),
                                dict(pruning=0), dict(pruning=1025)])
def test_sr_fit_refuses_bad_parameters(double, kw):
    m = _model('sr', **kw)
    with pytest.raises(ValueError):
        m.fit(make_sessions(n_items=20, n_events=100, seed=1))
    assert '_dev' not in m.__dict__


@pytest.mark.parametrize('pruning', [0, 1025, 3.5])
def test_ar_fit_refuses_bad_pruning(double, pruning):
    m = _model('ar', pruning=pruning)
    with pytest.raises(ValueError):
        m.fit(make_sessions(n_items=20, n_events=100, seed=1))
    assert '_dev' not in m.__dict__


@pytest.fixture(scope='module')
def fitted():
    mp_ = pytest.MonkeyPatch()
    mp_.setattr(_lib, 'Baselines', OracleRules)
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    models = {'sr': _model('sr', steps=5, weighting='div', pruning=8), 'ar': _model('ar', pruning=8)}
    for m in models.values():
        m.fit(train.copy())
    mp_.undo()
    return models, train


def _test_frame(seed):
    rs = np.random.RandomState(seed)
    te = make_sessions(n_items=60, n_events=400, seed=seed + 1)
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


def _oracle_rows(m, train):
    off, items = ro.sequences(train.SessionId.values, m.itemidmap[train.ItemId.values].values, train.Time.values)
    steps, weighting = m._steps()
    return m.n_items, ro.rows(off, items, m.n_items, m.pruning, steps, weighting)


@pytest.mark.parametrize('kind', ['sr', 'ar'])
@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_evaluate_events_frame_ranks_and_sums(double, fitted, kind, mode):
    import evaluation
    models, train = fitted
    m = models[kind]
    te = _test_frame(seed=11)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(m, te.copy(), cut_off=[1, 5, 20], mode=mode, k=4)
        rec, mrr = evaluation.evaluate_gpu(m, te.copy(), cut_off=[1, 5, 20], mode=mode)
    df, off = _sorted(m, te)
    ev = res['events']
    assert len(ev) == len(df) - (len(off) - 1)
    cnt, ti, ts = bo.rank_events('itemknn', _oracle_rows(m, train), m.n_items, df.ItemIdx.values, off, None, mode, None, False, 4)
    np.testing.assert_array_equal(ev['rank'].values, bo.ranks(cnt, mode))
    np.testing.assert_array_equal(res['topk_items'], m.itemidmap.index.values[ti])
    np.testing.assert_array_equal(res['topk_scores'], ts)
    assert res['recall'] == rec and res['mrr'] == mrr
    hits, rrs = bo.sums(cnt, mode, [1, 5, 20])
    assert rec == [h / len(cnt) for h in hits] and mrr == [r / len(cnt) for r in rrs]


@pytest.mark.parametrize('kind', ['sr', 'ar'])
def test_items_exclude_seen_and_history(double, fitted, kind):
    import evaluation
    models, train = fitted
    m = models[kind]
    model = _oracle_rows(m, train)
    te = _test_frame(seed=5)
    ids = m.itemidmap.index.values
    cand = list(ids[::3]) + [ids[0], ids[0]]                               # duplicates count
    df, off = _sorted(m, te)
    with contextlib.redirect_stdout(io.StringIO()):
        a = evaluation.evaluate_events(m, te.copy(), items=cand, cut_off=[3, 10], mode='conservative', k=3)
        b = evaluation.evaluate_events(m, te.copy(), cut_off=[5], exclude_seen=True, k=5)
    cnt, ti, ts = bo.rank_events('itemknn', model, m.n_items, df.ItemIdx.values, off, None, 'conservative', m.itemidmap[cand].values, k=3)
    np.testing.assert_array_equal(a['events']['rank'].values, bo.ranks(cnt, 'conservative'))
    np.testing.assert_array_equal(a['topk_scores'], ts)
    cnt, ti, ts = bo.rank_events('itemknn', model, m.n_items, df.ItemIdx.values, off, None, 'standard', None, True, k=5)
    np.testing.assert_array_equal(b['events']['rank'].values, bo.ranks(cnt, 'standard'))
    np.testing.assert_array_equal(b['topk_items'], ids[ti])
    assert np.isinf(b['events']['rank'].values).any()
    pos, size = df.groupby('SessionId').cumcount(), df.groupby('SessionId').SessionId.transform('size')
    hist = df[pos < size // 2][['SessionId', 'ItemId', 'Time']]
    rest = df.drop(hist.index)[['SessionId', 'ItemId', 'Time']]
    with contextlib.redirect_stdout(io.StringIO()):
        h = evaluation.evaluate_events(m, rest.copy(), cut_off=[5], history=hist.copy())
    nh = hist.groupby('SessionId').size().reindex(np.sort(df.SessionId.unique()), fill_value=0).values
    cnt = bo.rank_events('itemknn', model, m.n_items, df.ItemIdx.values, off, nh)[0]
    np.testing.assert_array_equal(h['events']['rank'].values, bo.ranks(cnt, 'standard'))


def test_pickle_round_trip_without_the_handle(double, fitted):
    import evaluation
    models, train = fitted
    te = _test_frame(seed=9)
    for m in models.values():
        with contextlib.redirect_stdout(io.StringIO()):
            want = evaluation.evaluate_gpu(m, te.copy(), cut_off=[5, 20])
        assert '_dev' in m.__dict__
        m2 = pickle.loads(pickle.dumps(m))
        assert '_dev' not in m2.__dict__ and m2.fit_stats == m.fit_stats
        with contextlib.redirect_stdout(io.StringIO()):
            assert evaluation.evaluate_gpu(m2, te.copy(), cut_off=[5, 20]) == want
        for a, b in zip(m.rows, m2._device().rows):                         # re-uploaded by rows_import, not refitted
            assert a.tobytes() == b.tobytes()
        assert not hasattr(m2._device(), 'fit_args')


@pytest.mark.parametrize('kind, ps', [('sr', 'steps=10,weighting=div,pruning=20'), ('ar', 'pruning=20')])
def test_run_py_baseline_sr_ar(double, tmp_path, capsys, kind, ps):
    import run
    df = make_sessions(n_items=40, n_events=800, seed=4)
    tr, te = df[df.SessionId < 200], df[df.SessionId >= 200]
    tr.to_csv(tmp_path / 'tr.tsv', sep='\t', index=False); te.to_csv(tmp_path / 'te.tsv', sep='\t', index=False)
    run.main([str(tmp_path / 'tr.tsv'), '--baseline', kind, '-ps', ps, '-t', str(tmp_path / 'te.tsv'), '-m', '5', '20'])
    out = capsys.readouterr().out
    assert 'Creating %s model' % kind.upper() in out and 'Total training time' in out
    # the printed lines equal the oracle's on the run's own data
    args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv')])
    trd, ted = run.load_data(str(tmp_path / 'tr.tsv'), args), run.load_data(str(tmp_path / 'te.tsv'), args)
    ids = pd.Index(pd.unique(trd.ItemId.values))
    off, items = ro.sequences(trd.SessionId.values, ids.get_indexer(trd.ItemId.values), trd.Time.values)
    rows = ro.rows(off, items, len(ids), 20, *((10, 'div') if kind == 'sr' else (None, None)))
    ted = ted[ted.ItemId.isin(ids)].assign(ItemIdx=lambda f: ids.get_indexer(f.ItemId.values))
    ted = ted.sort_values(['SessionId', 'Time'], kind='stable')
    toff = np.r_[0, np.cumsum(ted.groupby('SessionId', sort=True).size().values)]
    cnt = bo.rank_events('itemknn', (len(ids), rows), len(ids), ted.ItemIdx.values, toff)[0]
    hits, rrs = bo.sums(cnt, 'standard', [5, 20])
    for q, c in enumerate((5, 20)):
        assert 'Recall@{}: {:.6f} MRR@{}: {:.6f}'.format(c, hits[q] / len(cnt), c, rrs[q] / len(cnt)) in out
    m = run._train_baseline(run.build_parser().parse_args([str(tmp_path / 'tr.tsv'), '--baseline', kind, '-ps', ps]))
    assert type(m.pruning) is int and (kind == 'ar' or (type(m.steps) is int and m.weighting == 'div'))
    with pytest.raises(SystemExit):
        run.main([str(tmp_path / 'tr.tsv'), '--baseline', kind, '-t', str(tmp_path / 'te.tsv'), '--rest_of_session'])
    assert 'ERROR' in capsys.readouterr().out


# ---- the binding's refusals ------------------------------------------------------------------------------------------------
def _bare(kind, n_items=5, n_keep=3):
    dev = object.__new__(_lib.Baselines)                                   # no library behind it: a call would fail otherwise
    dev.kind, dev.n_items, dev.n_keep, dev.h = kind, n_items, n_keep, None
    return dev


def test_rules_bound():
    off, it = [0, 3, 5], [0, 1, 0, 2, 0]
    assert _lib.rules_bound(off, it, 3, None, None) == 3 + 3 + 2           # item 0: twice in a 3-event session, once in a 2-event one
    assert _lib.rules_bound(off, it, 3, 1, 'same') == 3 * 1
    assert _lib.rules_bound(off, it, 3, 20, 'div') == 3 * 2 * 232792560    # min(steps, longest session - 1) = 2
    assert _lib.rules_bound([0], [], 3, 5, 'div') == 0
    assert _lib.rules_scale(20, 'div') == ro.scale(20, 'div') and _lib.rules_scale(20, 'same') == 1


def test_binding_refuses_bad_arguments_before_the_library(monkeypatch):
    ok = dict(session_offsets=[0, 2, 3], items=[0, 1, 1])
    sr, ar = _bare('sr'), _bare('ar')
    for bad in (dict(steps=0, weighting='div'), dict(steps=21, weighting='div'), dict(steps=None, weighting='div'),
                dict(steps=3, weighting='log'), dict(steps=3, weighting=None), dict(steps=2.5, weighting='same')):
        with pytest.raises(ValueError):
            sr.rules_fit(**dict(ok, **bad))
    for bad in (dict(steps=1), dict(weighting='div')):
        with pytest.raises(ValueError):
            ar.rules_fit(**dict(ok, **bad))
    for n_keep in (0, 1025):
        with pytest.raises(ValueError):
            _bare('sr', n_keep=n_keep).rules_fit(steps=2, weighting='div', **ok)
        with pytest.raises(ValueError):
            _bare('ar', n_keep=n_keep).rules_fit(**ok)
    with pytest.raises(ValueError):
        ar.rules_fit([0, 3, 2], [0, 1, 1])
    with pytest.raises(IndexError):
        ar.rules_fit([0, 2, 3], [0, 1, 5])
    # the overflow bound: refused at 2^63, passed on to the library (absent here: AttributeError) just below it
    monkeypatch.setattr(_lib, 'rules_bound', lambda *a: 1 << 63)
    for dev, kw in ((sr, dict(steps=20, weighting='div')), (ar, {})):
        with pytest.raises(ValueError, match='2\\^63'):
            dev.rules_fit(**dict(ok, **kw))
    monkeypatch.setattr(_lib, 'rules_bound', lambda *a: (1 << 63) - 1)
    with pytest.raises(AttributeError):
        sr.rules_fit(steps=20, weighting='div', **ok)
    assert _lib.BASELINE_KINDS['sr'] == 8 and _lib.BASELINE_KINDS['ar'] == 9 and 'g4r_bl_rules_fit' in _lib.EXPORTS


SRC = r'''
#include <stdio.h>
#include "g4r.h"

int main(void) {
  int64_t o[3] = {0, 2, 3}, bad_o[3] = {0, 3, 2}, pw = 0;
  int32_t it[3] = {0, 1, 1}, big[3] = {0, 1, 10};
  size_t sb = 0;
  float ms = 0.0f;
  g4r_baselines* h = NULL;
  int rc;
  int (*fit)(g4r_baselines*, const int64_t*, int64_t, const int32_t*, int64_t, int32_t, int32_t, int64_t*, size_t*, float*) = g4r_bl_rules_fit;
  if (G4R_BL_SR != 8 || G4R_BL_AR != 9) return 1;
  if (fit(NULL, o, 2, it, 3, 10, 0, NULL, NULL, NULL) != G4R_ERR_INVALID) return 2;
  if (g4r_bl_create(G4R_BL_SR, 10, 0, 0, &h) != G4R_ERR_INVALID || h != NULL) return 3;
  if (g4r_bl_create(G4R_BL_SR, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 4;
  if (g4r_bl_create(G4R_BL_AR, 10, 0, 0, &h) != G4R_ERR_INVALID || h != NULL) return 5;
  if (g4r_bl_create(G4R_BL_AR, 10, 1025, 0, &h) != G4R_ERR_INVALID || h != NULL) return 6;
  if (g4r_bl_create(G4R_BL_AR, 0, 20, 0, &h) != G4R_ERR_INVALID || h != NULL) return 7;
  if (g4r_bl_create(4, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 8;
  if (g4r_bl_create(7, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 9;
  if (g4r_bl_create(10, 10, 8, 0, &h) != G4R_ERR_INVALID || h != NULL) return 10;
  if (g4r_bl_last_error(NULL)[0] == 0) return 11;
  rc = g4r_bl_create(G4R_BL_SR, 10, 1024, 0, &h);
  if (rc == G4R_ERR_CUDA) { printf("ok %d (no device)\n", g4r_version()); return 0; }
  if (rc != G4R_OK) return 12;
  if (fit(h, NULL, 2, it, 3, 10, 0, NULL, NULL, NULL) != G4R_ERR_INVALID) return 13;
  if (fit(h, o, 2, NULL, 3, 10, 0, NULL, NULL, NULL) != G4R_ERR_INVALID) return 14;
  if (fit(h, o, 2, it, 3, 0, 0, NULL, NULL, NULL) != G4R_ERR_INVALID) return 15;
  if (fit(h, o, 2, it, 3, 21, 0, NULL, NULL, NULL) != G4R_ERR_INVALID) return 16;
  if (fit(h, o, 2, it, 3, 10, 2, NULL, NULL, NULL) != G4R_ERR_INVALID) return 17;
  if (fit(h, o, 2, it, 3, 10, -1, NULL, NULL, NULL) != G4R_ERR_INVALID) return 18;
  if (fit(h, bad_o, 2, it, 3, 10, 0, NULL, NULL, NULL) != G4R_ERR_INVALID) return 19;
  if (fit(h, o, 2, big, 3, 10, 0, NULL, NULL, NULL) != G4R_ERR_INDEX) return 20;
  if (g4r_bl_knn_fit(h, o, 2, it, 3, NULL, NULL, NULL, NULL, NULL) != G4R_ERR_STATE) return 21;
  if (g4r_bl_sknn_fit(h, o, 2, it, 3, NULL, 10, 0) != G4R_ERR_STATE) return 22;
  if (g4r_bl_set_pop(h, NULL, 10) != G4R_ERR_STATE) return 23;
  if (g4r_bl_rows_export(h, it, NULL, it) != G4R_ERR_STATE) return 24;   /* not fitted yet */
  if (fit(h, o, 2, it, 3, 10, 0, &pw, &sb, &ms) != G4R_OK || pw != 1 || sb == 0) return 25;
  if (g4r_bl_destroy(h) != G4R_OK) return 26;
  h = NULL;
  if (g4r_bl_create(G4R_BL_AR, 10, 1, 0, &h) != G4R_OK) return 27;
  if (fit(h, o, 2, it, 3, 10, 0, NULL, NULL, NULL) != G4R_ERR_INVALID) return 28;
  if (fit(h, o, 2, it, 3, 0, 1, NULL, NULL, NULL) != G4R_ERR_INVALID) return 29;
  if (fit(h, o, 2, it, 3, 0, 0, &pw, NULL, NULL) != G4R_OK || pw != 2) return 30;
  if (g4r_bl_destroy(h) != G4R_OK) return 31;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_rules_abi(tmp_path):
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
