"""CPU tests of the session baselines (DESIGN §3j): oracle/baselines_oracle.py against the reference's recorded runs
(tests/golden/baselines: kept ItemKNN sims bitwise, tie-aware at the n_sims / top_n boundary, predict_next vectors exact), and the
Python surface -- baselines.Pop / SessionPop / ItemKNN, evaluate_gpu / evaluate_events with a baseline, run.py --baseline -- on a
CPU double of _lib.Baselines backed by the oracle.  The C ABI from a C99 caller at the end.  The device path is tested in
test_gpu_baselines.py."""
import contextlib
import io
import os
import pickle
import shutil
import subprocess

import numpy as np
import pandas as pd
import pytest
import torch.multiprocessing as mp

import baselines_oracle as bo
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'baselines')
CASES = ['int_ids', 'str_messy']
KNN = {'knn_100_20_05': (100, 20, 0.5), 'knn_5_0_1': (5, 0, 1.0), 'knn_20_20_0': (20, 20, 0.0)}
POP = {'top100': (100, None), 'top3': (3, None), 'top100_bysession': (100, 'SessionId')}


class OracleBaselines(object):
    """_lib.Baselines on the host: the oracle's rows, scores and ranking behind the binding's methods and argument checks"""

    def __init__(self, kind, n_items, n_keep, device=0):
        self.kind, self.n_items, self.n_keep = kind, n_items, n_keep

    def knn_fit(self, offsets, items, a, b):
        rows = bo.knn_rows_from_factors(offsets, items, self.n_items, self.n_keep, np.asarray(a), np.asarray(b))
        idx = np.full((self.n_items, self.n_keep), -1, np.int32); sim = np.zeros((self.n_items, self.n_keep))
        ln = np.zeros(self.n_items, np.int32)
        for i, (j, v) in rows.items():
            idx[i, :len(j)] = j; sim[i, :len(j)] = v; ln[i] = len(j)
        self.rows = (idx, sim, ln)
        return 0, 0, 0.0

    def set_pop(self, scores):
        assert np.count_nonzero(scores) <= self.n_keep
        self.pop = np.asarray(scores, dtype=np.float64)

    def rows_export(self):
        return tuple(a.copy() for a in self.rows)

    def rows_import(self, idx, sim, ln):
        self.rows = (np.asarray(idx), np.asarray(sim), np.asarray(ln))

    def model(self):
        if self.kind != 'itemknn':
            return self.pop
        idx, sim, ln = self.rows
        return self.n_items, {i: (idx[i, :ln[i]].astype(np.int64), sim[i, :ln[i]]) for i in range(self.n_items)}

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        name = [m for m, v in bo.MODES.items() if v == mode][0]
        cnt, ti, ts = bo.rank_events(self.kind, self.model(), self.n_items, items, offsets, n_history, name, cand, exclude_seen, k)
        rec, mrr = bo.sums(cnt, name, cut_off)
        return np.array(rec), np.array(mrr), len(cnt), cnt.astype(np.int32) if counts else None, ti, ts


@pytest.fixture
def double(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleBaselines)


def _golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + '.npz')))


def _train_csr(g):
    """the golden training data as session CSR of item indices (ids in unique() order, as the reference indexes them)"""
    sid, iid = g['train_sid'], g['train_iid']
    idx = pd.Index(g['itemids']).get_indexer(iid)
    codes = pd.Index(pd.unique(sid)).get_indexer(sid)
    order = np.argsort(codes, kind='stable')
    off = np.zeros(codes.max() + 2, np.int64)
    off[1:] = np.cumsum(np.bincount(codes))
    return off, idx[order], len(g['itemids'])


def _tie_aware(got_i, got_s, want_i, want_s):
    """equal kept entries: the values bitwise, the items above the last kept value exactly, the items at it from one tie set"""
    assert len(got_i) == len(want_i)
    if not len(got_i):
        return
    np.testing.assert_array_equal(np.sort(got_s), np.sort(want_s))
    v = want_s.min()
    assert set(got_i[got_s > v]) == set(want_i[want_s > v])
    for i, s in zip(got_i[got_s > v], got_s[got_s > v]):
        assert s == want_s[want_i == i][0]


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('tag', list(KNN))
def test_oracle_knn_rows_and_predictions_match_the_reference(case, tag):
    g = _golden(case)
    off, items, n = _train_csr(g)
    rows = bo.knn_rows(off, items, n, *KNN[tag])
    full = bo.knn_rows(off, items, n, n, *KNN[tag][1:])              # every positive sim (the tie sets)
    for i in range(n):
        wi, ws = g[tag + '_idx'][i], g[tag + '_sim'][i]
        wi, ws = wi[wi >= 0], ws[wi >= 0]
        gi, gs = rows[i]
        _tie_aware(gi, gs, wi, ws)
        if len(ws):
            ties = set(full[i][0][full[i][1] == ws.min()])
            assert set(gi[gs == ws.min()]) <= ties and set(wi[ws == ws.min()]) <= ties
    pos = pd.Index(g['itemids'])
    for q, x in enumerate(pos.get_indexer(g['test_iid'])):
        got = bo.scores('itemknn', (n, rows), x, None)
        want = g[tag + '_pred'][q]
        diff = got != want
        if diff.any():                                              # only where the two kept different members of a boundary tie
            v = rows[x][1].min()
            assert np.all((got[diff] == v) | (want[diff] == v)) and np.all((got[diff] == 0) | (want[diff] == 0))


def test_counts_are_per_distinct_item_not_the_product():
    """(0 0 1) then (0 1): item 0's row gains 1 per occurrence of 0 for each distinct item of the session"""
    cnt = bo.cooccurrence(np.array([0, 3, 5]), np.array([0, 0, 1, 0, 1]), 2).toarray()
    assert cnt.tolist() == [[0, 3], [2, 0]]                          # c_s(i) * c_s(j) would give 2 + 1 = 3 for (1, 0)
    g = _golden('str_messy')
    off, items, n = _train_csr(g)
    assert any(len(set(items[off[s]:off[s + 1]])) < off[s + 1] - off[s] for s in range(len(off) - 1))


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('tag', list(POP))
def test_oracle_pop_and_sessionpop_match_the_reference(case, tag):
    g = _golden(case)
    top_n, by = POP[tag]
    tr = pd.DataFrame({'SessionId': g['train_sid'], 'ItemId': g['train_iid']})
    grp = tr.groupby('ItemId')
    supp = (grp.size() if by is None else grp[by].nunique()).reindex(g['itemids']).values
    dense = bo.pop_scores(supp, top_n)
    pos = pd.Index(g['itemids'])
    wi, ws = pos.get_indexer(g['pop_%s_ids' % tag]), g['pop_%s_score' % tag]
    keep = np.flatnonzero(dense)
    _tie_aware(keep, dense[keep], wi, ws)
    prefix, last = [], None
    for q, (s, x) in enumerate(zip(g['test_sid'], pos.get_indexer(g['test_iid']))):
        prefix = prefix + [x] if s == last else [x]
        last = s
        for kind in ('pop', 'sessionpop'):
            got, want = bo.scores(kind, dense, x, prefix), g['%s_%s_pred' % (kind, tag)][q]
            diff = got != want
            if diff.any():
                assert top_n < len(supp) and np.all(np.isin(np.flatnonzero(diff), np.flatnonzero(supp / (supp + 1) == ws.min())))


# ---- the Python surface on the double ------------------------------------------------------------------------------------
def _frames(g):
    tr = pd.DataFrame({'SessionId': g['train_sid'], 'ItemId': g['train_iid'], 'Time': g['train_time']})
    return tr


@pytest.mark.parametrize('case', CASES)
def test_classes_fit_and_predict_next(double, case):
    import baselines
    g = _golden(case)
    tr = _frames(g)
    before = tr.copy()
    ids = g['itemids']
    knn = baselines.ItemKNN(n_sims=5, lmbd=0, alpha=1.0)
    knn.fit(tr)
    pd.testing.assert_frame_equal(tr, before)                        # fit leaves the caller's frame alone
    assert list(knn.itemidmap.index) == list(ids) and knn.n_items == len(ids) and knn.error_during_train is False
    supp = tr.groupby('ItemId').size().reindex(ids).values
    v = g['pop_top3_score'].min()
    ties = supp / (supp + 1) == v                                   # the items the top 3 may take at its boundary
    for kind, m, tag in (('pop', baselines.Pop(top_n=3), 'pop_top3'), ('sessionpop', baselines.SessionPop(top_n=3), 'sessionpop_top3')):
        m.fit(tr)
        for q, (s, x) in enumerate(zip(g['test_sid'], g['test_iid'])):
            got = m.predict_next(s, x, ids)
            assert list(got.index) == list(ids)
            want = g[tag + '_pred'][q]
            diff = got.values != want
            # only where the two kept different members of the boundary tie: one side has its Pop score, the other not
            assert np.all(ties[diff]) and np.all(np.abs(got.values[diff] - want[diff]) == v)
    for q, (s, x) in enumerate(zip(g['test_sid'], g['test_iid'])):
        got, want = knn.predict_next(s, x, ids).values, g['knn_5_0_1_pred'][q]
        diff = got != want
        i = knn.itemidmap[x]
        assert not diff.any() or np.all((got[diff] == knn.rows[1][i, knn.rows[2][i] - 1]) | (want[diff] == knn.rows[1][i, knn.rows[2][i] - 1]))
    with pytest.raises(KeyError):
        knn.predict_next(1, 'no such item' if case == 'str_messy' else -5, ids)


def _messy_test(train, seed):
    rs = np.random.RandomState(seed)
    te = make_sessions(n_items=60, n_events=500, seed=seed + 1)
    te['SessionId'] += 10000
    te.loc[rs.rand(len(te)) < 0.05, 'ItemId'] = 999999                      # unknown: dropped by the merge
    rep = np.flatnonzero(rs.rand(len(te)) < 0.2)
    rep = rep[(rep > 0) & (te.SessionId.values[rep] == te.SessionId.values[np.maximum(rep - 1, 0)])]
    te.loc[rep, 'ItemId'] = te.ItemId.values[rep - 1]                       # repeated items
    single = pd.DataFrame({'SessionId': [20000, 20001], 'ItemId': train.ItemId.values[:2], 'Time': [1.0, 2.0]})
    te = pd.concat([te, single], ignore_index=True)
    tied = te.SessionId == te.SessionId.iloc[3]
    te.loc[tied, 'Time'] = te.loc[tied, 'Time'].iloc[0]
    return te.sample(frac=1.0, random_state=seed).reset_index(drop=True)


@pytest.fixture(scope='module')
def fitted():
    import baselines
    mp_ = pytest.MonkeyPatch()
    mp_.setattr(_lib, 'Baselines', OracleBaselines)
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    models = {'pop': baselines.Pop(top_n=10), 'sessionpop': baselines.SessionPop(top_n=10), 'itemknn': baselines.ItemKNN(n_sims=8)}
    for m in models.values():
        m.fit(train.copy())
    mp_.undo()
    return models, train


def _expected(model, kind, df, mode, cand=None, exclude_seen=False, hist_n=None):
    """ranks replayed on the sorted, merged frame with the oracle, independent of evaluation.py's row mapping"""
    dev = model._device()
    items = df.ItemIdx.values
    off = np.zeros(df.SessionId.nunique() + 1, np.int64)
    off[1:] = df.groupby('SessionId', sort=True).size().cumsum()
    cnt, _, _ = bo.rank_events(kind, dev.model(), model.n_items, items, off, hist_n, mode, cand, exclude_seen)
    return bo.ranks(cnt, mode)


def _sorted(model, te):
    df = pd.merge(te, pd.DataFrame({'ItemIdx': model.itemidmap.values, 'ItemId': model.itemidmap.index}), on='ItemId', how='inner')
    df = df.sort_values(['SessionId', 'Time', 'ItemId']).reset_index(drop=True)
    first = np.r_[True, df.SessionId.values[1:] != df.SessionId.values[:-1]]
    return df, ~first


@pytest.mark.parametrize('kind', ['pop', 'sessionpop', 'itemknn'])
@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_evaluate_events_frame_ranks_and_sums(double, fitted, kind, mode):
    import evaluation
    models, train = fitted
    m = models[kind]
    te = _messy_test(train, seed=11)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(m, te.copy(), cut_off=[1, 5, 20], mode=mode, k=4)
        rec, mrr = evaluation.evaluate_gpu(m, te.copy(), cut_off=[1, 5, 20], mode=mode, batch_size=3)
    df, scored = _sorted(m, te)
    ev = res['events']
    assert list(ev.columns) == ['SessionId', 'Time', 'input_item', 'ItemId', 'rank'] and len(ev) == scored.sum()
    np.testing.assert_array_equal(ev.SessionId.values, df.SessionId.values[scored])
    np.testing.assert_array_equal(ev.ItemId.values, df.ItemId.values[scored])
    np.testing.assert_array_equal(ev.input_item.values, df.ItemId.values[np.flatnonzero(scored) - 1])
    np.testing.assert_array_equal(ev['rank'].values, _expected(m, kind, df, mode))
    assert res['recall'] == rec and res['mrr'] == mrr
    r = ev['rank'].values
    for j, c in enumerate([1, 5, 20]):
        assert abs(res['recall'][j] - np.mean(r <= c)) <= 1e-12
        assert abs(res['ndcg'][j] - np.mean(np.where(r <= c, 1.0 / np.log2(r + 1.0), 0.0))) <= 1e-12
    assert res['topk_scores'].dtype == np.float64 and res['topk_items'].shape == (len(ev), 4)
    assert set(res['topk_items'].reshape(-1)) <= set(m.itemidmap.index)
    assert res['coverage'] == len(np.unique(m.itemidmap[res['topk_items'].reshape(-1)].values)) / m.n_items


@pytest.mark.parametrize('kind', ['pop', 'sessionpop', 'itemknn'])
def test_items_exclude_seen_history_and_batch_size(double, fitted, kind):
    import evaluation
    models, train = fitted
    m = models[kind]
    te = _messy_test(train, seed=5)
    ids = m.itemidmap.index.values
    tgt = te[te.ItemId.isin(ids)].ItemId.values
    cand = list(ids[::3]) + [ids[0], ids[0]]                                 # duplicates count
    cand = [c for c in cand if c != tgt[5]]                                  # a listed target and an unlisted one
    df, scored = _sorted(m, te)
    out = {}
    with contextlib.redirect_stdout(io.StringIO()):
        for bs in (1, 100, 512):
            out[bs] = evaluation.evaluate_events(m, te.copy(), items=cand, cut_off=[3, 10], mode='conservative', batch_size=bs, k=3)
        seen = evaluation.evaluate_events(m, te.copy(), cut_off=[5], exclude_seen=True, k=5)
        with pytest.raises(KeyError):
            evaluation.evaluate_gpu(m, te.copy(), items=[123456789])
        with pytest.raises(NotImplementedError):
            evaluation.evaluate_gpu(m, te.copy(), mode='random')
        with pytest.raises(ValueError):
            evaluation.evaluate_events(m, te.copy(), items=list(ids[:2]) * 3, k=3)
    for bs in (100, 512):
        pd.testing.assert_frame_equal(out[bs]['events'], out[1]['events'])
        np.testing.assert_array_equal(out[bs]['topk_items'], out[1]['topk_items'])
        assert out[bs]['recall'] == out[1]['recall'] and out[bs]['mrr'] == out[1]['mrr']
    np.testing.assert_array_equal(out[1]['events']['rank'].values, _expected(m, kind, df, 'conservative', cand=m.itemidmap[cand].values))
    assert set(out[1]['topk_items'].reshape(-1)) <= set(cand)
    r = seen['events']['rank'].values
    np.testing.assert_array_equal(r, _expected(m, kind, df, 'standard', exclude_seen=True))
    assert np.isinf(r).any()                                                 # repeated items: exclude_seen misses
    # history: the first half of every test session's events come first; only the rest are counted
    pos, size = df.groupby('SessionId').cumcount(), df.groupby('SessionId').SessionId.transform('size')
    hist = df[pos < size // 2][['SessionId', 'ItemId', 'Time']]
    rest = df.drop(hist.index)[['SessionId', 'ItemId', 'Time']]
    with contextlib.redirect_stdout(io.StringIO()):
        h = evaluation.evaluate_events(m, rest.copy(), cut_off=[5], history=hist.copy())
    sids = np.sort(rest.SessionId.unique())
    both = pd.concat([df[df.index.isin(hist.index)], df[~df.index.isin(hist.index)]]).sort_values('SessionId', kind='stable')
    both = both[both.SessionId.isin(sids)]
    nh = hist.groupby('SessionId').size().reindex(sids, fill_value=0).values
    assert len(h['events']) == sum(max(0, n - max(k_, 1)) for n, k_ in zip(both.groupby('SessionId').size().values, nh))
    np.testing.assert_array_equal(h['events']['rank'].values, _expected(m, kind, both, 'standard', hist_n=nh))


def test_pickle_round_trip_without_the_handle(double, fitted, tmp_path):
    import evaluation
    models, train = fitted
    te = _messy_test(train, seed=9)
    for m in models.values():
        with contextlib.redirect_stdout(io.StringIO()):
            want = evaluation.evaluate_gpu(m, te.copy(), cut_off=[5, 20])
        assert '_dev' in m.__dict__
        m2 = pickle.loads(pickle.dumps(m))
        assert '_dev' not in m2.__dict__
        with contextlib.redirect_stdout(io.StringIO()):
            assert evaluation.evaluate_gpu(m2, te.copy(), cut_off=[5, 20]) == want
        if hasattr(m, 'rows'):
            for a, b in zip(m.rows, m2._device().rows):
                np.testing.assert_array_equal(a, b)


def _gloo_worker(rank, world, port, model, test, q):
    import sys
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle')); sys.path.insert(0, os.path.join(ROOT, 'tests'))
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    import torch.distributed as dist
    dist.init_process_group('gloo', rank=rank, world_size=world)
    import evaluation
    m, te = pd.read_pickle(model), pd.read_pickle(test)
    got = []
    for fn in (evaluation.evaluate_gpu, evaluation.evaluate_events):
        try:
            fn(m, te)
            got.append('returned')
        except NotImplementedError:
            got.append('NotImplementedError')
    q.put((rank, got))
    dist.barrier()
    dist.destroy_process_group()


def test_two_process_gloo_job_refuses(fitted, tmp_path):
    models, train = fitted
    pd.to_pickle(models['itemknn'], str(tmp_path / 'm.pickle'))
    _messy_test(train, seed=8).to_pickle(str(tmp_path / 'test.pickle'))
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29400 + os.getpid() % 150
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, str(tmp_path / 'm.pickle'), str(tmp_path / 'test.pickle'), q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = dict(q.get(timeout=5) for _ in range(2))
    assert res[0] == res[1] == ['NotImplementedError', 'NotImplementedError']


def test_run_py_baseline(double, tmp_path, capsys):
    import run
    df = make_sessions(n_items=40, n_events=800, seed=4)
    tr, te = df[df.SessionId < 200], df[df.SessionId >= 200]
    tr.to_csv(tmp_path / 'tr.tsv', sep='\t', index=False); te.to_csv(tmp_path / 'te.tsv', sep='\t', index=False)
    run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'itemknn', '-ps', 'n_sims=7,lmbd=0,alpha=1.0', '-t', str(tmp_path / 'te.tsv'),
              '-m', '5', '20', '-e', 'conservative', '--exclude_seen', '-lpm'])
    out = capsys.readouterr().out
    assert 'Creating ItemKNN model' in out and 'Total training time' in out and 'Recall@20:' in out and 'PRIMARY METRIC:' in out
    import baselines
    import evaluation
    m = baselines.ItemKNN(n_sims=7, lmbd=0, alpha=1.0)
    m.fit(run.load_data(str(tmp_path / 'tr.tsv'), run.build_parser().parse_args([str(tmp_path / 'tr.tsv')])))
    assert m.n_sims == 7 and type(m.lmbd) is int and type(m.alpha) is float
    capsys.readouterr()
    for bad in (['-pf', 'x.py'], ['-l'], ['--load_checkpoint', 'c.npz'], ['--fit_more'], ['-s', 'm.pickle'], ['--save_checkpoint', 'c.npz']):
        with pytest.raises(SystemExit):
            run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'pop'] + bad)
        assert 'ERROR' in capsys.readouterr().out
    del evaluation


SRC = r'''
#include <stdio.h>
#include "g4r.h"

int main(void) {
  double r[1] = {0.0}, m[1] = {0.0}, d[1] = {0.0};
  int32_t i[1] = {0}, c[1] = {20};
  int64_t o[2] = {0, 1}, n = 0;
  g4r_baselines* out = NULL;
  int (*ev)(g4r_baselines*, const int32_t*, int64_t, const int64_t*, int64_t, const int32_t*, int32_t, const int32_t*, int32_t,
            const int32_t*, int64_t, int32_t, int32_t, double*, double*, int64_t*, int32_t*, int32_t*, double*) = g4r_bl_evaluate;
  if (g4r_bl_create(7, 10, 5, 0, &out) != G4R_ERR_INVALID || out != NULL) return 1;
  if (g4r_bl_create(G4R_BL_ITEMKNN, 10, 5000, 0, &out) != G4R_ERR_INVALID) return 2;
  if (g4r_bl_last_error(NULL)[0] == 0) return 3;
  if (g4r_bl_knn_fit(NULL, o, 1, i, 1, d, d, NULL, NULL, NULL) != G4R_ERR_INVALID) return 4;
  if (g4r_bl_set_pop(NULL, d, 1) != G4R_ERR_INVALID) return 5;
  if (g4r_bl_rows_export(NULL, i, d, i) != G4R_ERR_INVALID || g4r_bl_rows_import(NULL, i, d, i) != G4R_ERR_INVALID) return 6;
  if (ev(NULL, i, 1, o, 1, NULL, 0, c, 1, NULL, 0, 0, 0, r, m, &n, NULL, NULL, NULL) != G4R_ERR_INVALID) return 7;
  if (g4r_bl_destroy(NULL) != G4R_OK) return 8;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_baselines_abi(tmp_path):
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
