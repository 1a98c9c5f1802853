"""CPU tests of BPR-MF (DESIGN §3k): the vectorised draws against the reference's loop, oracle/bpr_oracle.py against the
reference's recorded runs (tests/golden/baselines/bpr_*.npz: U and I after the fit, the printed means, predict_next), the
numpy mean the session vector restates, and the Python surface -- baselines.BPR, evaluate_gpu / evaluate_events, pickles,
run.py --baseline bpr -- on a CPU double of _lib.Baselines backed by the oracle.  Argument refusals of the binding, and the C ABI
from a C99 caller at the end.  The device path is tested in test_gpu_bpr.py."""
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
import bpr_oracle as bpo
from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'baselines')
SEED = 7
PARAMS = {'f16_uniform': dict(n_factors=16, n_iterations=3, learning_rate=0.05),
          'f100_normal': dict(n_factors=100, n_iterations=3, learning_rate=0.02, lambda_session=0.01, lambda_item=0.02, sigma=0.1,
                              init_normal=True)}
FIXTURES = [(case, tag) for case in ('int_ids', 'str_messy') for tag in PARAMS]


class OracleBpr(object):
    """_lib.Baselines('bpr', ...) on the host: the oracle's fit and ranking behind the binding's methods"""

    def __init__(self, kind, n_items, n_keep, device=0):
        assert kind == 'bpr'
        self.kind, self.n_items, self.n_keep = kind, n_items, n_keep

    def bpr_begin(self, row_session, row_item, n_sessions, U, I, bI):
        self.rs, self.ri = np.asarray(row_session), np.asarray(row_item)
        self.U, self.I, self.bI = np.array(U, dtype=np.float64), np.array(I, dtype=np.float64), np.array(bI, dtype=np.float64)

    def bpr_iterate(self, perm, negrow, learning_rate, lambda_session, lambda_item, max_warps=1 << 30):
        self.U, self.I, means, levels = bpo.fit(self.rs, self.ri, self.U, self.I, self.bI, [(perm, negrow)], learning_rate, lambda_session,
                                                lambda_item)
        return means[0], levels[0], 0.0

    def bpr_export(self):
        return self.U.copy(), self.I.copy()

    def bpr_import(self, I, bI):
        self.I, self.bI = np.array(I, dtype=np.float64), np.array(bI, dtype=np.float64)

    def evaluate(self, items, offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        name = [m for m, v in bo.MODES.items() if v == mode][0]
        cnt, ti, ts = bpo.rank_events(self.I, self.bI, items, offsets, n_history, name, cand, exclude_seen, k)
        rec, mrr = bo.sums(cnt, name, cut_off)
        return np.array(rec), np.array(mrr), len(cnt), cnt.astype(np.int32) if counts else None, ti, ts


@pytest.fixture
def double(monkeypatch):
    monkeypatch.setattr(_lib, 'Baselines', OracleBpr)


def _golden(case, tag):
    return dict(np.load(os.path.join(GOLDEN, 'bpr_%s_%s.npz' % (case, tag))))


@pytest.mark.parametrize('n', [7, 150, 1000, 2 ** 31 - 1, 2 ** 32 + 5, 2 ** 33])
def test_vectorised_draws_consume_the_stream_as_the_loop(n):
    np.random.seed(3)
    want = bpo.iteration_draws_loop(500, n)
    state = np.random.get_state()
    np.random.seed(3)
    got = bpo.iteration_draws(500, n)
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])
    after = np.random.get_state()
    assert after[2:] == state[2:] and np.array_equal(after[1], state[1])


@pytest.mark.parametrize('length', [1, 2, 33, 700, 5000])
def test_session_vector_is_numpys_mean(length):
    """predict_next's uF = I[session].mean(axis=0) equals the sequential row sum / k the device forms, duplicates included"""
    rs = np.random.RandomState(length)
    I = rs.randn(40, 100) * 0.3
    prefix = rs.randint(0, 40, length)
    assert np.array_equal(bpo.session_vector(I, prefix), I[prefix].mean(axis=0))


@pytest.mark.parametrize('case,tag', FIXTURES)
def test_oracle_fit_and_class_match_the_reference(double, case, tag):
    """np.random.seed(s); BPR(...).fit(train): U and I within 1e-12 of the reference's, the printed means within 1e-12, and
    predict_next over the catalogue for the first test events within 1e-12"""
    import baselines
    g = _golden(case, tag)
    tr = pd.DataFrame({'SessionId': g['train_sid'], 'ItemId': g['train_iid'], 'Time': g['train_time']})
    np.random.seed(int(g['seed']))
    m = baselines.BPR(**PARAMS[tag])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        m.fit(tr)
    lines = buf.getvalue().splitlines()
    assert [int(x.split()[0]) for x in lines] == [0, 1, 2]
    np.testing.assert_allclose([float(x.split()[1]) for x in lines], g['means'], rtol=0, atol=1e-12)
    assert np.abs(m.U - g['U']).max() <= 1e-12 and np.abs(m.I - g['I']).max() <= 1e-12
    assert list(m.itemidmap.index) == list(g['itemids']) and m.n_sessions == g['U'].shape[0] and m.n_items == len(g['itemids'])
    assert np.all(m.bU == 0) and np.all(m.bI == 0)
    assert all(1 <= lv <= len(tr) for _, lv, _ in m.fit_stats)
    for q, (s, x) in enumerate(zip(g['test_sid'], g['test_iid'])):
        got = m.predict_next(s, x, g['itemids'])
        assert list(got.index) == list(g['itemids'])
        assert np.abs(got.values - g['pred'][q]).max() <= 1e-12
    assert m.current_session == g['test_sid'][-1] and m.session[-1] == m.itemidmap[g['test_iid'][-1]]


def test_level_is_the_longest_chain():
    """three events on one session: a chain of three; two sessions sharing no item: chains of one"""
    U, I, bI = np.zeros((2, 3)), np.ones((4, 3)) * 0.1, np.zeros(4)
    _, _, _, lv = bpo.fit(np.array([0, 0, 0]), np.array([0, 1, 2]), U, I, bI, [(np.arange(3), np.array([0, 1, 2]))], 0.1, 0, 0)
    assert lv == [3]
    _, _, _, lv = bpo.fit(np.array([0, 1]), np.array([0, 1]), U, I, bI, [(np.arange(2), np.array([0, 1]))], 0.1, 0, 0)
    assert lv == [1]


@pytest.fixture(scope='module')
def fitted():
    import baselines
    mp_ = pytest.MonkeyPatch()
    mp_.setattr(_lib, 'Baselines', OracleBpr)
    train = make_sessions(n_items=60, n_events=1200, seed=3)
    np.random.seed(1)
    m = baselines.BPR(n_factors=8, n_iterations=2, learning_rate=0.1)
    with contextlib.redirect_stdout(io.StringIO()):
        m.fit(train.copy())
    mp_.undo()
    return m, train


def _test_frame(train, seed):
    rs = np.random.RandomState(seed)
    te = make_sessions(n_items=60, n_events=300, seed=seed + 1)
    te['SessionId'] += 10000
    te.loc[rs.rand(len(te)) < 0.05, 'ItemId'] = 999999                      # unknown: dropped by the merge
    rep = np.flatnonzero(rs.rand(len(te)) < 0.2)
    rep = rep[(rep > 0) & (te.SessionId.values[rep] == te.SessionId.values[np.maximum(rep - 1, 0)])]
    te.loc[rep, 'ItemId'] = te.ItemId.values[rep - 1]                       # repeated items
    return te.sample(frac=1.0, random_state=seed).reset_index(drop=True)


def _sorted(model, te):
    df = pd.merge(te, pd.DataFrame({'ItemIdx': model.itemidmap.values, 'ItemId': model.itemidmap.index}), on='ItemId', how='inner')
    df = df.sort_values(['SessionId', 'Time', 'ItemId']).reset_index(drop=True)
    off = np.zeros(df.SessionId.nunique() + 1, np.int64)
    off[1:] = df.groupby('SessionId', sort=True).size().cumsum()
    return df, off


@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_evaluate_events_frame_ranks_and_sums(double, fitted, mode):
    import evaluation
    m, train = fitted
    te = _test_frame(train, seed=11)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(m, te.copy(), cut_off=[1, 5, 20], mode=mode, k=4)
        rec, mrr = evaluation.evaluate_gpu(m, te.copy(), cut_off=[1, 5, 20], mode=mode)
    df, off = _sorted(m, te)
    ev = res['events']
    assert list(ev.columns) == ['SessionId', 'Time', 'input_item', 'ItemId', 'rank'] and len(ev) == len(df) - (len(off) - 1)
    cnt, ti, ts = bpo.rank_events(m.I, m.bI, df.ItemIdx.values, off, None, mode, None, False, 4)
    np.testing.assert_array_equal(ev['rank'].values, bo.ranks(cnt, mode))
    np.testing.assert_array_equal(res['topk_items'], m.itemidmap.index.values[ti])
    np.testing.assert_array_equal(res['topk_scores'], ts)
    assert res['recall'] == rec and res['mrr'] == mrr


def test_items_exclude_seen_and_history(double, fitted):
    import evaluation
    m, train = fitted
    te = _test_frame(train, seed=5)
    ids = m.itemidmap.index.values
    cand = list(ids[::3]) + [ids[0], ids[0]]                                 # duplicates count
    df, off = _sorted(m, te)
    with contextlib.redirect_stdout(io.StringIO()):
        a = evaluation.evaluate_events(m, te.copy(), items=cand, cut_off=[3, 10], mode='conservative', k=3)
        b = evaluation.evaluate_events(m, te.copy(), cut_off=[5], exclude_seen=True, k=5)
    cnt = bpo.rank_events(m.I, m.bI, df.ItemIdx.values, off, None, 'conservative', m.itemidmap[cand].values)[0]
    np.testing.assert_array_equal(a['events']['rank'].values, bo.ranks(cnt, 'conservative'))
    cnt = bpo.rank_events(m.I, m.bI, df.ItemIdx.values, off, None, 'standard', None, True)[0]
    np.testing.assert_array_equal(b['events']['rank'].values, bo.ranks(cnt, 'standard'))
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
    cnt = bpo.rank_events(m.I, m.bI, both.ItemIdx.values, boff, nh)[0]
    np.testing.assert_array_equal(h['events']['rank'].values, bo.ranks(cnt, 'standard'))


def test_pickle_round_trip_without_the_handle(double, fitted):
    import evaluation
    m, train = fitted
    te = _test_frame(train, seed=9)
    with contextlib.redirect_stdout(io.StringIO()):
        want = evaluation.evaluate_gpu(m, te.copy(), cut_off=[5, 20])
    assert '_dev' in m.__dict__
    m2 = pickle.loads(pickle.dumps(m))
    assert '_dev' not in m2.__dict__
    for name in ('U', 'I', 'bI', 'bU', 'n_sessions', 'n_items', 'n_factors', 'init_normal'):
        assert np.array_equal(getattr(m2, name), getattr(m, name))
    with contextlib.redirect_stdout(io.StringIO()):
        assert evaluation.evaluate_gpu(m2, te.copy(), cut_off=[5, 20]) == want
    assert np.array_equal(m2._device().I, m.I) and np.array_equal(m2._device().bI, m.bI)


def test_run_py_baseline_bpr(double, tmp_path, capsys):
    import run
    df = make_sessions(n_items=40, n_events=800, seed=4)
    tr, te = df[df.SessionId < 200], df[df.SessionId >= 200]
    tr.to_csv(tmp_path / 'tr.tsv', sep='\t', index=False); te.to_csv(tmp_path / 'te.tsv', sep='\t', index=False)
    np.random.seed(0)
    run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'bpr', '-ps', 'n_factors=8,n_iterations=2,init_normal=False', '-t', str(tmp_path / 'te.tsv'),
              '-m', '5', '20'])
    out = capsys.readouterr().out
    assert 'Creating BPR model' in out and 'Total training time' in out and 'Recall@20:' in out
    lines = out.splitlines()
    assert any(x.startswith('0 -') for x in lines) and any(x.startswith('1 -') for x in lines)
    for flag, want in (('False', False), ('True', True)):
        args = run.build_parser().parse_args([str(tmp_path / 'tr.tsv'), '--baseline', 'bpr', '-ps', 'n_factors=4,n_iterations=1,init_normal=' + flag])
        with contextlib.redirect_stdout(io.StringIO()):
            m = run._train_baseline(args)
        assert m.init_normal is want and m.n_factors == 4 and type(m.n_factors) is int
    capsys.readouterr()
    with pytest.raises(SystemExit):
        run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'bpr', '-ps', 'init_normal=yes'])
    assert 'ERROR' in capsys.readouterr().out
    with pytest.raises(SystemExit):
        run.main([str(tmp_path / 'tr.tsv'), '--baseline', 'bpr', '-s', 'm.pickle'])
    assert 'ERROR' in capsys.readouterr().out


def test_binding_refuses_bad_arguments_before_the_library():
    dev = object.__new__(_lib.Baselines)
    dev.n_items, dev.n_keep, dev.bpr_rows, dev.bpr_sessions, dev.h = 5, 3, 4, 2, None
    with pytest.raises(ValueError):
        dev.bpr_begin([0, 1], [0, 1, 2], 2, np.zeros((2, 3)), np.zeros((5, 3)), np.zeros(5))
    with pytest.raises(ValueError):
        dev.bpr_begin([0, 1], [0, 1], 2, np.zeros((2, 4)), np.zeros((5, 3)), np.zeros(5))
    with pytest.raises(ValueError):
        dev.bpr_iterate(np.arange(3), np.zeros(3), 0.1, 0, 0)
    with pytest.raises(IndexError):
        dev.bpr_iterate(np.arange(4), np.array([0, 1, 5, 0]), 0.1, 0, 0)
    with pytest.raises(IndexError):
        dev.bpr_iterate(np.array([0, 1, 2, 2 ** 32]), np.zeros(4, np.int64), 0.1, 0, 0)
    with pytest.raises(ValueError):                     # 4 rows, 5 items: a negative draw could name a row that does not exist
        dev.bpr_begin([0, 1, 0, 1], [0, 1, 2, 3], 2, np.zeros((2, 3)), np.zeros((5, 3)), np.zeros(5))
    with pytest.raises(IndexError):                     # negrow == n_rows < n_items
        dev.bpr_iterate(np.arange(4), np.array([0, 1, 4, 0]), 0.1, 0, 0)
    with pytest.raises(ValueError):
        dev.bpr_import(np.zeros((5, 2)), np.zeros(5))


SRC = r'''
#include <stdio.h>
#include "g4r.h"

int main(void) {
  double d[4] = {0.0, 0.0, 0.0, 0.0}, mean = 0.0;
  int32_t i[2] = {0, 0};
  int64_t level = 0;
  float ms = 0.0f;
  g4r_baselines* out = NULL;
  if (G4R_BL_BPR != 3) return 1;
  if (g4r_bl_create(G4R_BL_BPR, 10, 1025, 0, &out) != G4R_ERR_INVALID || out != NULL) return 2;
  if (g4r_bl_create(G4R_BL_BPR, 10, 0, 0, &out) != G4R_ERR_INVALID || out != NULL) return 3;
  if (g4r_bl_create(4, 10, 8, 0, &out) != G4R_ERR_INVALID) return 4;
  if (g4r_bl_last_error(NULL)[0] == 0) return 5;
  if (g4r_bl_bpr_begin(NULL, i, i, 2, 1, d, d, d) != G4R_ERR_INVALID) return 6;
  if (g4r_bl_bpr_iterate(NULL, i, i, 0.01, 0.0, 0.0, 1, &mean, &level, &ms) != G4R_ERR_INVALID) return 7;
  if (g4r_bl_bpr_export(NULL, d, d) != G4R_ERR_INVALID) return 8;
  if (g4r_bl_bpr_import(NULL, d, d) != G4R_ERR_INVALID) return 9;
  printf("ok %d\n", g4r_version());
  return 0;
}
'''


def test_c99_caller_of_the_bpr_abi(tmp_path):
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
