"""CPU tests of evaluation.evaluate_events on the engine double (tests/oracle_engine.py, extended here by an eval_events made of
the double's own forward): row alignment with the sorted, merged test frame on messy data, ranks in all four modes, Recall / MRR
against evaluate_gpu, NDCG, coverage, items= and argument errors.  The device path is tested in test_gpu_eval_events.py."""
import contextlib
import io

import numpy as np
import pandas as pd
import pytest

from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
import oracle_engine


class EventsOracleEngine(oracle_engine.OracleEngine):
    """the engine double plus Engine.eval_events: the double's eval_schedule for the sums, its forward for the per-event counts
    and, from a copy of the same state, the top-k over the catalogue (or the distinct candidates)"""

    def eval_events(self, sched, cuts, mode=0, k=0):
        rec, mrr, n = self.eval_schedule(sched, cuts, mode)
        m, e = self.m, sched.export()
        H = [np.zeros((sched.batch_size, L), dtype=np.float32) for L in m.layers]
        cand = None if self.eval_items is None else np.unique(self.eval_items)
        counts, items, scores = [], [], []
        for s in range(sched.n_steps):
            M = int(e['M'][s])
            X, Y = e['X'][s, :M].astype(np.int64), e['Y'][s, :M].astype(np.int64)
            slots, zero = e['slots'][s, :M].astype(np.int64), (e['F'][s, :M] & 2) != 0
            H0 = [h.copy() for h in H]
            ycols = None if self.eval_items is None else np.concatenate([Y, self.eval_items])
            yhat = m.predict_step(X, H, slots=slots, zero=zero, Y=ycols)
            tg = yhat[np.arange(M), Y if ycols is None else np.arange(M)]
            others = yhat if ycols is None else yhat[:, M:]
            counts.append(np.stack([(others > tg[:, None]).sum(1), (others == tg[:, None]).sum(1)], 1))
            if k:
                sc = m.predict_step(X, H0, slots=slots, zero=zero, Y=cand)
                order = np.argsort(-sc, axis=1, kind='stable')[:, :k]
                items.append(order if cand is None else cand[order])
                scores.append(np.take_along_axis(sc, order, axis=1))
        counts = np.concatenate(counts).astype(np.int32)
        if not k:
            return rec, mrr, n, counts, None, None
        return rec, mrr, n, counts, np.concatenate(items).astype(np.int32), np.concatenate(scores).astype(np.float32)


def _install(monkeypatch, gru):
    def make(cfg, device=0):
        return EventsOracleEngine(cfg, oracle_engine.model_kwargs_of(gru), device)
    monkeypatch.setattr(_lib, 'Engine', make)


def _messy_test(train, seed):
    """test sessions with single-event sessions, item ids the model does not know, tied times and unsorted rows"""
    rs = np.random.RandomState(seed)
    te = make_sessions(n_items=60, n_events=400, seed=seed + 1)
    te['SessionId'] += 10000
    te.loc[rs.rand(len(te)) < 0.05, 'ItemId'] = 999999                      # unknown: dropped by the merge
    single = pd.DataFrame({'SessionId': [20000, 20001], 'ItemId': train.ItemId.values[:2], 'Time': [1.0, 2.0]})
    te = pd.concat([te, single], ignore_index=True)
    tied = te.SessionId == te.SessionId.iloc[3]
    te.loc[tied, 'Time'] = te.loc[tied, 'Time'].iloc[0]                      # tied times: the item id decides the order
    return te.sample(frac=1.0, random_state=seed).reset_index(drop=True)


@pytest.fixture(scope='module')
def trained():
    import gru4rec
    train = make_sessions(n_items=60, n_events=1500, seed=3)
    gru = gru4rec.GRU4Rec(loss='cross-entropy', final_act='softmax', layers=[12], batch_size=16, n_epochs=1, n_sample=0)
    mp = pytest.MonkeyPatch()
    _install(mp, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(train.copy())
    mp.undo()
    return gru, train


def _frame(gru, te):
    """the sorted, merged test frame and its scored rows (all but the first of each session)"""
    df = pd.merge(te, pd.DataFrame({'ItemIdx': gru.itemidmap.values, 'ItemId': gru.itemidmap.index}), on='ItemId', how='inner')
    df = df.sort_values(['SessionId', 'Time', 'ItemId']).reset_index(drop=True)
    first = np.r_[True, df.SessionId.values[1:] != df.SessionId.values[:-1]]
    return df, ~first


def _expected_ranks(gru, df, mode, batch_size, items=None):
    """per-row ranks replayed on the oracle: the schedule's steps mapped to rows by their exported inputs (independent of
    evaluate_events' own mapping), the reference's rank formula of oracle.ranks"""
    m = gru._engine.m                                         # the double's model (predict_step leaves the weights alone)
    off = np.zeros(df.SessionId.nunique() + 1, np.int32)
    off[1:] = df.groupby('SessionId').size().cumsum()
    sched = _lib.Schedule(df.ItemIdx.values, off, None, batch_size, 0, mode=1 | _lib.SCHED_POSITIONS)
    e, pos = sched.export(), sched.positions()
    H = [np.zeros((batch_size, L), dtype=np.float32) for L in m.layers]
    out = np.full(len(df), np.nan)
    for s in range(sched.n_steps):
        M = int(e['M'][s])
        X, Y = e['X'][s, :M].astype(np.int64), e['Y'][s, :M].astype(np.int64)
        np.testing.assert_array_equal(df.ItemIdx.values[pos[s, :M]], X)
        np.testing.assert_array_equal(df.ItemIdx.values[pos[s, :M] + 1], Y)
        ycols = None if items is None else np.concatenate([Y, items])
        yhat = m.predict_step(X, H, slots=e['slots'][s, :M].astype(np.int64), zero=(e['F'][s, :M] & 2) != 0, Y=ycols)
        out[pos[s, :M] + 1] = m.ranks(yhat, Y, mode, items)
    return out


@pytest.mark.parametrize('mode', ['standard', 'conservative', 'median', 'tiebreaking'])
def test_rows_and_ranks_match_the_sorted_frame(trained, mode, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    te = _messy_test(train, seed=11)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(gru, te.copy(), cut_off=[1, 5, 20], batch_size=7, mode=mode)
        rec, mrr = evaluation.evaluate_gpu(gru, te.copy(), cut_off=[1, 5, 20], batch_size=7, mode=mode)
    df, scored = _frame(gru, te)
    ev = res['events']
    assert list(ev.columns) == ['SessionId', 'Time', 'input_item', 'ItemId', 'rank'] and ev['rank'].dtype == np.float64
    assert len(ev) == scored.sum()
    np.testing.assert_array_equal(ev.SessionId.values, df.SessionId.values[scored])
    np.testing.assert_array_equal(ev.Time.values, df.Time.values[scored])
    np.testing.assert_array_equal(ev.ItemId.values, df.ItemId.values[scored])
    np.testing.assert_array_equal(ev.input_item.values, df.ItemId.values[np.flatnonzero(scored) - 1])
    assert 20000 not in set(ev.SessionId) and 999999 not in set(ev.ItemId)
    np.testing.assert_array_equal(ev['rank'].values, _expected_ranks(gru, df, mode, 7)[scored])
    assert res['recall'] == rec and res['mrr'] == mrr            # the double's sums, as evaluate_gpu returns them
    r = ev['rank'].values
    for j, c in enumerate([1, 5, 20]):
        want = np.mean([1.0 / np.log2(x + 1.0) if x <= c else 0.0 for x in r])
        assert abs(res['ndcg'][j] - want) <= 1e-12
        assert abs(res['recall'][j] - np.mean(r <= c)) <= 1e-12
    assert 'topk_items' not in res


def test_topk_lists_and_coverage(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    te = _messy_test(train, seed=5)
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(gru, te.copy(), cut_off=[20], batch_size=5, k=6)
    ti, ts = res['topk_items'], res['topk_scores']
    assert ti.shape == (len(res['events']), 6) and ts.dtype == np.float32
    assert set(ti.reshape(-1)) <= set(gru.itemidmap.index.values)          # original item ids
    assert np.all(np.diff(ts, axis=1) <= 0)
    assert res['coverage'] == len(np.unique(ti)) / gru.n_items
    # a target ranked first (standard rank 1) is the first item of its list unless an equal score precedes it
    first = res['events']['rank'].values == 1
    assert np.mean(ti[first, 0] == res['events'].ItemId.values[first]) > 0.9


def test_items_restrict_ranks_and_lists(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    te = _messy_test(train, seed=7)
    cand = list(gru.itemidmap.index.values[::3]) + [gru.itemidmap.index.values[0]]     # a duplicate
    with contextlib.redirect_stdout(io.StringIO()):
        res = evaluation.evaluate_events(gru, te.copy(), items=cand, cut_off=[3, 10], batch_size=6, mode='conservative', k=4)
        rec, mrr = evaluation.evaluate_gpu(gru, te.copy(), items=cand, cut_off=[3, 10], batch_size=6, mode='conservative')
    assert res['recall'] == rec and res['mrr'] == mrr
    assert set(res['topk_items'].reshape(-1)) <= set(cand)
    df, scored = _frame(gru, te)
    exp = _expected_ranks(gru, df, 'conservative', 6, items=gru.itemidmap[cand].values)[scored]
    np.testing.assert_array_equal(res['events']['rank'].values, exp)
    assert gru._engine.eval_items is None                                  # restored


def test_argument_errors(trained, monkeypatch):
    import evaluation
    gru, train = trained
    _install(monkeypatch, gru)
    te = _messy_test(train, seed=2)
    for k in (-1, gru.n_items + 1, 2.5, True):
        with pytest.raises(ValueError):
            evaluation.evaluate_events(gru, te.copy(), k=k)
    with pytest.raises(ValueError):                                        # k beyond the distinct candidates
        evaluation.evaluate_events(gru, te.copy(), items=list(gru.itemidmap.index.values[:3]) * 2, k=4)
    with pytest.raises(NotImplementedError):
        evaluation.evaluate_events(gru, te.copy(), mode='random')
    with pytest.raises(KeyError):
        evaluation.evaluate_events(gru, te.copy(), items=[123456789])
    monkeypatch.setattr(type(gru), '_world', staticmethod(lambda: (2, 0)))
    with pytest.raises(NotImplementedError):
        evaluation.evaluate_events(gru, te.copy())
