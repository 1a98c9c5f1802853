"""CPU tests of GRU4Rec.recommend_next_batch on the engine double (tests/oracle_engine.py, extended here by a predict_topk made of
its own predict() and a stable sort): item-ID mapping, the session state it shares with predict_next_batch, and lane resets on
a new session id.  The device top-k itself is tested in test_gpu_topk.py."""
import contextlib
import io

import numpy as np
import pytest

from gru4rec_b200 import _lib
from gru4rec_b200.synth import make_sessions
import oracle_engine


class TopkOracleEngine(oracle_engine.OracleEngine):
    """the engine double plus Engine.predict_topk, built from the double's own predict() and a stable sort"""

    def predict_topk(self, X, k, reset_mask=None):
        k = _lib.check_topk(k, int(self.cfg.n_items))
        scores = self.predict(X, reset_mask)
        order = np.argsort(-scores, axis=1, kind='stable')[:, :k]
        return order.astype(np.int32), np.take_along_axis(scores, order, axis=1).astype(np.float32)


def _install(monkeypatch, gru):
    """route the engines `gru` builds to TopkOracleEngine (as oracle_engine.install does for the plain double)"""
    def make(cfg, device=0):
        return TopkOracleEngine(cfg, oracle_engine.model_kwargs_of(gru), device)
    monkeypatch.setattr(_lib, 'Engine', make)


def _twins(monkeypatch, tmp_path, mk):
    """two models with the same trained weights and fresh serving state, each on its own engine double"""
    import gru4rec
    df = make_sessions(n_items=60, n_events=800, seed=5, item_as_str=True)
    gru = gru4rec.GRU4Rec(**mk)
    _install(monkeypatch, gru)
    with contextlib.redirect_stdout(io.StringIO()):
        gru.fit(df.copy(), sample_store=mk['n_sample'] * 8)
    fn = str(tmp_path / 'model.pickle')
    gru.savemodel(fn)
    out = []
    for _ in range(2):
        g = gru4rec.GRU4Rec.loadmodel(fn)
        _install(monkeypatch, g)
        out.append(g)
    return out


def _expected(preds, k):
    """top k of predict_next_batch's frame (items x batch): original item IDs and scores, ties to the earlier item"""
    v = preds.values.T
    order = np.argsort(-v, axis=1, kind='stable')[:, :k]
    return preds.index.to_numpy()[order], np.take_along_axis(v, order, axis=1)


@pytest.mark.parametrize('mk', [
    dict(loss='bpr-max', final_act='elu-0.5', layers=[12], batch_size=8, n_epochs=1, n_sample=16),
    dict(loss='cross-entropy', final_act='softmax', layers=[10], batch_size=6, n_epochs=1, constrained_embedding=True, n_sample=12),
])
def test_recommend_next_batch_shares_state_with_predict_next_batch(mk, monkeypatch, tmp_path):
    a, b = _twins(monkeypatch, tmp_path, mk)           # a alternates recommend / predict, b only predicts
    ids = a.itemidmap.index.values
    rs = np.random.RandomState(0)
    sess = np.arange(5)
    for step in range(6):
        inp = ids[rs.randint(0, len(ids), 5)]
        if step == 3:
            sess = sess.copy(); sess[2] = 99            # a new session in lane 2: its state starts from zero
        ref = b.predict_next_batch(sess, inp, batch=5)
        if step % 2 == 0:
            items, scores = a.recommend_next_batch(sess, inp, k=7, batch=5)
            e_items, e_scores = _expected(ref, 7)
            assert items.shape == (5, 7) and scores.shape == (5, 7) and scores.dtype == np.float32
            assert set(items.reshape(-1)) <= set(ids) and isinstance(items[0, 0], str)     # original item IDs
            np.testing.assert_array_equal(items, e_items)
            np.testing.assert_array_equal(scores, e_scores)
        else:
            got = a.predict_next_batch(sess, inp, batch=5)
            np.testing.assert_array_equal(got.values, ref.values)
    # the lane reset is real: the same input after a fresh session differs from the carried state
    fresh = b.predict_next_batch(np.array([0, 1, 100, 3, 4]), inp, batch=5).values[:, 2]
    carried = a.predict_next_batch(sess, inp, batch=5).values[:, 2]
    assert not np.array_equal(fresh, carried)


def test_recommend_next_batch_argument_errors(monkeypatch, tmp_path):
    a, _ = _twins(monkeypatch, tmp_path, dict(loss='bpr-max', final_act='linear', layers=[8], batch_size=4, n_epochs=1, n_sample=8))
    ids = a.itemidmap.index.values[:3]
    for k in (0, -1, a.n_items + 1, 2.5):
        with pytest.raises(ValueError):
            a.recommend_next_batch(np.arange(3), ids, k=k, batch=3)
    items, _ = a.recommend_next_batch(np.arange(3), ids, k=a.n_items, batch=3)
    assert sorted(items[0]) == sorted(a.itemidmap.index.values)
    a.error_during_train = True
    with pytest.raises(Exception):
        a.recommend_next_batch(np.arange(3), ids, k=3, batch=3)
