"""TEST INFRASTRUCTURE ONLY.  Runs the reference's unmodified baselines.py (plain pandas / NumPy) on small synthetic data and
records what it computed -> tests/golden/baselines/<case>.npz: the data, every item's kept ItemKNN (ids, sims) with positive sim,
the Pop lists, and predict_next over the whole catalogue for the first test events (SessionPop replayed in order).
tests/test_host_baselines.py holds oracle/baselines_oracle.py to them.

Usage: python oracle/make_baselines_golden.py <directory of the reference checkout>"""
import importlib.util
import os
import sys
import warnings

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from gru4rec_b200.synth import make_sessions, train_test_split  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'baselines')
KNN = {'knn_100_20_05': (100, 20, 0.5), 'knn_5_0_1': (5, 0, 1.0), 'knn_20_20_0': (20, 20, 0.0)}
POP = {'top100': (100, None), 'top3': (3, None), 'top100_bysession': (100, 'SessionId')}
N_PRED = 60


def cases():
    tr, te = train_test_split(make_sessions(n_items=150, n_events=2500, seed=1), 0.2)
    yield 'int_ids', tr, te
    df = make_sessions(n_items=80, n_events=1200, seed=2, item_as_str=True)
    rs = np.random.RandomState(3)
    rep = rs.rand(len(df)) < 0.25                                   # repeated items inside sessions
    src = np.flatnonzero(rep)
    src = src[(src > 0) & (df.SessionId.values[src] == df.SessionId.values[src - 1])]
    df.loc[src, 'ItemId'] = df.ItemId.values[src - 1]
    tied = df.SessionId.isin(df.SessionId.unique()[::7])             # tied times
    df.loc[tied, 'Time'] = df.loc[tied].groupby('SessionId').Time.transform('min')
    single = pd.DataFrame({'SessionId': [90000, 90001], 'ItemId': df.ItemId.values[:2], 'Time': [1e9, 1e9 + 1]})
    df = pd.concat([df, single], ignore_index=True)                 # single-event sessions
    tr, te = train_test_split(df[df.SessionId < 90000], 0.2)
    yield 'str_messy', pd.concat([tr, single]).reset_index(drop=True), te


def main(ref_dir):
    spec = importlib.util.spec_from_file_location('ref_baselines', os.path.join(ref_dir, 'baselines.py'))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    os.makedirs(OUT, exist_ok=True)
    warnings.simplefilter('ignore', DeprecationWarning)            # np.in1d in the reference
    for name, tr, te in cases():
        itemids = tr.ItemId.unique()
        te = te[te.ItemId.isin(itemids)].sort_values(['SessionId', 'Time'], kind='stable').head(N_PRED)
        out = dict(train_sid=tr.SessionId.values, train_iid=tr.ItemId.values, train_time=tr.Time.values,
                   test_sid=te.SessionId.values, test_iid=te.ItemId.values, itemids=itemids)
        for tag, (n_sims, lmbd, alpha) in KNN.items():
            m = ref.ItemKNN(n_sims=n_sims, lmbd=lmbd, alpha=alpha)
            m.fit(tr.copy())
            pos = pd.Index(itemids)
            idx = np.full((len(itemids), n_sims), -1, np.int32); sim = np.zeros((len(itemids), n_sims))
            for i, iid in enumerate(itemids):
                ser = m.sims[iid]
                ser = ser[ser.values > 0]
                idx[i, :len(ser)] = pos.get_indexer(ser.index); sim[i, :len(ser)] = ser.values
            out[tag + '_idx'], out[tag + '_sim'] = idx, sim
            out[tag + '_pred'] = np.stack([m.predict_next(s, i, itemids).values for s, i in zip(te.SessionId.values, te.ItemId.values)])
        for tag, (top_n, by) in POP.items():
            for cls in ('Pop', 'SessionPop'):
                m = getattr(ref, cls)(top_n=top_n, support_by_key=by)
                m.fit(tr.copy())
                key = '%s_%s' % (cls.lower(), tag)
                if cls == 'Pop':
                    out[key + '_ids'] = m.pop_list.index.values; out[key + '_score'] = m.pop_list.values
                out[key + '_pred'] = np.stack([m.predict_next(s, i, itemids).values for s, i in zip(te.SessionId.values, te.ItemId.values)])
        path = os.path.join(OUT, name + '.npz')
        np.savez_compressed(path, **{k: (np.asarray(v).astype(str) if np.asarray(v).dtype == object else np.asarray(v)) for k, v in out.items()})
        print('wrote', path)


if __name__ == '__main__':
    main(sys.argv[1])
