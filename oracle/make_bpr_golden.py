"""TEST INFRASTRUCTURE ONLY.  Runs the reference's unmodified BPR (baselines.py:303-418) on the data of make_baselines_golden.py
with a seeded np.random and records what it computed -> tests/golden/baselines/bpr_<case>_<params>.npz: the data, U and I after
the fit, each iteration's printed mean(log sigm), and predict_next over the whole catalogue for the first test events.
tests/test_host_bpr.py holds oracle/bpr_oracle.py to them.

Usage: python oracle/make_bpr_golden.py <directory of the reference checkout>"""
import contextlib
import importlib.util
import io
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_baselines_golden import OUT, N_PRED, cases  # noqa: E402

SEED = 7
N_ITER = 3
PARAMS = {'f16_uniform': dict(n_factors=16, n_iterations=N_ITER, learning_rate=0.05),
          'f100_normal': dict(n_factors=100, n_iterations=N_ITER, learning_rate=0.02, lambda_session=0.01, lambda_item=0.02, sigma=0.1,
                              init_normal=True)}


def main(ref_dir):
    spec = importlib.util.spec_from_file_location('ref_baselines', os.path.join(ref_dir, 'baselines.py'))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    os.makedirs(OUT, exist_ok=True)
    warnings.simplefilter('ignore', DeprecationWarning)
    for name, tr, te in cases():
        itemids = tr.ItemId.unique()
        te = te[te.ItemId.isin(itemids)].sort_values(['SessionId', 'Time'], kind='stable').head(N_PRED)
        for tag, params in PARAMS.items():
            np.random.seed(SEED)
            m = ref.BPR(**params)
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                m.fit(tr.copy())
            means = [float(line.split()[1]) for line in buf.getvalue().splitlines()]
            assert len(means) == N_ITER
            pred = np.stack([m.predict_next(s, i, itemids).values for s, i in zip(te.SessionId.values, te.ItemId.values)])
            out = dict(train_sid=tr.SessionId.values, train_iid=tr.ItemId.values, train_time=tr.Time.values, test_sid=te.SessionId.values,
                       test_iid=te.ItemId.values, itemids=itemids, seed=SEED, U=m.U, I=m.I, means=np.array(means), pred=pred)
            path = os.path.join(OUT, 'bpr_%s_%s.npz' % (name, tag))
            np.savez_compressed(path, **{k: (np.asarray(v).astype(str) if np.asarray(v).dtype == object else np.asarray(v)) for k, v in out.items()})
            print('wrote', path)


if __name__ == '__main__':
    main(sys.argv[1])
