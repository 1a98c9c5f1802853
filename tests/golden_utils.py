"""Helpers to replay tests/golden/*.npz (made by oracle/make_golden.py from the reference's own code)."""
import glob
import os
import numpy as np
import pandas as pd

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def golden_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, '*.npz')))


def load_golden(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + '.npz'), allow_pickle=True))
    from collections import OrderedDict  # noqa: F401  (repr of kwargs may reference it)
    g['model_kwargs'] = eval(str(g['model_kwargs']))
    g['fit_kwargs'] = eval(str(g['fit_kwargs']))
    return g


def frames(g):
    tr = pd.DataFrame({'SessionId': g['train_SessionId'], 'ItemId': g['train_ItemId'], 'Time': g['train_Time']})
    te = pd.DataFrame({'SessionId': g['test_SessionId'], 'ItemId': g['test_ItemId'], 'Time': g['test_Time']})
    return tr, te


def init_weights(g, prefix='init_'):
    nl = len(g['model_kwargs']['layers'])
    w = dict(Wx=[g['%sWx%d' % (prefix, i)] for i in range(nl)], Wh=[g['%sWh%d' % (prefix, i)] for i in range(nl)],
             Wrz=[g['%sWrz%d' % (prefix, i)] for i in range(nl)], Bh=[g['%sBh%d' % (prefix, i)] for i in range(nl)],
             Wy=g[prefix + 'Wy'], By=g[prefix + 'By'])
    if (prefix + 'E') in g:
        w['E'] = g[prefix + 'E']
    return w


def dropout_sites(mk):
    """creation order of the reference's dropout sites: embed first (gru4rec.py:443/451), then hidden layers."""
    sites = []
    if mk.get('dropout_p_embed', 0) > 0 and (mk.get('constrained_embedding') or mk.get('embedding')):
        sites.append('e')
    if mk.get('dropout_p_hidden', 0) > 0:
        for i in range(len(mk['layers'])):
            sites.append(('h', i))
    return sites


def step_masks(g, s, M):
    mk = g['model_kwargs']
    out = {}
    for j, site in enumerate(dropout_sites(mk)):
        p = mk['dropout_p_embed'] if site == 'e' else mk['dropout_p_hidden']
        b = g['dropmask_site%d' % j][s, :M]
        out[site] = (b / np.float32(1.0 - p)).astype(np.float32)
    return out


def step_samples(g, s):
    """negative samples the reference used at train step s (row STI of the current store)."""
    if 'sample_stores' not in g:
        return None
    fs = g['store_first_step']
    k = int(np.searchsorted(fs, s, side='right') - 1)
    return g['sample_stores'][k][s - fs[k]]


def fit_data(orc, g, tr):
    """prepare_fit_data with the model's time_sort option (gru4rec.py:585)."""
    return orc.prepare_fit_data(tr, time_sort=g['model_kwargs'].get('time_sort', True))


def epoch_order(g, d, e):
    """session order of epoch e: recorded np.random.permutation for train_random_order (gru4rec.py:593), else base_order"""
    return g['epoch_orders'][e] if 'epoch_orders' in g else d['base_order']


def datatools_cases():
    """(frame, key columns, any_order) of the sort_if_needed / compute_offset comparison (tests/golden/datatools/cases.npz): random
    frames of 1..300 events, unsorted, sorted by (session, time), by (session, time, item), and grouped by session in random order."""
    rs = np.random.RandomState(0)
    for n in (1, 2, 50, 300):
        for trial in range(8):
            df = pd.DataFrame({'SessionId': rs.randint(0, max(2, n // 4), n), 'Time': rs.randint(0, 40, n), 'ItemId': rs.randint(0, 9, n)})
            if trial % 4 == 1: df = df.sort_values(['SessionId', 'Time']).reset_index(drop=True)
            if trial % 4 == 2: df = df.sort_values(['SessionId', 'Time', 'ItemId']).reset_index(drop=True)
            if trial % 4 == 3:      # sessions grouped but in arbitrary order
                df = df.sort_values(['SessionId', 'Time']).reset_index(drop=True)
                df = pd.concat([df[df.SessionId == s] for s in rs.permutation(df['SessionId'].unique())]).reset_index(drop=True)
            for cols in (['SessionId', 'Time'], ['SessionId', 'Time', 'ItemId'], ['SessionId']):
                for any_order in (False, True):
                    yield df, cols, any_order


def datatools_outcome(mod, df, cols, any_order):
    """what sort_if_needed of module `mod` printed (minus the timing line), the frame it left (index and columns) and the offsets"""
    import contextlib
    import io
    a, out = df.copy(), io.StringIO()
    with contextlib.redirect_stdout(out):
        mod.sort_if_needed(a, cols, any_order)
    lines = [l for l in out.getvalue().splitlines() if not l.startswith('Data is sorted in')]
    frame = np.stack([a.index.values] + [a[c].values for c in ('SessionId', 'Time', 'ItemId')], axis=1)
    return lines, frame, mod.compute_offset(a, 'SessionId')
