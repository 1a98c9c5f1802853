"""float64 NumPy restatement of the session baselines (the reference's baselines.py:52-301) and of their evaluation
(DESIGN §3j): the ItemKNN rows, the Pop scores, predict_next, and the per-event ranking in every mode with items=, exclude_seen,
history and top-k lists.  Test infrastructure: the device (g4r_baselines.cuh) is compared against it, and it is compared
against the reference's recorded runs (tests/golden/baselines)."""
import numpy as np
import scipy.sparse as sp

M32 = 0xFFFFFFFF
TIE_SEED = 0x6A09E667
MODES = {'standard': 0, 'conservative': 1, 'median': 2, 'tiebreaking': 3}


def norm_factors(supp, lmbd, alpha):
    """a[i] = (supp_i + lmbd)^alpha with numpy's scalar power (one row at a time, as the reference), b = the array power"""
    supp = np.asarray(supp, dtype=np.int64)
    a = np.array([np.power((s + lmbd), alpha) for s in supp], dtype=np.float64)
    return a, np.power((supp + lmbd), (1.0 - alpha)).astype(np.float64)


def cooccurrence(offsets, items, n_items, rows=None):
    """cnt [len(rows) x n_items] (scipy CSR, int64): cnt(i, j) = sum over sessions of (occurrences of i) * [j in session],
    the diagonal zero"""
    offsets = np.asarray(offsets, dtype=np.int64)
    sess = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    occ = sp.csr_matrix((np.ones(len(items), np.int64), (sess, np.asarray(items))), shape=(len(offsets) - 1, n_items))
    occ.sum_duplicates()
    pres = occ.copy()
    pres.data[:] = 1
    left = occ.T.tocsr() if rows is None else occ.T.tocsr()[np.asarray(rows)]
    cnt = (left @ pres).tocoo()
    rr = np.arange(n_items) if rows is None else np.asarray(rows)
    off_diag = cnt.col != rr[cnt.row]
    return sp.csr_matrix((cnt.data[off_diag], (cnt.row[off_diag], cnt.col[off_diag])), shape=cnt.shape)


def knn_rows(offsets, items, n_items, n_sims, lmbd, alpha, rows=None):
    """{item index: (kept indices, kept sims)} in (sim desc, index asc) order, positive sims only"""
    supp = np.bincount(np.asarray(items), minlength=n_items)
    return knn_rows_from_factors(offsets, items, n_items, n_sims, *norm_factors(supp, lmbd, alpha), rows=rows)


def knn_rows_from_factors(offsets, items, n_items, n_sims, a, b, rows=None):
    """knn_rows with the norm factors given"""
    cnt = cooccurrence(offsets, items, n_items, rows)
    out = {}
    for q, i in enumerate(np.arange(n_items) if rows is None else rows):
        lo, hi = cnt.indptr[q], cnt.indptr[q + 1]
        j = cnt.indices[lo:hi].astype(np.int64)
        norm = a[i] * b[j]
        norm[norm == 0] = 1
        s = cnt.data[lo:hi].astype(np.float64) / norm
        o = np.lexsort((j, -s))[:n_sims]
        out[int(i)] = (j[o], s[o])
    return out


def pop_scores(supp, top_n):
    """dense Pop scores: supp / (supp + 1) for the top_n items by (score desc, index asc), 0 elsewhere"""
    supp = np.asarray(supp, dtype=np.int64)
    score = supp / (supp + 1)
    keep = np.lexsort((np.arange(len(supp)), -score))[:top_n]
    dense = np.zeros(len(supp))
    dense[keep] = score[keep]
    return dense


def scores(kind, model, x, prefix):
    """float64 score of every item after input item x with the session's inputs so far `prefix` (x included):
    kind 'itemknn' (model: knn_rows' dict), 'pop' / 'sessionpop' (model: dense Pop scores)"""
    if kind == 'itemknn':
        n_items, rows = model
        s = np.zeros(n_items)
        j, v = rows[int(x)]
        s[j] = v
        return s
    s = np.array(model, dtype=np.float64)
    if kind == 'sessionpop':
        u, c = np.unique(np.asarray(prefix), return_counts=True)
        s[u] = s[u] + c.astype(np.float64)
    return s


def mix32(x):
    x = np.asarray(x, dtype=np.uint64) & M32
    x ^= x >> np.uint64(16); x = (x * np.uint64(0x7feb352d)) & M32
    x ^= x >> np.uint64(15); x = (x * np.uint64(0x846ca68b)) & M32
    x ^= x >> np.uint64(16)
    return x


def tie_noise(e, items):
    """U(0,1) * 1e-10 of `items` in counted event e: a counter hash of (e, item)"""
    k = mix32(TIE_SEED ^ ((0x9E3779B9 * ((e + 1) & M32)) & M32))
    k = mix32((k + ((e >> 32) * 0x85EBCA6B)) & M32)
    r = mix32((k + np.asarray(items, dtype=np.uint64)) & M32)
    return (r >> np.uint64(8)).astype(np.float64) * (1.0 / 16777216.0) * 1e-10


def rank_events(kind, model, n_items, items, offsets, n_history=None, mode='standard', cand=None, exclude_seen=False, k=0):
    """per counted event (data order): counts int64 [n, 2] (#greater, #equal incl. the target; (-1, -1) for an exclude_seen
    miss), and with k > 0 the lists (items [n, k] (-1 past the eligible ones), scores [n, k] float64 (NaN there))"""
    items = np.asarray(items, dtype=np.int64)
    w0 = np.ones(n_items, np.int64) if cand is None else np.bincount(np.asarray(cand, dtype=np.int64), minlength=n_items)
    counts, li, ls = [], [], []
    e = 0
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for p in range(st + max(h, 1) - 1, en - 1):
            x, y = items[p], items[p + 1]
            prefix = items[st:p + 1]
            sc = scores(kind, model, x, prefix)
            w = w0.copy()
            if exclude_seen:
                w[prefix] = 0
            cmp = sc + tie_noise(e, np.arange(n_items)) if mode == 'tiebreaking' else sc
            t = cmp[y]
            if exclude_seen and y in set(prefix.tolist()):
                counts.append((-1, -1))
            else:
                counts.append((int(w[cmp > t].sum()), int(w[cmp == t].sum())))
            if k:
                elig = np.flatnonzero(w > 0)
                o = elig[np.lexsort((elig, -sc[elig]))][:k]
                row_i = np.full(k, -1, np.int64); row_s = np.full(k, np.nan)
                row_i[:len(o)] = o; row_s[:len(o)] = sc[o]
                li.append(row_i); ls.append(row_s)
            e += 1
    counts = np.array(counts, dtype=np.int64).reshape(-1, 2)
    if not k:
        return counts, None, None
    return counts, np.array(li).reshape(-1, k), np.array(ls).reshape(-1, k)


def ranks(counts, mode):
    gt, eq = counts[:, 0].astype(np.float64), counts[:, 1].astype(np.float64)
    r = gt + eq if mode == 'conservative' else (gt + 0.5 * (eq - 1.0) + 1.0 if mode == 'median' else gt + 1.0)
    r[counts[:, 0] < 0] = np.inf
    return r


def sums(counts, mode, cuts):
    """(hit sums, reciprocal-rank sums) per cut-off: a hit when rank <= N"""
    r = ranks(counts, mode)
    with np.errstate(divide='ignore'):
        return [float((r <= c).sum()) for c in cuts], [float(np.where(r <= c, 1.0 / r, 0.0).sum()) for c in cuts]
