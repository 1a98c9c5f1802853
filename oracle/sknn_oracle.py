"""float64 NumPy restatement of session-based kNN (baselines.SessionKNN, DESIGN §3o): the index of the training sessions (their
distinct items, the recency order), the scores after a session prefix for both similarities, and the per-event ranking of
evaluate_gpu / evaluate_events with items=, exclude_seen, history and top-k lists (the rank rules of baselines_oracle).  Test
infrastructure: the device (g4r_sknn.cuh) and the host predict_next are compared against it; never imported by the package."""
import numpy as np
import pandas as pd
import scipy.sparse as sp

from baselines_oracle import MODES, ranks, sums, tie_noise  # noqa: F401


class Index(object):
    """sess: the training events' session ids, items: their item indices, times: their time values.  Sessions are numbered by
    first appearance; rank 0 is the most recent (largest T, ties by first appearance)."""

    def __init__(self, sess, items, times, n_items):
        code = pd.Index(pd.unique(np.asarray(sess))).get_indexer(np.asarray(sess))
        S = int(code.max()) + 1
        T = [None] * S
        for c, x in zip(code.tolist(), np.asarray(times).tolist()):
            T[c] = x if T[c] is None or x > T[c] else T[c]
        self.order = sorted(range(S), key=lambda s: (-T[s], s))          # session of each rank
        self.rank = np.empty(S, np.int64)
        self.rank[self.order] = np.arange(S)
        m = sp.csr_matrix((np.ones(len(code)), (self.rank[code], np.asarray(items))), shape=(S, n_items))
        m.sum_duplicates()
        m.data[:] = 1
        m.sort_indices()
        self.by_rank = m                                                  # [rank x item]: I(s)
        self.post = m.T.tocsr()                                           # [item x rank]: its sessions, ranks ascending
        self.post.sort_indices()
        self.n_items = n_items

    def items_of(self, r):
        return self.by_rank.indices[self.by_rank.indptr[r]:self.by_rank.indptr[r + 1]]

    def csr(self):
        """(offsets, distinct items ascending) of the sessions in first-appearance order, and each session's rank"""
        m = self.by_rank[self.rank]
        return m.indptr.astype(np.int64), m.indices.astype(np.int32), self.rank.astype(np.int32)


def neighbours(index, prefix, k, sample_size, similarity):
    """(ranks of the neighbours, their similarities), in neighbour order"""
    t = len(prefix)
    last = {}
    for q, x in enumerate(np.asarray(prefix).tolist(), 1):
        last[x] = q
    ci = sorted(last, key=last.get)                                       # I(c) by ascending last position
    P = index.post
    cand = np.unique(np.concatenate([P.indices[P.indptr[i]:P.indptr[i + 1]][:sample_size] for i in ci]))[:sample_size]
    sub = index.by_rank[cand][:, ci].toarray() > 0
    lens = np.diff(index.by_rank.indptr)[cand]
    if similarity == 'cosine':
        sims = sub.sum(axis=1) / np.sqrt((len(ci) * lens).astype(np.float64))
    else:
        sims = np.zeros(len(cand))
        for m, i in enumerate(ci):
            sims = sims + np.where(sub[:, m], last[i] / t, 0.0)
    o = np.lexsort((cand, -sims))[:k]
    return cand[o], sims[o]


def scores(index, prefix, k, sample_size, similarity):
    """float64 score of every item after the session's inputs so far `prefix` (the current input last)"""
    s = np.zeros(index.n_items)
    for r, v in zip(*neighbours(index, prefix, k, sample_size, similarity)):
        j = index.items_of(r)
        s[j] = s[j] + v
    return s


def rank_events(index, k_nb, sample_size, similarity, items, offsets, n_history=None, mode='standard', cand=None, exclude_seen=False,
                k=0, only=None):
    """baselines_oracle.rank_events for SessionKNN: per counted event (data order) counts int64 [n, 2] ((-1, -1) for an
    exclude_seen miss), and with k > 0 the lists (items [n, k], -1 past the eligible ones; scores [n, k] float64, NaN there).
    only: the counted event numbers to compute (the rows come in that order); None: every one"""
    n_items = index.n_items
    items = np.asarray(items, dtype=np.int64)
    w0 = np.ones(n_items, np.int64) if cand is None else np.bincount(np.asarray(cand, dtype=np.int64), minlength=n_items)
    want = None if only is None else {int(e): q for q, e in enumerate(only)}
    rows = {}
    e = 0
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        for p in range(st + max(h, 1) - 1, en - 1):
            if want is not None and e not in want:
                e += 1
                continue
            y = items[p + 1]
            prefix = items[st:p + 1]
            sc = scores(index, prefix, k_nb, sample_size, similarity)
            w = w0.copy()
            if exclude_seen:
                w[prefix] = 0
            cmp = sc + tie_noise(e, np.arange(n_items)) if mode == 'tiebreaking' else sc
            t = cmp[y]
            if exclude_seen and y in set(prefix.tolist()):
                cnt = (-1, -1)
            else:
                cnt = (int(w[cmp > t].sum()), int(w[cmp == t].sum()))
            row_i, row_s = None, None
            if k:
                elig = np.flatnonzero(w > 0)
                o = elig[np.lexsort((elig, -sc[elig]))][:k]
                row_i = np.full(k, -1, np.int64); row_s = np.full(k, np.nan)
                row_i[:len(o)] = o; row_s[:len(o)] = sc[o]
            rows[e] = (cnt, row_i, row_s)
            e += 1
    keys = sorted(rows) if only is None else [int(x) for x in only]
    counts = np.array([rows[x][0] for x in keys], dtype=np.int64).reshape(-1, 2)
    if not k:
        return counts, None, None
    return counts, np.array([rows[x][1] for x in keys]).reshape(-1, k), np.array([rows[x][2] for x in keys]).reshape(-1, k)
