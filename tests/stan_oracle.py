"""float64 NumPy restatement of STAN-style session kNN (baselines.STAN, DESIGN §3p) on top of oracle/sknn_oracle.py's index: each
training session's last position of every item and its recency weight, the three decay tables, the neighbours and scores after a
session prefix, and the per-event ranking of evaluate_gpu / evaluate_events with items=, exclude_seen, history and top-k lists
(the rank rules of baselines_oracle).  Test infrastructure: the device (g4r_sknn.cuh) and the host predict_next are compared
against it; never imported by the package."""
import numpy as np
import pandas as pd
import scipy.sparse as sp

import sknn_oracle as sko
from baselines_oracle import tie_noise

INF = float('inf')


class Index(sko.Index):
    """sknn_oracle.Index plus q[rank]: {item: 1-based position of its last occurrence} (events ordered by time, ties by row
    order), w2[rank] = exp(-(float64(T_max - T) / lambda_snh)) with the subtraction in the time column's dtype, w3[d] = exp(-(d /
    lambda_inh)) for d < the longest session's length, and W1[d] = exp(-(d / lambda_spw))"""

    def __init__(self, sess, items, times, n_items, lambda_spw=INF, lambda_snh=INF, lambda_inh=INF):
        sess, items, times = np.asarray(sess), np.asarray(items), np.asarray(times)
        sko.Index.__init__(self, sess, items, times, n_items)
        code = pd.Index(pd.unique(sess)).get_indexer(sess)
        S = len(self.rank)
        rows = [[] for _ in range(S)]
        for r, c in enumerate(code.tolist()):
            rows[c].append(r)
        tl = times.tolist()
        self.q = [None] * S
        for c, rr in enumerate(rows):
            d = {}
            for p, r in enumerate(sorted(rr, key=lambda r: (tl[r], r)), 1):
                d[int(items[r])] = p
            self.q[self.rank[c]] = d
        T = np.array([times[rr].max() for rr in rows])                    # the time column's dtype
        w2 = np.exp(-((times.max() - T).astype(np.float64) / lambda_snh))  # sessions in first-appearance order
        self.w2 = np.empty(S)
        self.w2[self.rank] = w2
        self.w3 = np.exp(-(np.arange(max(len(rr) for rr in rows)) / lambda_inh))
        self.lambda_spw, self.table = lambda_spw, None
        self._positions()

    def _positions(self):
        """qm: [rank x item] the positions of q as a sparse matrix (the neighbour search reads it by column)"""
        r = np.repeat(np.arange(len(self.q)), [len(d) for d in self.q])
        c = np.fromiter((j for d in self.q for j in d), np.int64, len(r))
        v = np.fromiter((p for d in self.q for p in d.values()), np.int64, len(r))
        self.qm = sp.csr_matrix((v, (r, c)), shape=(len(self.q), self.n_items))

    @classmethod
    def from_arrays(cls, offsets, items, positions, recency, w2, w3, w1, n_items):
        """the index the device is given: distinct items per session (CSR), their positions, ranks, W2 per session, W3 and W1"""
        off = np.asarray(offsets)
        ix = cls.__new__(cls)
        lens = np.diff(off)
        sko.Index.__init__(ix, np.repeat(np.arange(len(lens)), lens), np.asarray(items), -np.repeat(np.asarray(recency), lens), n_items)
        ix.q = [None] * len(lens)
        for s in range(len(lens)):
            ix.q[int(recency[s])] = dict(zip(np.asarray(items)[off[s]:off[s + 1]].tolist(), np.asarray(positions)[off[s]:off[s + 1]].tolist()))
        ix.w2 = np.empty(len(lens))
        ix.w2[np.asarray(recency)] = w2
        ix.w3, ix.table = np.asarray(w3), np.asarray(w1)
        ix._positions()
        return ix

    def w1(self, t):
        if self.table is not None:
            assert len(self.table) >= t
            return self.table[:t]
        return np.exp(-(np.arange(t) / self.lambda_spw))


def neighbours(index, prefix, k, sample_size):
    """(ranks of the neighbours, their sims, q_n(r(n)) of each), in neighbour order"""
    t = len(prefix)
    last = {}
    for p, x in enumerate(np.asarray(prefix).tolist(), 1):
        last[x] = p
    ci = sorted(last, key=last.get)                                       # I(c) by ascending last position
    P = index.post
    cand = np.unique(np.concatenate([P.indices[P.indptr[i]:P.indptr[i + 1]][:sample_size] for i in ci]))[:sample_size]
    w1 = index.w1(t)
    pos = index.qm[cand][:, ci].toarray()                                 # q_n(i) of every candidate and shared item, 0: not shared
    lens = np.diff(index.by_rank.indptr)[cand]
    v, qr = np.zeros(len(cand)), np.zeros(len(cand), np.int64)
    for m, i in enumerate(ci):
        hit = pos[:, m] > 0
        v = v + np.where(hit, w1[t - last[i]], 0.0)
        qr = np.where(hit, pos[:, m], qr)                                 # ends at the shared item with the largest p_i
    sims = (v / np.sqrt((len(ci) * lens).astype(np.float64))) * index.w2[cand]
    o = np.lexsort((cand, -sims))[:k]
    return cand[o], sims[o], qr[o]


def scores(index, prefix, k, sample_size):
    """float64 score of every item after the session's inputs so far `prefix` (the current input last)"""
    s = np.zeros(index.n_items)
    for r, v, qr in zip(*neighbours(index, prefix, k, sample_size)):
        for j, qj in index.q[r].items():
            s[j] = s[j] + v * index.w3[abs(qj - qr)]
    return s


def rank_events(index, k_nb, sample_size, items, offsets, n_history=None, mode='standard', cand=None, exclude_seen=False, k=0, only=None):
    """sknn_oracle.rank_events for STAN: per counted event (data order) counts int64 [n, 2] ((-1, -1) for an exclude_seen miss),
    and with k > 0 the lists (items [n, k], -1 past the eligible ones; scores [n, k] float64, NaN there): the positive scores by
    (score desc, index asc), then every zero-score item by index.  only: the counted event numbers to compute (rows in that
    order); None: every one"""
    n_items = index.n_items
    items = np.asarray(items, dtype=np.int64)
    w0 = np.ones(n_items, np.int64) if cand is None else np.bincount(np.asarray(cand, dtype=np.int64), minlength=n_items)
    want = None if only is None else {int(e) for e in only}
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
            sc = scores(index, prefix, k_nb, sample_size)
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
