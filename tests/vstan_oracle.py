"""float64 NumPy restatement of VSTAN-style session kNN (baselines.VSTAN, DESIGN §3r) on top of tests/stan_oracle.py's index: the
similarity switch, the F and W4 tables, the neighbours with their g(n), the scores after a session prefix, and the per-event ranking
of evaluate_gpu / evaluate_events with items=, exclude_seen, history and top-k lists (stan_oracle.rank_events's rank rules, with
these scores).  Test infrastructure: the device (g4r_sknn.cuh) and the host predict_next are compared against it; never imported
by the package."""
import numpy as np

import stan_oracle as sto
from baselines_oracle import tie_noise

INF = float('inf')


class Index(sto.Index):
    """stan_oracle.Index plus similarity ('cosine' or 'vector'), f[j] = 1 + lambda_idf * log(n_sessions / df_j) with df_j the
    number of training sessions that contain j (1.0 for an item in none: it is never scored) and W4[d] = exp(-(d / lambda_ipw))"""

    def __init__(self, sess, items, times, n_items, similarity='cosine', lambda_spw=INF, lambda_snh=INF, lambda_inh=INF, lambda_ipw=INF,
                 lambda_idf=0.0):
        sto.Index.__init__(self, sess, items, times, n_items, lambda_spw, lambda_snh, lambda_inh)
        df = np.diff(self.post.indptr)                                     # the posting list lengths
        self.similarity, self.lambda_ipw, self.table4 = similarity, lambda_ipw, None
        self.f = np.ones(n_items)
        self.f[df > 0] = 1.0 + lambda_idf * np.log(len(self.q) / df[df > 0])

    @classmethod
    def from_arrays(cls, offsets, items, positions, recency, w2, w3, w1, n_items, similarity, f, w4):
        """the index the device is given: stan_oracle.Index.from_arrays's plus the similarity, F and W4"""
        ix = sto.Index.from_arrays.__func__(cls, offsets, items, positions, recency, w2, w3, w1, n_items)
        ix.similarity, ix.f, ix.table4 = similarity, np.asarray(f), np.asarray(w4)
        return ix

    def w4(self, t):
        if self.table4 is not None:
            assert len(self.table4) >= t
            return self.table4[:t]
        return np.exp(-(np.arange(t) / self.lambda_ipw))


def neighbours(index, prefix, k, sample_size):
    """(ranks of the neighbours, their sim2, q_n(r(n)), t - p_r(n), g(n)), in neighbour order"""
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
    v, qr, dr = np.zeros(len(cand)), np.zeros(len(cand), np.int64), np.zeros(len(cand), np.int64)
    for m, i in enumerate(ci):
        hit = pos[:, m] > 0
        v = v + np.where(hit, w1[t - last[i]], 0.0)
        qr = np.where(hit, pos[:, m], qr)                                 # ends at the shared item with the largest p_i
        dr = np.where(hit, t - last[i], dr)
    sim1 = v if index.similarity == 'vector' else v / np.sqrt((len(ci) * lens).astype(np.float64))
    sim2 = sim1 * index.w2[cand]
    o = np.lexsort((cand, -sim2))[:k]
    g = sim2[o] * index.w4(t)[dr[o]]
    return cand[o], sim2[o], qr[o], dr[o], g


def scores(index, prefix, k, sample_size):
    """float64 score of every item after the session's inputs so far `prefix` (the current input last): acc(j) * F[j] for the
    items the neighbours hold, 0 for every other"""
    s = np.zeros(index.n_items)
    held = np.zeros(index.n_items, bool)
    r_, _, q_, _, g_ = neighbours(index, prefix, k, sample_size)
    for r, qr, g in zip(r_, q_, g_):
        for j, qj in index.q[r].items():
            s[j] = s[j] + g * index.w3[abs(qj - qr)]
            held[j] = True
    s[held] = s[held] * index.f[held]
    return s


def rank_events(index, k_nb, sample_size, items, offsets, n_history=None, mode='standard', cand=None, exclude_seen=False, k=0, only=None):
    """stan_oracle.rank_events with VSTAN's scores: per counted event (data order) counts int64 [n, 2] ((-1, -1) for an
    exclude_seen miss), and with k > 0 the lists (items [n, k], -1 past the eligible ones; scores [n, k] float64, NaN there): the
    positive scores by (score desc, index asc), then every zero-score item by index.  only: the counted event numbers to compute
    (rows in that order); None: every one"""
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
