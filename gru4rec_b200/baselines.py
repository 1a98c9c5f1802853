"""Session baselines of the reference (baselines.py:52-418): Pop, SessionPop, ItemKNN and BPR (BPR-MF), with its constructor
signatures, fit(data) and predict_next(session_id, input_item_id, predict_for_item_ids), session-based kNN (SessionKNN, DESIGN
§3o; STAN, §3p; VSTAN, §3r), the rule-based baselines (SR and AR, §3q, fitted on the device) and the neural NARM (§3s), SASRec
(§3t), SR-GNN (§3u), STAMP (§3v), NextItNet (§3w) and BERT4Rec (§3x), trained on the device, with the same surface.  ItemKNN's fit runs on the
device (the co-occurrence counts, the normalisation and the top n_sims per row, DESIGN §3j), and so does BPR's SGD, equal to the reference's
sequential run for the same np.random state (DESIGN §3k); evaluate_gpu / evaluate_events rank every test event of a baseline on the
device under the same protocol as a GRU4Rec model.  predict_next is computed on the host from the fitted model.  RandomPred is not
provided: it has nothing to fit, and its scores are unseeded noise."""
import math

import numpy as np
import pandas as pd

from . import _lib
from .gru4rec import GRU4Rec as _GRU4Rec


class Baseline(object):
    """What the baselines share: the item index (ids in unique() order, as GRU4Rec builds it), the device handle (created on
    first use, never pickled) and the evaluation hooks of evaluation.py."""
    error_during_train = False
    _kind = None
    _world = staticmethod(_GRU4Rec._world)
    _caches = ('_dev', '_post', '_p64')          # built on first use from the fitted model; never pickled, dropped by fit

    def _drop_caches(self):
        for name in self._caches:
            self.__dict__.pop(name, None)

    def _index(self, data):
        """itemidmap / n_items from the training data; returns the item index of every row"""
        ids = data[self.item_key].values
        itemids = pd.unique(ids)
        self.n_items = len(itemids)
        self.itemidmap = pd.Series(data=np.arange(self.n_items), index=itemids)
        return pd.Index(itemids).get_indexer(ids)

    def _sessions(self, data, order=None):
        """the session index of the training data, after the item index (_index): (item index of every row, session code of
        every row with the sessions in order of first appearance, session CSR offsets [n_sessions + 1], event order).  The event
        order groups the rows by session, each session's events in row order (order='rows') or by time_key with ties by row
        order (order='time'); it is None for order=None"""
        idx = self._index(data)
        sess = data[self.session_key].values
        code = pd.Index(pd.unique(sess)).get_indexer(sess)
        S = int(code.max()) + 1 if len(code) else 0
        offsets = np.zeros(S + 1, np.int64)
        offsets[1:] = np.cumsum(np.bincount(code, minlength=S))
        if order is None:
            return idx, code, offsets, None
        o = np.argsort(code, kind='stable') if order == 'rows' else np.lexsort((data[self.time_key].values, code))
        return idx, code, offsets, o

    def _prefix(self, session_id, x):
        """the session's inputs so far with x appended, or [x] when session_id is not the current session"""
        if self.current_session is None or self.current_session != session_id:
            self.current_session = session_id
            self.session = [x]
        else:
            self.session.append(x)
        return self.session

    def _integer(self, name, lo, hi):
        v = getattr(self, name)
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
            raise ValueError('%s must be an integer in %d .. %d, not %r' % (name, lo, hi, v))

    def _n_keep(self):
        raise NotImplementedError

    def _upload(self, dev):
        raise NotImplementedError

    def _cover(self, max_len):
        """prepares the device model for test sessions of up to max_len events (history included); only STAN needs to"""

    def _device(self):
        dev = self.__dict__.get('_dev')
        if dev is None:
            dev = _lib.Baselines(self._kind, self.n_items, self._n_keep())
            self._upload(dev)
            self._dev = dev
        return dev

    def __getstate__(self):
        state = self.__dict__.copy()
        for name in self._caches:
            state.pop(name, None)
        return state


def _pop_scores(model, data):
    """(dense scores [n_items] float64, 0 past top_n) of Pop / SessionPop: supp / (supp + 1) of the top_n items by (score desc,
    index asc); supp counts the events of an item, or with support_by_key the distinct values of that column"""
    model._index(data)
    grp = data.groupby(model.item_key)
    supp = grp.size() if model.support_by_key is None else grp[model.support_by_key].nunique()
    supp = supp.reindex(model.itemidmap.index).values.astype(np.int64)
    score = supp / (supp + 1)
    keep = np.lexsort((np.arange(model.n_items), -score))[:model.top_n]
    dense = np.zeros(model.n_items)
    dense[keep] = score[keep]
    model.pop_list = pd.Series(data=score[keep], index=model.itemidmap.index.values[keep])
    return dense


class Pop(Baseline):
    '''
    Pop(top_n=100, item_key='ItemId', support_by_key=None)

    Popularity predictor (baselines.py:52-118): the score of an item is supp / (supp + 1) for the top_n items by support and 0
    for the rest.  supp counts the events of the item, or with support_by_key the distinct values of that column.
    '''
    _kind = 'pop'

    def __init__(self, top_n=100, item_key='ItemId', support_by_key=None):
        self.top_n = top_n
        self.item_key = item_key
        self.support_by_key = support_by_key

    def fit(self, data):
        self.pop_scores = _pop_scores(self, data)
        self._drop_caches()

    def _n_keep(self):
        return self.top_n

    def _upload(self, dev):
        dev.set_pop(self.pop_scores)

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        preds = np.zeros(len(predict_for_item_ids))
        mask = np.isin(predict_for_item_ids, self.pop_list.index)
        preds[mask] = self.pop_list[predict_for_item_ids[mask]]
        return pd.Series(data=preds, index=predict_for_item_ids)


class SessionPop(Pop):
    '''
    SessionPop(top_n=100, item_key='ItemId', support_by_key=None)

    Session popularity predictor (baselines.py:120-197): the Pop score plus the number of times the item occurs among the
    session's inputs so far, the current input included.
    '''
    _kind = 'sessionpop'

    def fit(self, data):
        Pop.fit(self, data)
        self.prev_session_id = -1

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        if self.prev_session_id != session_id:
            self.prev_session_id = session_id
            self.pers = dict()
        self.pers[input_item_id] = self.pers.get(input_item_id, 0) + 1
        preds = np.array(Pop.predict_next(self, session_id, input_item_id, predict_for_item_ids).values)
        ser = pd.Series(self.pers)
        mask = np.isin(predict_for_item_ids, ser.index)
        preds[mask] += ser[predict_for_item_ids[mask]].values
        return pd.Series(data=preds, index=predict_for_item_ids)


class ItemKNN(Baseline):
    '''
    ItemKNN(n_sims=100, lmbd=20, alpha=0.5, session_key='SessionId', item_key='ItemId', time_key='Time')

    Item-to-item predictor (baselines.py:199-301).  For every occurrence of item i in a session, each distinct item j of the
    session gains 1: cnt(i, j) = sum over sessions of (occurrences of i) * [j in session], cnt(i, i) = 0.  The similarity is
    cnt / ((supp_i + lmbd)^alpha * (supp_j + lmbd)^(1 - alpha)) in float64 (supp: events of the item); each item keeps its n_sims
    largest positive similarities (ties by the smaller item index), every other item scores 0.
    '''
    _kind = 'itemknn'

    def __init__(self, n_sims=100, lmbd=20, alpha=0.5, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.n_sims = n_sims
        self.lmbd = lmbd
        self.alpha = alpha
        self.item_key = item_key
        self.session_key = session_key
        self.time_key = time_key

    def _n_keep(self):
        return self.n_sims

    def norm_factors(self, supp):
        """(a, b): a[i] = (supp_i + lmbd)^alpha, b[j] = (supp_j + lmbd)^(1 - alpha), computed as the reference computes them
        (baselines.py:272: a per row with numpy's scalar power, b over the support array), so that the device's sims are
        bitwise the reference's"""
        a = np.array([np.power((s + self.lmbd), self.alpha) for s in supp], dtype=np.float64)
        b = np.power((supp + self.lmbd), (1.0 - self.alpha)).astype(np.float64)
        return a, b

    def fit(self, data):
        idx, _, offsets, order = self._sessions(data, 'rows')
        supp = np.bincount(idx, minlength=self.n_items).astype(np.int64)
        a, b = self.norm_factors(supp)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.n_sims)
        self.fit_stats = dev.knn_fit(offsets, idx[order], a, b)
        self.rows = dev.rows_export()
        self._dev = dev

    def _upload(self, dev):
        dev.rows_import(*self.rows)

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        i = self.itemidmap[input_item_id]
        idx, sim, ln = self.rows
        kept = pd.Series(data=sim[i, :ln[i]], index=self.itemidmap.index.values[idx[i, :ln[i]]])
        preds = np.zeros(len(predict_for_item_ids))
        mask = np.isin(predict_for_item_ids, kept.index)
        preds[mask] = kept[predict_for_item_ids[mask]].values
        return pd.Series(data=preds, index=predict_for_item_ids)


class BPR(Baseline):
    '''
    BPR(n_factors=100, n_iterations=10, learning_rate=0.01, lambda_session=0.0, lambda_item=0.0, sigma=0.05, init_normal=False,
        session_key='SessionId', item_key='ItemId')

    Bayesian Personalized Ranking matrix factorisation (baselines.py:303-418) with sessions as users.  fit draws from the global
    np.random state exactly as the reference does (U, then I, then per iteration a permutation of the training rows and one
    randint(n_items) per event, which indexes a training *row* whose item is the negative) and runs each iteration's SGD on the
    device in the reference's order, bit for bit a sequential run (DESIGN §3k).  It prints `it, mean(log sigm)` per iteration.
    predict_next scores I[j] . mean(I[session inputs so far]) + bI[j].  After fit, `fit_stats` holds per iteration (mean log
    sigm, largest level = the longest chain of dependent updates, device ms).
    '''
    _kind = 'bpr'

    def __init__(self, n_factors=100, n_iterations=10, learning_rate=0.01, lambda_session=0.0, lambda_item=0.0, sigma=0.05, init_normal=False,
                 session_key='SessionId', item_key='ItemId'):
        self.n_factors = n_factors
        self.n_iterations = n_iterations
        self.learning_rate = learning_rate
        self.lambda_session = lambda_session
        self.lambda_item = lambda_item
        self.sigma = sigma
        self.init_normal = init_normal
        self.session_key = session_key
        self.item_key = item_key
        self.current_session = None

    def _n_keep(self):
        return self.n_factors

    def init(self, data):
        """the reference's init (baselines.py:343-347): U, then I, from the global np.random state"""
        if not self.init_normal:
            self.U = np.random.rand(self.n_sessions, self.n_factors) * 2 * self.sigma - self.sigma
            self.I = np.random.rand(self.n_items, self.n_factors) * 2 * self.sigma - self.sigma
        else:
            self.U = np.random.randn(self.n_sessions, self.n_factors) * self.sigma
            self.I = np.random.randn(self.n_items, self.n_factors) * self.sigma
        self.bU = np.zeros(self.n_sessions)
        self.bI = np.zeros(self.n_items)

    def fit(self, data):
        itemids = data[self.item_key].unique()
        self.n_items = len(itemids)
        self.itemidmap = pd.Series(data=np.arange(self.n_items), index=itemids)
        sessionids = data[self.session_key].unique()
        self.n_sessions = len(sessionids)
        # the reference's two merges: the random draws index rows of the merged frame, so its row order is kept
        data = pd.merge(data, pd.DataFrame({self.item_key: itemids, 'ItemIdx': np.arange(self.n_items)}), on=self.item_key, how='inner')
        data = pd.merge(data, pd.DataFrame({self.session_key: sessionids, 'SessionIdx': np.arange(self.n_sessions)}), on=self.session_key, how='inner')
        self.init(data)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.n_factors)
        dev.bpr_begin(data.SessionIdx.values, data.ItemIdx.values, self.n_sessions, self.U, self.I, self.bI)
        self.fit_stats = []
        N = len(data)
        for it in range(self.n_iterations):
            perm = np.random.permutation(N)
            negrow = np.random.randint(self.n_items, size=N)   # consumes the stream as N scalar randint(n_items) calls do
            stats = dev.bpr_iterate(perm, negrow, self.learning_rate, self.lambda_session, self.lambda_item)
            self.fit_stats.append(stats)
            print(it, np.float64(stats[0]))
        self.U, self.I = dev.bpr_export()
        dev.bpr_import(self.I, self.bI)                        # ends the fit: U and the per-row buffers leave the device
        self._dev = dev

    def _upload(self, dev):
        dev.bpr_import(self.I, self.bI)

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        uF = self.I[self._prefix(session_id, self.itemidmap[input_item_id])].mean(axis=0)
        iIdxs = self.itemidmap[predict_for_item_ids]
        return pd.Series(data=self.I[iIdxs].dot(uF) + self.bI[iIdxs], index=predict_for_item_ids)


class SessionKNN(Baseline):
    '''
    SessionKNN(k=100, sample_size=500, similarity='cosine', session_key='SessionId', item_key='ItemId', time_key='Time')

    Session-based kNN: S-KNN (similarity='cosine', Jannach & Ludewig, RecSys 2017) and a position-weighted variant in the style
    of V-SKNN (similarity='vector', Ludewig & Jannach, UMUAI 2018).  These are this project's definitions of the two methods
    (DESIGN §3o); they are not claimed to match any other implementation bit for bit.

    A training session s has its distinct items I(s) and time T(s), the largest time_key of its events; the recency order sorts
    the sessions by T descending, then by first appearance in the training data.  For the session's inputs so far c = (x_1 ..
    x_t), the current input included, the candidates are the first sample_size sessions in recency order that share an item
    with c.  Their similarity is |I(c) & I(s)| / sqrt(|I(c)| |I(s)|) ('cosine'), or ('vector') the sum, in order of position,
    of w(i) = p / t over the shared items, p the position of i's last occurrence in c.  The k most similar candidates (ties: the
    more recent) are the neighbours; item j scores the sum of the similarities of the neighbours that contain j, in float64 in
    neighbour order, and every other item scores 0.  Items of the current session are scored like any others.  evaluate_gpu /
    evaluate_events rank every event on the device; predict_next computes the same scores on the host.
    '''
    _kind = 'sknn'

    def __init__(self, k=100, sample_size=500, similarity='cosine', session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.k = k
        self.sample_size = sample_size
        self.similarity = similarity
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def _n_keep(self):
        return self.k

    def _check_similarity(self):
        if self.similarity not in _lib.SKNN_SIMILARITY:
            raise ValueError('similarity must be one of %s, not %r' % (sorted(_lib.SKNN_SIMILARITY), self.similarity))

    def _check_neighbours(self):
        if not 1 <= self.sample_size <= 8192:
            raise ValueError('sample_size must be in 1 .. 8192, not %r' % (self.sample_size,))
        if not 1 <= self.k <= min(self.sample_size, 1024):
            raise ValueError('k must be in 1 .. min(sample_size, 1024), not %r' % (self.k,))

    def _recency(self, code, times):
        """T per session (the largest time of its events); sets n_sessions and the recency ranks (T descending, ties by first
        appearance)"""
        T = pd.Series(times).groupby(code).max().values
        self.n_sessions = S = len(T)
        self.recency = np.empty(S, np.int32)
        self.recency[np.argsort(-T, kind='stable')] = np.arange(S, dtype=np.int32)
        return T

    def fit(self, data):
        self._check_similarity()
        self._check_neighbours()
        idx, code, _, _ = self._sessions(data)
        self._recency(code, data[self.time_key].values)
        pairs = np.unique(code.astype(np.int64) * self.n_items + idx.astype(np.int64))   # (session, item) distinct, items ascending per session
        self.session_items = (pairs % self.n_items).astype(np.int32)
        self.session_offsets = np.zeros(self.n_sessions + 1, np.int64)
        self.session_offsets[1:] = np.cumsum(np.bincount(pairs // self.n_items, minlength=self.n_sessions))
        self.current_session = None
        self._drop_caches()
        self._device()

    def _upload(self, dev):
        dev.sknn_fit(self.session_offsets, self.session_items, self.recency, self.sample_size, self.similarity)

    def _postings(self):
        """(per item offsets, the ranks of its sessions ascending, the session of each rank), built on first use"""
        post = self.__dict__.get('_post')
        if post is None:
            rank = np.repeat(self.recency, np.diff(self.session_offsets))
            o = np.lexsort((rank, self.session_items))
            ioff = np.zeros(self.n_items + 1, np.int64)
            ioff[1:] = np.cumsum(np.bincount(self.session_items, minlength=self.n_items))
            post = self._post = (ioff, rank[o], np.argsort(self.recency))
        return post

    def _knn_scores(self, prefix, weight, normalise, w2=None, w3=None, w4=None, f=None):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last), from the
        candidates and the k neighbours every kNN baseline shares.  Each class supplies: weight(t, p), the weight of a shared
        item whose last position in the prefix is p; normalise, whether v / sqrt(|I(c)| |I(n)|) is the similarity (else v, the
        weights' sum); W2 per session; W3 by distance inside a neighbour (None: no positions); W4(t), the table by the prefix
        distance of the neighbour's most recent shared item; F per item"""
        prefix = np.asarray(prefix, dtype=np.int64)
        t = len(prefix)
        u, first_rev = np.unique(prefix[::-1], return_index=True)
        last = t - first_rev                                      # 1-based position of the last occurrence
        o = np.argsort(last)
        ci, pos = u[o], last[o]
        wp = weight(t, pos)
        ioff, ranks, by_rank = self._postings()
        S = self.sample_size
        cand = np.unique(np.concatenate([ranks[ioff[i]:ioff[i] + min(ioff[i + 1] - ioff[i], S)] for i in ci]))[:S]
        sess = by_rank[cand]
        starts, lens = self.session_offsets[sess], np.diff(self.session_offsets)[sess]
        owner = np.repeat(np.arange(len(cand)), lens)
        at = np.repeat(starts - np.r_[0, np.cumsum(lens)[:-1]], lens) + np.arange(lens.sum())
        flat = self.session_items[at]
        fpos = None if w3 is None else self.positions[at]
        v, qr, dr = np.zeros(len(cand)), np.zeros(len(cand), np.int64), np.zeros(len(cand), np.int64)
        for m, i in enumerate(ci):                                # c's items in order of their last position
            sel = flat == i
            hit = np.zeros(len(cand), bool)
            hit[owner[sel]] = True
            v = v + np.where(hit, wp[m], 0.0)
            if w3 is not None:
                qr[owner[sel]] = fpos[sel]                        # ends at the shared item with the largest p_i
                dr[owner[sel]] = t - pos[m]
        sims = v / np.sqrt((len(ci) * lens).astype(np.float64)) if normalise else v
        if w2 is not None:
            sims = sims * w2[sess]
        g = sims if w4 is None else sims * w4(t)[dr]
        score = np.zeros(self.n_items)
        for q in np.lexsort((cand, -sims))[:self.k]:
            sel = owner == q
            score[flat[sel]] = score[flat[sel]] + (g[q] if w3 is None else g[q] * w3[np.abs(fpos[sel] - qr[q])])
        return score if f is None else score * f

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        if self.similarity == 'cosine':
            return self._knn_scores(prefix, lambda t, p: np.ones(len(p)), True)
        return self._knn_scores(prefix, lambda t, p: p / t, False)

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        score = self.score_prefix(self._prefix(session_id, self.itemidmap[input_item_id]))
        return pd.Series(data=score[self.itemidmap[predict_for_item_ids].values], index=predict_for_item_ids)


class STAN(SessionKNN):
    '''
    STAN(k=100, sample_size=500, lambda_spw=1.02, lambda_snh=432000.0, lambda_inh=2.05, session_key='SessionId', item_key='ItemId',
         time_key='Time')

    Session kNN with the three decays of STAN (Garg et al., SIGIR 2019): recent items of the current session, recent neighbour
    sessions and items close to the neighbour's most recent shared item count more.  This is this project's definition in the
    style of STAN (DESIGN §3p); it is not claimed to match any other implementation bit for bit.

    Everything SessionKNN defines stays: the item index, T(s), the recency order, the prefix c = (x_1 .. x_t), I(c) and the
    candidates.  A training session's events are ordered by time_key (ties by row order); q_n(j) is the 1-based position of item
    j's last occurrence in session n, p_i the last position of i in c.  The tables, computed by NumPy: W1[d] = exp(-(d /
    lambda_spw)), W2[n] = exp(-(float64(T_max - T(n)) / lambda_snh)) with T_max the largest training time, W3[d] = exp(-(d /
    lambda_inh)).  sim(n) = (sum of W1[t - p_i] over I(c) & I(n) in ascending p_i) / sqrt(|I(c)| |I(n)|) * W2[n]; the k
    largest (ties: the more recent) are the neighbours; score(j) is the float64 sum, in neighbour order, of sim(n) *
    W3[|q_n(j) - q_n(r(n))|] over the neighbours containing j, r(n) the shared item with the largest p_i.  A lambda of inf
    switches its decay off; with all three at inf the scores are SessionKNN(similarity='cosine')'s.  lambda_snh is in time_key
    units (the default is 5 days in seconds).
    '''
    _kind = 'stan'

    def __init__(self, k=100, sample_size=500, lambda_spw=1.02, lambda_snh=432000.0, lambda_inh=2.05, session_key='SessionId', item_key='ItemId',
                 time_key='Time'):
        self.k = k
        self.sample_size = sample_size
        self.lambda_spw = lambda_spw
        self.lambda_snh = lambda_snh
        self.lambda_inh = lambda_inh
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def fit(self, data):
        self._fit_index(data)
        self._device()

    def _fit_index(self, data):
        """the parameter checks, the index, positions, W2 and W3 on the host (no device work)"""
        self._check_neighbours()
        for name in ('lambda_spw', 'lambda_snh', 'lambda_inh'):
            if not float(getattr(self, name)) > 0.0:
                raise ValueError('%s must be in (0, inf], not %r' % (name, getattr(self, name)))
        col = data[self.time_key]
        if not pd.api.types.is_numeric_dtype(col) or pd.api.types.is_bool_dtype(col):
            raise ValueError('%s needs a numeric time column %r, not %s' % (type(self).__name__, self.time_key, col.dtype))
        idx, code, offsets, o = self._sessions(data, 'time')
        T = self._recency(code, col.values)
        S = self.n_sessions
        lens = np.diff(offsets)
        pos = np.arange(len(o)) - np.repeat(offsets[:-1], lens) + 1
        key = code[o].astype(np.int64) * self.n_items + idx[o].astype(np.int64)
        o2 = np.lexsort((pos, key))
        key, pos = key[o2], pos[o2]
        last = np.r_[key[1:] != key[:-1], True]                  # (session, item) distinct, items ascending; its last position
        self.session_items = (key[last] % self.n_items).astype(np.int32)
        self.positions = pos[last].astype(np.int32)
        self.session_offsets = np.zeros(S + 1, np.int64)
        self.session_offsets[1:] = np.cumsum(np.bincount(key[last] // self.n_items, minlength=S))
        self.w2 = np.exp(-((T.max() - T).astype(np.float64) / float(self.lambda_snh)))
        self.w3 = np.exp(-(np.arange(int(lens.max())) / float(self.lambda_inh)))
        self.current_session = None
        self._drop_caches()

    def _w1(self, n):
        return np.exp(-(np.arange(n) / float(self.lambda_spw)))

    def _upload(self, dev):
        dev.stan_fit(self.session_offsets, self.session_items, self.positions, self.recency, self.w2, self.w3, self.sample_size)
        dev.stan_set_w1(self._w1(len(self.w3)))

    def _cover(self, max_len):
        dev = self._device()
        if dev.n_w1 < max_len:
            dev.stan_set_w1(self._w1(max_len))

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        return self._knn_scores(prefix, lambda t, p: self._w1(t)[t - p], True, self.w2, self.w3)


class VSTAN(STAN):
    '''
    VSTAN(k=100, sample_size=500, similarity='cosine', lambda_spw=1.02, lambda_snh=432000.0, lambda_inh=2.05, lambda_ipw=1.02,
          lambda_idf=1.0, session_key='SessionId', item_key='ItemId', time_key='Time')

    STAN with the ideas of V-SKNN added back, in the style of VSTAN (Ludewig et al., RecSys 2019): an unnormalised ("vector")
    similarity, a neighbour that counts less when its most recent item shared with the session lies further back in the session,
    and IDF-weighted item scores.  This is this project's definition (DESIGN §3r); it is not claimed to match any other
    implementation bit for bit.

    Everything STAN defines stays: the index, T(s), the recency order, the candidates, p_i, q_n(j), W1, W2, W3 and r(n).  Two more
    tables, computed by NumPy: W4[d] = exp(-(d / lambda_ipw)) for the prefix distance d, and F[j] = 1 + lambda_idf * log(n_sessions /
    df_j), df_j the number of training sessions that contain j.  sim1 = v / sqrt(|I(c)| |I(n)|) ('cosine', STAN's) or v
    ('vector'), v the W1 sum; sim2 = sim1 * W2[n]; the k largest sim2 (ties: the more recent) are the neighbours; g(n) = sim2 *
    W4[t - p_r(n)]; score(j) = F[j] * (the float64 sum, in neighbour order, of g(n) * W3[|q_n(j) - q_n(r(n))|] over the neighbours
    containing j).  lambda_ipw = inf switches W4 off and lambda_idf = 0 sets F to 1: with similarity='cosine' and both, the scores
    are STAN's bit for bit.
    '''
    _kind = 'vstan'

    def __init__(self, k=100, sample_size=500, similarity='cosine', lambda_spw=1.02, lambda_snh=432000.0, lambda_inh=2.05, lambda_ipw=1.02,
                 lambda_idf=1.0, session_key='SessionId', item_key='ItemId', time_key='Time'):
        STAN.__init__(self, k, sample_size, lambda_spw, lambda_snh, lambda_inh, session_key, item_key, time_key)
        self.similarity = similarity
        self.lambda_ipw = lambda_ipw
        self.lambda_idf = lambda_idf

    def fit(self, data):
        self._check_similarity()
        if not float(self.lambda_ipw) > 0.0:
            raise ValueError('lambda_ipw must be in (0, inf], not %r' % (self.lambda_ipw,))
        if not 0.0 <= float(self.lambda_idf) < np.inf:
            raise ValueError('lambda_idf must be finite and >= 0, not %r' % (self.lambda_idf,))
        self._fit_index(data)
        df = np.bincount(self.session_items, minlength=self.n_items)   # the sessions that contain each item
        self.f = 1.0 + float(self.lambda_idf) * np.log(self.n_sessions / df)
        self._device()

    def _w4(self, n):
        return np.exp(-(np.arange(n) / float(self.lambda_ipw)))

    def _upload(self, dev):
        STAN._upload(self, dev)
        dev.vstan_set(self.similarity, self.f, self._w4(len(self.w3)))

    def _cover(self, max_len):
        STAN._cover(self, max_len)
        dev = self._device()
        if dev.n_w4 < max_len:
            dev.vstan_set(self.similarity, self.f, self._w4(max_len))

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        return self._knn_scores(prefix, lambda t, p: self._w1(t)[t - p], self.similarity != 'vector', self.w2, self.w3, self._w4, self.f)


class _Rules(Baseline):
    """What SR and AR share (DESIGN §3q): the training sequences, the device fit, the kept rows and predict_next from them"""

    def _n_keep(self):
        return self.pruning

    def _steps(self):
        return None, None

    def fit(self, data):
        self._integer('pruning', 1, _lib.KEEP_MAX)
        steps, weighting = self._steps()
        idx, _, offsets, o = self._sessions(data, 'time')
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.pruning)
        self.fit_stats = dev.rules_fit(offsets, idx[o], steps, weighting)
        self.rows = dev.rows_export()
        self._dev = dev

    def _upload(self, dev):
        dev.rows_import(*self.rows)

    predict_next = ItemKNN.predict_next


class SR(_Rules):
    '''
    SR(steps=10, weighting='div', pruning=20, session_key='SessionId', item_key='ItemId', time_key='Time')

    Sequential rules: a directed rule from an item to each item that follows it within `steps` events of a training session,
    weighted by the distance.  This is this project's definition (DESIGN §3q); it is not claimed to match any other implementation
    bit for bit.  A session's events are ordered by time_key (ties by row order): x_1 .. x_n, repeats kept.  w(i, j) is the sum
    over sessions and position pairs p < q <= p + steps with x_p = i, x_q = j and i != j of f(q - p), f(d) = 1 / d ('div') or 1
    ('same').  The device counts W = w * L exactly in uint64 (L = lcm(1 .. steps) for 'div', else 1) and divides once in float64.
    Each item keeps its `pruning` (1 .. 1024) largest weights (ties by the smaller item index); after input x, item j scores w(x, j)
    if kept, else 0.  SR(steps=1, weighting='same') is the first-order Markov baseline: transition counts, self-transitions
    dropped.  After fit, `rows` holds the kept rows (ItemKNN's layout) and `fit_stats` (pair work, scratch bytes, device ms).
    '''
    _kind = 'sr'

    def __init__(self, steps=10, weighting='div', pruning=20, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.steps = steps
        self.weighting = weighting
        self.pruning = pruning
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key

    def _steps(self):
        self._integer('steps', 1, _lib.RULES_STEPS_MAX)
        if self.weighting not in _lib.RULES_WEIGHTING:
            raise ValueError('weighting must be one of %s, not %r' % (sorted(_lib.RULES_WEIGHTING), self.weighting))
        return int(self.steps), self.weighting


class AR(_Rules):
    '''
    AR(pruning=20, session_key='SessionId', item_key='ItemId', time_key='Time')

    Association rules: co-occurrence within a training session, without normalisation.  This is this project's definition (DESIGN
    §3q).  w(i, j) = sum over sessions of occ_s(i) * occ_s(j) for i != j: every ordered pair of distinct positions holding i and
    j counts 1 (ItemKNN's cnt counts occ_s(i) * [j in s] instead, and divides by a norm).  Rows, scores and `fit_stats` as SR's.
    '''
    _kind = 'ar'

    def __init__(self, pruning=20, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.pruning = pruning
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key


def narm_pieces(offsets, items, max_len):
    """(piece offsets int64, piece items int32): every session of >= 2 events (items[offsets[s] .. offsets[s+1]) in time order)
    cut into pieces of at most max_len events, consecutive pieces overlapping by one event, so that every (input, next item)
    pair lies in exactly one piece; pieces in session order"""
    off = np.asarray(offsets, dtype=np.int64)
    items = np.asarray(items)
    lens = np.diff(off)
    m = int(max_len) - 1
    npc = np.where(lens >= 2, (lens - 1 + m - 1) // m, 0)
    sess = np.repeat(np.arange(len(lens)), npc)
    k = np.arange(int(npc.sum())) - np.repeat(np.cumsum(npc) - npc, npc)
    start = off[sess] + k * m
    plen = np.minimum(start + int(max_len), off[sess + 1]) - start
    poff = np.zeros(len(plen) + 1, np.int64)
    poff[1:] = np.cumsum(plen)
    at = np.repeat(start - poff[:-1], plen) + np.arange(int(poff[-1]))
    return poff, items[at].astype(np.int32)


NARM_PARAMS = ('E', 'Wx', 'Wrz', 'Wh', 'Bh', 'A1', 'A2', 'v', 'B')


def narm_shapes(n_items, d, H):
    """the parameters in the order of the flat vector (DESIGN §3s)"""
    return dict(E=(n_items, d), Wx=(d, 3 * H), Wrz=(H, 2 * H), Wh=(H, H), Bh=(3 * H,), A1=(H, H), A2=(H, H), v=(H,), B=(d, 2 * H))


def narm_unpack(flat, n_items, d, H):
    """name -> view of the flat parameter vector"""
    out, o = {}, 0
    for name, shp in narm_shapes(n_items, d, H).items():
        n = int(np.prod(shp))
        out[name] = flat[o:o + n].reshape(shp)
        o += n
    return out


def narm_init(n_items, d, H, rs):
    """the initial parameters, float32 flat: in the order of the vector each matrix [r x c] (v as [H x 1]) drawn from
    rs.uniform(-s, s) with s = sqrt(6 / (r + c)); Bh is 0 and takes no draw"""
    parts = []
    for name, shp in narm_shapes(n_items, d, H).items():
        if name == 'Bh':
            parts.append(np.zeros(shp))
            continue
        r, c = (shp[0], 1) if len(shp) == 1 else shp
        s = np.sqrt(6.0 / (r + c))
        parts.append(rs.uniform(-s, s, size=shp))
    return np.concatenate([p.ravel() for p in parts]).astype(np.float32)


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def narm_encode(p, x):
    """q (float64) of the inputs x (item indices, oldest first) in eval mode: p maps the parameter names to float64 arrays"""
    H = p['Wh'].shape[0]
    h = np.zeros(H)
    hs = []
    for it in x:
        vec = p['E'][it] @ p['Wx'] + p['Bh']
        rz = _sig(vec[H:] + h @ p['Wrz'])
        r, z = rz[:H], rz[H:]
        ht = np.tanh((h * r) @ p['Wh'] + vec[:H])
        h = (1.0 - z) * h + z * ht
        hs.append(h)
    hs = np.array(hs)
    alpha = _sig(p['A1'] @ h + hs @ p['A2'].T) @ p['v']
    return p['B'] @ np.concatenate([h, alpha @ hs])


class NARM(Baseline):
    '''
    NARM(embedding=50, hidden=100, n_epochs=10, batch_size=512, learning_rate=0.001, dropout_emb=0.25, dropout_ct=0.5, max_len=50,
         seed=42, session_key='SessionId', item_key='ItemId', time_key='Time')

    Neural attentive session model in the style of NARM (Li et al., CIKM 2017), trained on the device with full-catalogue
    cross-entropy and Adam.  This is this project's definition (DESIGN §3s); no parity with another framework is claimed.

    One item table E [n_items x embedding] is the input embedding and the decoder's item side.  For the last max_len inputs x_1 ..
    x_t of a session prefix: h_1 .. h_t is GRU4Rec's GRU cell over E[x] from a zero state, alpha_j = v . sig(A1 h_t + A2 h_j),
    c = [h_t ; sum_j alpha_j h_j], q = B c and item i scores E[i] . q.  Training cuts each session (events by time_key, ties by
    row order) into pieces of at most max_len events overlapping by one, encodes each piece causally, and per mini-batch of
    batch_size pieces takes one Adam step on the mean cross-entropy, with dropout_emb on the embeddings and dropout_ct on c.
    The parameters are float32 and drawn, like the epochs' piece orders, from np.random.RandomState(seed).  fit prints the
    epoch's mean loss; `fit_stats` holds per epoch (mean loss, device ms, per-step losses).  predict_next computes the scores on
    the host in float64 from the float32 parameters.
    '''
    _kind = 'narm'

    def __init__(self, embedding=50, hidden=100, n_epochs=10, batch_size=512, learning_rate=0.001, dropout_emb=0.25, dropout_ct=0.5,
                 max_len=50, seed=42, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.embedding = embedding
        self.hidden = hidden
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.learning_rate = learning_rate
        self.dropout_emb = dropout_emb
        self.dropout_ct = dropout_ct
        self.max_len = max_len
        self.seed = seed
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def _n_keep(self):
        return self.embedding

    def _check(self):
        self._integer('embedding', 1, 1024)
        self._integer('hidden', 1, 1024)
        self._integer('n_epochs', 0, 1 << 30)
        self._integer('batch_size', 1, 1 << 20)
        self._integer('max_len', 2, 512)
        if not 0.0 < float(self.learning_rate) < np.inf:
            raise ValueError('learning_rate must be finite and > 0, not %r' % (self.learning_rate,))
        for name in ('dropout_emb', 'dropout_ct'):
            if not 0.0 <= float(getattr(self, name)) < 1.0:
                raise ValueError('%s must be in [0, 1), not %r' % (name, getattr(self, name)))

    def pieces(self, data):
        """(piece offsets, piece items) of the training data, after the item index (_index)"""
        idx, _, offsets, o = self._sessions(data, 'time')
        return narm_pieces(offsets, idx[o], self.max_len)

    def fit(self, data):
        self._check()
        poff, pitems = self.pieces(data)
        if len(poff) < 2:
            raise ValueError('NARM needs a training session of at least 2 events')
        rs = np.random.RandomState(self.seed)
        params = narm_init(self.n_items, self.embedding, self.hidden, rs)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.embedding)
        dev.narm_begin(self.hidden, self.max_len, self.batch_size, poff, pitems, params)
        self.fit_stats = []
        for epoch in range(self.n_epochs):
            losses, ms = dev.narm_epoch(rs.permutation(len(poff) - 1), self.seed, self.learning_rate, self.dropout_emb, self.dropout_ct)
            mean = float(np.mean(losses.astype(np.float64)))
            self.fit_stats.append((mean, ms, losses))
            print(epoch, mean)
        self.params = dev.narm_export()
        dev.narm_import(self.hidden, self.max_len, self.params)   # ends the fit: the scratch leaves the device
        self.current_session = None
        self._dev = dev

    def _upload(self, dev):
        dev.narm_import(self.hidden, self.max_len, self.params)

    def params64(self):
        """name -> float64 copy of each parameter"""
        p = self.__dict__.get('_p64')
        if p is None:
            p = self._p64 = {k: v.astype(np.float64) for k, v in narm_unpack(self.params, self.n_items, self.embedding, self.hidden).items()}
        return p

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        p = self.params64()
        return p['E'] @ narm_encode(p, list(prefix)[-self.max_len:])

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        score = self.score_prefix(self._prefix(session_id, self.itemidmap[input_item_id]))
        return pd.Series(data=score[self.itemidmap[predict_for_item_ids].values], index=predict_for_item_ids)


SASREC_BLOCK = ('g1', 'c1', 'Wq', 'bq', 'Wk', 'bk', 'Wv', 'bv', 'Wo', 'bo', 'g2', 'c2', 'W1', 'b1', 'W2', 'b2')
SASREC_LN_EPS = 1e-8


def sasrec_shapes(n_items, d, n_blocks, max_len):
    """the parameters in the order of the flat vector (DESIGN §3t): E, Pe, per block b the SASREC_BLOCK names with suffix _b
    (W*: [d x d], the rest [d]), gf, cf"""
    out = dict(E=(n_items, d), Pe=(max_len, d))
    for b in range(n_blocks):
        for name in SASREC_BLOCK:
            out['%s_%d' % (name, b)] = (d, d) if name[0] == 'W' else (d,)
    out['gf'], out['cf'] = (d,), (d,)
    return out


def sasrec_unpack(flat, n_items, d, n_blocks, max_len):
    """name -> view of the flat parameter vector"""
    out, o = {}, 0
    for name, shp in sasrec_shapes(n_items, d, n_blocks, max_len).items():
        n = int(np.prod(shp))
        out[name] = flat[o:o + n].reshape(shp)
        o += n
    return out


def sasrec_init(n_items, d, n_blocks, max_len, rs):
    """the initial parameters, float32 flat: in the order of the vector each matrix [r x c] (E and Pe included) drawn from
    rs.uniform(-s, s) with s = sqrt(6 / (r + c)); biases 0 and gains 1, without draws"""
    parts = []
    for name, shp in sasrec_shapes(n_items, d, n_blocks, max_len).items():
        if len(shp) == 2:
            s = np.sqrt(6.0 / (shp[0] + shp[1]))
            parts.append(rs.uniform(-s, s, size=shp))
        else:
            parts.append(np.full(shp, 1.0 if name[0] == 'g' else 0.0))
    return np.concatenate([p.ravel() for p in parts]).astype(np.float32)


def sasrec_scales(d, n_heads):
    """(s_d, s_h): the float32 of sqrt(d) and of 1 / sqrt(d / n_heads), as float64"""
    return float(np.float32(np.sqrt(float(d)))), float(np.float32(1.0 / np.sqrt(float(d // n_heads))))


def _layer_norm(x, g, c):
    mu = x.mean(axis=-1, keepdims=True)
    var = ((x - mu) ** 2).mean(axis=-1, keepdims=True)
    return g * (x - mu) / np.sqrt(var + SASREC_LN_EPS) + c


def sasrec_encode(p, x, n_heads):
    """q (float64) of the inputs x (item indices, oldest first, at most max_len) in eval mode: p maps the parameter names to
    float64 arrays"""
    d = p['E'].shape[1]
    dh = d // n_heads
    sd, sh = sasrec_scales(d, n_heads)
    n = len(x)
    h = p['E'][list(x)] * sd + p['Pe'][:n]
    causal = np.tril(np.ones((n, n), bool))
    b = 0
    while 'g1_%d' % b in p:
        w = {name: p['%s_%d' % (name, b)] for name in SASREC_BLOCK}
        u = _layer_norm(h, w['g1'], w['c1'])
        Q, K, V = u @ w['Wq'] + w['bq'], u @ w['Wk'] + w['bk'], u @ w['Wv'] + w['bv']
        A = np.empty_like(h)
        for k in range(n_heads):
            cs = slice(k * dh, (k + 1) * dh)
            S = np.where(causal, (Q[:, cs] @ K[:, cs].T) * sh, -np.inf)
            P = np.exp(S - S.max(axis=1, keepdims=True))
            A[:, cs] = (P / P.sum(axis=1, keepdims=True)) @ V[:, cs]
        a = h + A @ w['Wo'] + w['bo']
        h = a + np.maximum(_layer_norm(a, w['g2'], w['c2']) @ w['W1'] + w['b1'], 0.0) @ w['W2'] + w['b2']
        b += 1
    return _layer_norm(h[-1], p['gf'], p['cf'])


class SASRec(Baseline):
    '''
    SASRec(embedding=50, n_blocks=2, n_heads=1, n_epochs=10, batch_size=128, learning_rate=0.001, dropout=0.2, max_len=50, seed=42,
           session_key='SessionId', item_key='ItemId', time_key='Time')

    Self-attentive sequential recommender in the style of SASRec (Kang & McAuley, ICDM 2018), trained on the device with
    full-catalogue cross-entropy and Adam.  This is this project's definition (DESIGN §3t); no parity with another framework is
    claimed.

    One item table E [n_items x embedding] is the input embedding and the output item side.  For the last max_len inputs x_0 ..
    x_(n-1) of a session prefix: h_t = E[x_t] sqrt(d) + Pe[t]; n_blocks pre-LN Transformer blocks, each causal multi-head
    attention (n_heads heads) and a position-wise ReLU FFN with residuals; q_t = LN(h_t) and item i scores E[i] . q.  Training
    cuts each session (events by time_key, ties by row order) into pieces of at most max_len + 1 events overlapping by one,
    encodes each piece causally, and per mini-batch of batch_size pieces takes one Adam step on the mean cross-entropy over its
    positions, with dropout on h0 and on both residual branches of every block.  The parameters are float32 and drawn, like the
    epochs' piece orders, from np.random.RandomState(seed).  fit prints the epoch's mean loss; `fit_stats` holds per epoch (mean
    loss, device ms, per-step losses).  predict_next computes the scores on the host in float64 from the float32 parameters.
    '''
    _kind = 'sasrec'

    def __init__(self, embedding=50, n_blocks=2, n_heads=1, n_epochs=10, batch_size=128, learning_rate=0.001, dropout=0.2, max_len=50,
                 seed=42, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.embedding = embedding
        self.n_blocks = n_blocks
        self.n_heads = n_heads
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.learning_rate = learning_rate
        self.dropout = dropout
        self.max_len = max_len
        self.seed = seed
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def _n_keep(self):
        return self.embedding

    def _check(self):
        self._integer('embedding', 1, 1024)
        self._integer('n_heads', 1, self.embedding)
        if self.embedding % self.n_heads:
            raise ValueError('n_heads must divide embedding, not %r into %r' % (self.n_heads, self.embedding))
        self._integer('n_blocks', 1, 8)
        self._integer('n_epochs', 0, 1 << 30)
        self._integer('batch_size', 1, 1 << 20)
        self._integer('max_len', 1, 512)
        if (self.n_blocks + 1) * self.batch_size * self.max_len * self.embedding >= 1 << 32:
            raise ValueError('(n_blocks + 1) * batch_size * max_len * embedding must stay below 2^32 (dropout indices)')
        if not 0.0 < float(self.learning_rate) < np.inf:
            raise ValueError('learning_rate must be finite and > 0, not %r' % (self.learning_rate,))
        if not 0.0 <= float(self.dropout) < 1.0:
            raise ValueError('dropout must be in [0, 1), not %r' % (self.dropout,))

    def pieces(self, data):
        """(piece offsets, piece items) of the training data, after the item index (_index): pieces of at most max_len inputs"""
        idx, _, offsets, o = self._sessions(data, 'time')
        return narm_pieces(offsets, idx[o], self.max_len + 1)

    def fit(self, data):
        self._check()
        poff, pitems = self.pieces(data)
        if len(poff) < 2:
            raise ValueError('SASRec needs a training session of at least 2 events')
        rs = np.random.RandomState(self.seed)
        params = sasrec_init(self.n_items, self.embedding, self.n_blocks, self.max_len, rs)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.embedding)
        dev.sasrec_begin(self.n_blocks, self.n_heads, self.max_len, self.batch_size, poff, pitems, params)
        self.fit_stats = []
        for epoch in range(self.n_epochs):
            losses, ms = dev.sasrec_epoch(rs.permutation(len(poff) - 1), self.seed, self.learning_rate, self.dropout)
            mean = float(np.mean(losses.astype(np.float64)))
            self.fit_stats.append((mean, ms, losses))
            print(epoch, mean)
        self.params = dev.sasrec_export()
        self._upload(dev)                        # ends the fit: the scratch leaves the device
        self.current_session = None
        self._dev = dev

    def _upload(self, dev):
        dev.sasrec_import(self.n_blocks, self.n_heads, self.max_len, self.params)

    def params64(self):
        """name -> float64 copy of each parameter"""
        p = self.__dict__.get('_p64')
        if p is None:
            flat = self.params
            p = self._p64 = {k: v.astype(np.float64) for k, v in
                             sasrec_unpack(flat, self.n_items, self.embedding, self.n_blocks, self.max_len).items()}
        return p

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        p = self.params64()
        return p['E'] @ sasrec_encode(p, list(prefix)[-self.max_len:], self.n_heads)

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        score = self.score_prefix(self._prefix(session_id, self.itemidmap[input_item_id]))
        return pd.Series(data=score[self.itemidmap[predict_for_item_ids].values], index=predict_for_item_ids)


SRGNN_PARAMS = ('E', 'W_in', 'W_out', 'b_in', 'b_out', 'b_iah', 'b_oah', 'W_ih', 'b_ih', 'W_hh', 'b_hh', 'W1', 'W2', 'b1', 'b2', 'q', 'W3', 'b3')


def srgnn_shapes(n_items, d):
    """the parameters in the order of the flat vector (DESIGN §3u)"""
    sq, v = (d, d), (d,)
    return dict(E=(n_items, d), W_in=sq, W_out=sq, b_in=v, b_out=v, b_iah=v, b_oah=v, W_ih=(2 * d, 3 * d), b_ih=(3 * d,), W_hh=(d, 3 * d),
                b_hh=(3 * d,), W1=sq, W2=sq, b1=v, b2=v, q=v, W3=(2 * d, d), b3=v)


def srgnn_unpack(flat, n_items, d):
    """name -> view of the flat parameter vector"""
    out, o = {}, 0
    for name, shp in srgnn_shapes(n_items, d).items():
        n = int(np.prod(shp))
        out[name] = flat[o:o + n].reshape(shp)
        o += n
    return out


def srgnn_init(n_items, d, rs):
    """the initial parameters, float32 flat: every entry (biases and E included), in the order of the vector, drawn from
    rs.uniform(-s, s) with s = 1 / sqrt(d)"""
    s = 1.0 / np.sqrt(d)
    n = sum(int(np.prod(shp)) for shp in srgnn_shapes(n_items, d).values())
    return rs.uniform(-s, s, size=n).astype(np.float32)


def srgnn_graph(x):
    """the graph of inputs x: (nodes: the distinct items ascending, alias: the node of each position, A_in, A_out [K x K]) with
    an edge u -> v for each consecutive pair (a repeat once, self-loops kept), A_in[v][u] = 1 / indeg(v), A_out[u][v] =
    1 / outdeg(u) and zero rows for nodes without such edges"""
    nodes, alias = np.unique(np.asarray(x, dtype=np.int64), return_inverse=True)
    K = len(nodes)
    adj = np.zeros((K, K))
    adj[alias[:-1], alias[1:]] = 1.0
    indeg, outdeg = adj.sum(axis=0), adj.sum(axis=1)
    a_in = adj.T / np.where(indeg > 0, indeg, 1.0)[:, None]
    a_out = adj / np.where(outdeg > 0, outdeg, 1.0)[:, None]
    return nodes, alias, a_in, a_out


def srgnn_encode(p, x, step):
    """s_h (float64) of the inputs x (item indices, oldest first, at most max_len): p maps the parameter names to float64 arrays"""
    d = p['E'].shape[1]
    nodes, alias, a_in, a_out = srgnn_graph(x)
    H = p['E'][nodes]
    for _ in range(step):
        a = np.concatenate([a_in @ (H @ p['W_in'] + p['b_in']) + p['b_iah'], a_out @ (H @ p['W_out'] + p['b_out']) + p['b_oah']], axis=1)
        gi, gh = a @ p['W_ih'] + p['b_ih'], H @ p['W_hh'] + p['b_hh']
        r = _sig(gi[:, :d] + gh[:, :d])
        z = _sig(gi[:, d:2 * d] + gh[:, d:2 * d])
        n = np.tanh(gi[:, 2 * d:] + r * gh[:, 2 * d:])
        H = n + z * (H - n)
    h = H[alias]
    alpha = _sig(h[-1] @ p['W1'] + p['b1'] + h @ p['W2'] + p['b2']) @ p['q']
    return np.concatenate([alpha @ h, h[-1]]) @ p['W3'] + p['b3']


class SRGNN(Baseline):
    '''
    SRGNN(embedding=100, step=1, n_epochs=10, batch_size=100, learning_rate=0.001, lr_decay=0.1, lr_decay_step=3, l2=1e-5, max_len=50,
          seed=42, session_key='SessionId', item_key='ItemId', time_key='Time')

    Session-graph model in the style of SR-GNN (Wu et al., AAAI 2019), trained on the device with full-catalogue cross-entropy and
    Adam.  This is this project's definition (DESIGN §3u); no parity with another framework is claimed.

    One item table E [n_items x embedding] is the node embedding and the scored item side.  The last max_len inputs of a session
    prefix become a directed graph of their distinct items (an edge per consecutive pair, a repeat once) with in- and
    out-adjacency normalised by degree; `step` gated propagation steps with shared weights update the node states; the hybrid
    readout s_h = W3 [s_g ; s_l] + b3 joins the last position's state s_l with s_g = sum_t alpha_t h_t, alpha_t = q . sig(W1 s_l +
    b1 + W2 h_t + b2); item i scores E[i] . s_h.  Training takes every (prefix, next item) pair of every session (events by
    time_key, ties by row order) as its own sample, and per mini-batch of batch_size samples one Adam step on the mean
    cross-entropy plus l2 theta (coupled L2), at learning_rate lr_decay^(epoch // lr_decay_step).  The parameters are float32
    and drawn, like the epochs' sample orders, from np.random.RandomState(seed).  fit prints the epoch's mean loss;
    `fit_stats` holds per epoch (mean loss, device ms, per-step losses).  predict_next computes the scores on the host in float64
    from the float32 parameters.
    '''
    _kind = 'srgnn'

    def __init__(self, embedding=100, step=1, n_epochs=10, batch_size=100, learning_rate=0.001, lr_decay=0.1, lr_decay_step=3, l2=1e-5,
                 max_len=50, seed=42, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.embedding = embedding
        self.step = step
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.learning_rate = learning_rate
        self.lr_decay = lr_decay
        self.lr_decay_step = lr_decay_step
        self.l2 = l2
        self.max_len = max_len
        self.seed = seed
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def _n_keep(self):
        return self.embedding

    def _check(self):
        self._integer('embedding', 1, 1024)
        self._integer('step', 1, 8)
        self._integer('n_epochs', 0, 1 << 30)
        self._integer('batch_size', 1, 1 << 20)
        self._integer('max_len', 1, 512)
        self._integer('lr_decay_step', 1, 1 << 30)
        if self.batch_size * self.max_len * (self.step + 1) * 3 * self.embedding >= 1 << 31:
            raise ValueError('batch_size * max_len * (step + 1) * 3 * embedding must stay below 2^31 (flat indices of a batch)')
        if not 0.0 < float(self.learning_rate) < np.inf:
            raise ValueError('learning_rate must be finite and > 0, not %r' % (self.learning_rate,))
        if not 0.0 < float(self.lr_decay) < np.inf:
            raise ValueError('lr_decay must be finite and > 0, not %r' % (self.lr_decay,))
        if not 0.0 <= float(self.l2) < np.inf:
            raise ValueError('l2 must be finite and >= 0, not %r' % (self.l2,))

    def sessions(self, data):
        """(session offsets, items in time order) of the training data, after the item index (_index)"""
        idx, _, offsets, o = self._sessions(data, 'time')
        return offsets, idx[o].astype(np.int32)

    def learning_rates(self):
        """the learning rate of each epoch: learning_rate lr_decay^(epoch // lr_decay_step), as the float32 the device takes"""
        return [float(np.float32(self.learning_rate * self.lr_decay ** (e // self.lr_decay_step))) for e in range(self.n_epochs)]

    def fit(self, data):
        self._check()
        offsets, items = self.sessions(data)
        n_samples = int(np.maximum(np.diff(offsets) - 1, 0).sum())
        if n_samples < 1:
            raise ValueError('SRGNN needs a training session of at least 2 events')
        rates = self.learning_rates()
        if not all(0.0 < r < np.inf for r in rates):
            raise ValueError('every epoch\'s learning rate must be finite and > 0 in float32, not %r' % (rates,))
        rs = np.random.RandomState(self.seed)
        params = srgnn_init(self.n_items, self.embedding, rs)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.embedding)
        dev.srgnn_begin(self.step, self.max_len, self.batch_size, offsets, items, params)
        self.fit_stats = []
        for epoch, lr in enumerate(rates):
            losses, ms = dev.srgnn_epoch(rs.permutation(n_samples), lr, self.l2)
            mean = float(np.mean(losses.astype(np.float64)))
            self.fit_stats.append((mean, ms, losses))
            print(epoch, mean)
        self.params = dev.srgnn_export()
        self._upload(dev)                        # ends the fit: the scratch leaves the device
        self.current_session = None
        self._dev = dev

    def _upload(self, dev):
        dev.srgnn_import(self.step, self.max_len, self.params)

    def params64(self):
        """name -> float64 copy of each parameter"""
        p = self.__dict__.get('_p64')
        if p is None:
            p = self._p64 = {k: v.astype(np.float64) for k, v in srgnn_unpack(self.params, self.n_items, self.embedding).items()}
        return p

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        p = self.params64()
        return p['E'] @ srgnn_encode(p, list(prefix)[-self.max_len:], self.step)

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        score = self.score_prefix(self._prefix(session_id, self.itemidmap[input_item_id]))
        return pd.Series(data=score[self.itemidmap[predict_for_item_ids].values], index=predict_for_item_ids)


STAMP_PARAMS = ('E', 'W1', 'W2', 'W3', 'b_a', 'w0', 'Ws', 'bs', 'Wt', 'bt')
STAMP_BIASES = ('b_a', 'bs', 'bt')


def stamp_shapes(n_items, d):
    """the parameters in the order of the flat vector (DESIGN §3v)"""
    sq, v = (d, d), (d,)
    return dict(E=(n_items, d), W1=sq, W2=sq, W3=sq, b_a=v, w0=v, Ws=sq, bs=v, Wt=sq, bt=v)


def stamp_unpack(flat, n_items, d):
    """name -> view of the flat parameter vector"""
    out, o = {}, 0
    for name, shp in stamp_shapes(n_items, d).items():
        n = int(np.prod(shp))
        out[name] = flat[o:o + n].reshape(shp)
        o += n
    return out


def stamp_init(n_items, d, init_std, rs):
    """the initial parameters, float32 flat: in the order of the vector every weight (E and w0 included) drawn from
    rs.normal(0, init_std); the biases b_a, bs and bt are 0 and take no draw"""
    parts = [np.zeros(shp) if name in STAMP_BIASES else rs.normal(0.0, init_std, size=shp) for name, shp in stamp_shapes(n_items, d).items()]
    return np.concatenate([p.ravel() for p in parts]).astype(np.float32)


def stamp_encode(p, x):
    """q (float64) of the inputs x (item indices, oldest first, at most max_len): p maps the parameter names to float64 arrays"""
    X = p['E'][list(x)]
    mt, ms = X[-1], X.mean(axis=0)
    a = _sig(X @ p['W1'] + mt @ p['W2'] + ms @ p['W3'] + p['b_a']) @ p['w0']
    return np.tanh(a @ X @ p['Ws'] + p['bs']) * np.tanh(mt @ p['Wt'] + p['bt'])


class STAMP(Baseline):
    '''
    STAMP(embedding=100, n_epochs=10, batch_size=512, learning_rate=0.005, init_std=0.05, max_len=50, seed=42, session_key='SessionId',
          item_key='ItemId', time_key='Time')

    Short-term attention/memory priority model in the style of STAMP (Liu et al., KDD 2018), trained on the device with
    full-catalogue cross-entropy and Adam.  This is this project's definition (DESIGN §3v); no parity with another framework is
    claimed.

    One item table E [n_items x embedding] is the input embedding and the scored item side.  For the last max_len inputs x_1 ..
    x_n of a session prefix: the session mean m_s, the last click m_t = x_n, the attention a_i = w0 . sig(x_i W1 + m_t W2 + m_s W3
    + b_a) (not normalised), m_a = sum_i a_i x_i, h_s = tanh(m_a Ws + bs), h_t = tanh(m_t Wt + bt) and q = h_s * h_t; item i scores
    E[i] . q (the paper's sigmoid around it is left out: it does not change a ranking).  Training takes every (prefix, next item)
    pair of every session (events by time_key, ties by row order) as its own sample, and per mini-batch of batch_size samples one
    Adam step on the mean cross-entropy.  The weights are float32 and drawn from N(0, init_std^2), the biases 0; the draws and
    the epochs' sample orders come from np.random.RandomState(seed).  fit prints the epoch's mean loss; `fit_stats` holds per
    epoch (mean loss, device ms, per-step losses).  predict_next computes the scores on the host in float64 from the float32
    parameters.
    '''
    _kind = 'stamp'

    def __init__(self, embedding=100, n_epochs=10, batch_size=512, learning_rate=0.005, init_std=0.05, max_len=50, seed=42,
                 session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.embedding = embedding
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.learning_rate = learning_rate
        self.init_std = init_std
        self.max_len = max_len
        self.seed = seed
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def _n_keep(self):
        return self.embedding

    def _check(self):
        self._integer('embedding', 1, 1024)
        self._integer('n_epochs', 0, 1 << 30)
        self._integer('batch_size', 1, 1 << 20)
        self._integer('max_len', 1, 512)
        if self.batch_size * self.max_len * 2 * self.embedding >= 1 << 31:
            raise ValueError('batch_size * max_len * 2 * embedding must stay below 2^31 (flat indices of a batch)')
        if not 0.0 < float(self.learning_rate) < np.inf:
            raise ValueError('learning_rate must be finite and > 0, not %r' % (self.learning_rate,))
        if not 0.0 < float(self.init_std) < np.inf:
            raise ValueError('init_std must be finite and > 0, not %r' % (self.init_std,))

    def sessions(self, data):
        """(session offsets, items in time order) of the training data, after the item index (_index)"""
        idx, _, offsets, o = self._sessions(data, 'time')
        return offsets, idx[o].astype(np.int32)

    def fit(self, data):
        self._check()
        offsets, items = self.sessions(data)
        n_samples = int(np.maximum(np.diff(offsets) - 1, 0).sum())
        if n_samples < 1:
            raise ValueError('STAMP needs a training session of at least 2 events')
        rs = np.random.RandomState(self.seed)
        params = stamp_init(self.n_items, self.embedding, self.init_std, rs)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.embedding)
        dev.stamp_begin(self.max_len, self.batch_size, offsets, items, params)
        self.fit_stats = []
        for epoch in range(self.n_epochs):
            losses, ms = dev.stamp_epoch(rs.permutation(n_samples), self.learning_rate)
            mean = float(np.mean(losses.astype(np.float64)))
            self.fit_stats.append((mean, ms, losses))
            print(epoch, mean)
        self.params = dev.stamp_export()
        self._upload(dev)                        # ends the fit: the scratch leaves the device
        self.current_session = None
        self._dev = dev

    def _upload(self, dev):
        dev.stamp_import(self.max_len, self.params)

    def params64(self):
        """name -> float64 copy of each parameter"""
        p = self.__dict__.get('_p64')
        if p is None:
            p = self._p64 = {k: v.astype(np.float64) for k, v in stamp_unpack(self.params, self.n_items, self.embedding).items()}
        return p

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        p = self.params64()
        return p['E'] @ stamp_encode(p, list(prefix)[-self.max_len:])

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        score = self.score_prefix(self._prefix(session_id, self.itemidmap[input_item_id]))
        return pd.Series(data=score[self.itemidmap[predict_for_item_ids].values], index=predict_for_item_ids)


NEXTITNET_BLOCK = ('C1', 'c1', 'g1', 'n1', 'C2', 'c2', 'g2', 'n2')


def nextitnet_shapes(n_items, d, dilations, kernel_size):
    """the parameters in the order of the flat vector (DESIGN §3w): E, per block b the NEXTITNET_BLOCK names with suffix _b (C*:
    [kernel_size d x d], row k d + i tap k and input channel i; the rest [d]), W, bW"""
    out = dict(E=(n_items, d))
    for b in range(len(dilations)):
        for name in NEXTITNET_BLOCK:
            out['%s_%d' % (name, b)] = (kernel_size * d, d) if name[0] == 'C' else (d,)
    out['W'], out['bW'] = (n_items, d), (n_items,)
    return out


def nextitnet_unpack(flat, n_items, d, dilations, kernel_size):
    """name -> view of the flat parameter vector"""
    out, o = {}, 0
    for name, shp in nextitnet_shapes(n_items, d, dilations, kernel_size).items():
        n = int(np.prod(shp))
        out[name] = flat[o:o + n].reshape(shp)
        o += n
    return out


def nextitnet_init(n_items, d, dilations, kernel_size, rs):
    """the initial parameters, float32 flat: in the order of the vector each matrix [r x c] (E and W included) drawn from
    rs.uniform(-s, s) with s = sqrt(6 / (r + c)); biases 0 and gains 1, without draws"""
    parts = []
    for name, shp in nextitnet_shapes(n_items, d, dilations, kernel_size).items():
        if len(shp) == 2:
            s = np.sqrt(6.0 / (shp[0] + shp[1]))
            parts.append(rs.uniform(-s, s, size=shp))
        else:
            parts.append(np.full(shp, 1.0 if name[0] == 'g' else 0.0))
    return np.concatenate([p.ravel() for p in parts]).astype(np.float32)


def _causal_taps(x, K, l):
    """[n, K d]: row t holds x[t - (K - 1 - k) l] for k = 0 .. K - 1, zeros before the start"""
    n, d = x.shape
    out = np.zeros((n, K * d))
    for k in range(K):
        back = (K - 1 - k) * l
        if back < n:
            out[back:, k * d:(k + 1) * d] = x[:n - back]
    return out


def nextitnet_encode(p, x, dilations, kernel_size):
    """q (float64) of the inputs x (item indices, oldest first, at most max_len): the encoder's last position; p maps the parameter
    names to float64 arrays"""
    h = p['E'][list(x)]
    for b, l in enumerate(dilations):
        w = {name: p['%s_%d' % (name, b)] for name in NEXTITNET_BLOCK}
        a = np.maximum(_layer_norm(_causal_taps(h, kernel_size, l) @ w['C1'] + w['c1'], w['g1'], w['n1']), 0.0)
        h = h + np.maximum(_layer_norm(_causal_taps(a, kernel_size, 2 * l) @ w['C2'] + w['c2'], w['g2'], w['n2']), 0.0)
    return h[-1]


class NextItNet(Baseline):
    '''
    NextItNet(embedding=100, dilations=(1, 2, 1, 2, 1, 2), kernel_size=3, n_epochs=10, batch_size=128, learning_rate=0.001, max_len=50,
              seed=42, session_key='SessionId', item_key='ItemId', time_key='Time')

    Convolutional sequence model in the style of NextItNet (Yuan et al., WSDM 2019), trained on the device with full-catalogue
    cross-entropy and Adam.  This is this project's definition (DESIGN §3w); no parity with another framework is claimed.  The
    defaults follow the style of the published code's configuration and were not checked against the paper's experiments.

    The input embedding E [n_items x embedding] and the output side W [n_items x embedding], bW [n_items] are separate tables.  For
    the last max_len inputs x_0 .. x_(n-1) of a session prefix, positions before 0 reading zeros: h_t = E[x_t]; one residual block
    per dilation l, u_t = c1 + sum_k h_(t - (K-1-k) l) C1[k], a = relu(LN1(u)), v_t = c2 + sum_k a_(t - (K-1-k) 2l) C2[k] and
    h'_t = h_t + relu(LN2(v)), with K = kernel_size; q is the last position's h and item i scores W[i] . q + bW[i].  Training cuts
    each session (events by time_key, ties by row order) into pieces of at most max_len + 1 events overlapping by one, encodes each
    piece causally, and per mini-batch of batch_size pieces takes one Adam step on the mean cross-entropy over its positions.
    There is no dropout.  The parameters are float32 and drawn, like the epochs' piece orders, from np.random.RandomState(seed).
    fit prints the epoch's mean loss; `fit_stats` holds per epoch (mean loss, device ms, per-step losses).  predict_next computes
    the scores on the host in float64 from the float32 parameters.
    '''
    _kind = 'nextitnet'

    def __init__(self, embedding=100, dilations=(1, 2, 1, 2, 1, 2), kernel_size=3, n_epochs=10, batch_size=128, learning_rate=0.001,
                 max_len=50, seed=42, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.embedding = embedding
        self.dilations = dilations
        self.kernel_size = kernel_size
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.learning_rate = learning_rate
        self.max_len = max_len
        self.seed = seed
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def _n_keep(self):
        return self.embedding

    def _check(self):
        self._integer('embedding', 1, 1024)
        self._integer('kernel_size', 1, 8)
        dl = self.dilations
        if (isinstance(dl, (str, bytes)) or not hasattr(dl, '__len__') or not 1 <= len(dl) <= 16 or
                any(isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 1 <= v <= 256 for v in dl)):
            raise ValueError('dilations must be 1 .. 16 integers, each in 1 .. 256, not %r' % (dl,))
        self._integer('n_epochs', 0, 1 << 30)
        self._integer('batch_size', 1, 1 << 20)
        self._integer('max_len', 1, 512)
        if not 0.0 < float(self.learning_rate) < np.inf:
            raise ValueError('learning_rate must be finite and > 0, not %r' % (self.learning_rate,))

    def pieces(self, data):
        """(piece offsets, piece items) of the training data, after the item index (_index): pieces of at most max_len inputs"""
        idx, _, offsets, o = self._sessions(data, 'time')
        return narm_pieces(offsets, idx[o], self.max_len + 1)

    def fit(self, data):
        self._check()
        poff, pitems = self.pieces(data)
        if len(poff) < 2:
            raise ValueError('NextItNet needs a training session of at least 2 events')
        rs = np.random.RandomState(self.seed)
        params = nextitnet_init(self.n_items, self.embedding, self.dilations, self.kernel_size, rs)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.embedding)
        dev.nextitnet_begin(self.dilations, self.kernel_size, self.max_len, self.batch_size, poff, pitems, params)
        self.fit_stats = []
        for epoch in range(self.n_epochs):
            losses, ms = dev.nextitnet_epoch(rs.permutation(len(poff) - 1), self.learning_rate)
            mean = float(np.mean(losses.astype(np.float64)))
            self.fit_stats.append((mean, ms, losses))
            print(epoch, mean)
        self.params = dev.nextitnet_export()
        self._upload(dev)                        # ends the fit: the scratch leaves the device
        self.current_session = None
        self._dev = dev

    def _upload(self, dev):
        dev.nextitnet_import(self.dilations, self.kernel_size, self.max_len, self.params)

    def params64(self):
        """name -> float64 copy of each parameter"""
        p = self.__dict__.get('_p64')
        if p is None:
            p = self._p64 = {k: v.astype(np.float64) for k, v in
                             nextitnet_unpack(self.params, self.n_items, self.embedding, self.dilations, self.kernel_size).items()}
        return p

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        p = self.params64()
        return p['W'] @ nextitnet_encode(p, list(prefix)[-self.max_len:], self.dilations, self.kernel_size) + p['bW']

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        score = self.score_prefix(self._prefix(session_id, self.itemidmap[input_item_id]))
        return pd.Series(data=score[self.itemidmap[predict_for_item_ids].values], index=predict_for_item_ids)


BERT4REC_BLOCK = ('Wq', 'bq', 'Wk', 'bk', 'Wv', 'bv', 'Wo', 'bo', 'g1', 'c1', 'W1', 'b1', 'W2', 'b2', 'g2', 'c2')


def bert4rec_shapes(n_items, d, n_blocks, max_len):
    """the parameters in the order of the flat vector (DESIGN §3x): E (n_items + 1 rows, the last the mask token), Pe, g0, c0, per
    block b the BERT4REC_BLOCK names with suffix _b (Wq .. Wo: [d x d], W1: [d x 4d], b1: [4d], W2: [4d x d], the rest [d]), Wp,
    bp, gp, cp, bO [n_items]"""
    out = dict(E=(n_items + 1, d), Pe=(max_len, d), g0=(d,), c0=(d,))
    for b in range(n_blocks):
        for name in BERT4REC_BLOCK:
            out['%s_%d' % (name, b)] = {'W1': (d, 4 * d), 'b1': (4 * d,), 'W2': (4 * d, d)}.get(name, (d, d) if name[0] == 'W' else (d,))
    out['Wp'], out['bp'], out['gp'], out['cp'], out['bO'] = (d, d), (d,), (d,), (d,), (n_items,)
    return out


def bert4rec_unpack(flat, n_items, d, n_blocks, max_len):
    """name -> view of the flat parameter vector"""
    out, o = {}, 0
    for name, shp in bert4rec_shapes(n_items, d, n_blocks, max_len).items():
        n = int(np.prod(shp))
        out[name] = flat[o:o + n].reshape(shp)
        o += n
    return out


def bert4rec_init(n_items, d, n_blocks, max_len, rs):
    """the initial parameters, float32 flat, by sasrec_init's rule: in the order of the vector each matrix [r x c] (E and Pe
    included) drawn from rs.uniform(-s, s) with s = sqrt(6 / (r + c)); biases 0 and gains 1, without draws"""
    parts = []
    for name, shp in bert4rec_shapes(n_items, d, n_blocks, max_len).items():
        if len(shp) == 2:
            s = np.sqrt(6.0 / (shp[0] + shp[1]))
            parts.append(rs.uniform(-s, s, size=shp))
        else:
            parts.append(np.full(shp, 1.0 if name[0] == 'g' else 0.0))
    return np.concatenate([p.ravel() for p in parts]).astype(np.float32)


def bert4rec_masks(piece_offsets, mask_prob, rs):
    """the cloze masks of one epoch, uint8 per stored entry: one rs.random_sample over the entries in storage order, an entry masked
    when its draw is below mask_prob, and a piece with no masked entry gets its last entry masked"""
    off = np.asarray(piece_offsets, dtype=np.int64)
    mk = (rs.random_sample(int(off[-1])) < mask_prob).astype(np.uint8)
    none = np.add.reduceat(mk.astype(np.int64), off[:-1]) == 0 if len(off) > 1 else np.zeros(0, bool)
    mk[off[1:][none] - 1] = 1
    return mk


_erf = np.frompyfunc(math.erf, 1, 1)


def _gelu(x):
    """exact-erf GELU, x Phi(x)"""
    return 0.5 * x * (1.0 + _erf(x / np.sqrt(2.0)).astype(np.float64))


def bert4rec_encode(p, x, n_heads):
    """q (float64) of the inputs x (item indices, oldest first, at most max_len - 1) followed by the mask token: the head's output at
    the mask; p maps the parameter names to float64 arrays"""
    d = p['E'].shape[1]
    dh = d // n_heads
    sh = sasrec_scales(d, n_heads)[1]
    x = list(x) + [p['E'].shape[0] - 1]
    n = len(x)
    h = _layer_norm(p['E'][x] + p['Pe'][:n], p['g0'], p['c0'])
    b = 0
    while 'g1_%d' % b in p:
        w = {name: p['%s_%d' % (name, b)] for name in BERT4REC_BLOCK}
        Q, K, V = h @ w['Wq'] + w['bq'], h @ w['Wk'] + w['bk'], h @ w['Wv'] + w['bv']
        A = np.empty_like(h)
        for k in range(n_heads):
            cs = slice(k * dh, (k + 1) * dh)
            S = (Q[:, cs] @ K[:, cs].T) * sh
            P = np.exp(S - S.max(axis=1, keepdims=True))
            A[:, cs] = (P / P.sum(axis=1, keepdims=True)) @ V[:, cs]
        a = _layer_norm(h + A @ w['Wo'] + w['bo'], w['g1'], w['c1'])
        h = _layer_norm(a + _gelu(a @ w['W1'] + w['b1']) @ w['W2'] + w['b2'], w['g2'], w['c2'])
        b += 1
    return _layer_norm(_gelu(h[-1] @ p['Wp'] + p['bp']), p['gp'], p['cp'])


class BERT4Rec(Baseline):
    '''
    BERT4Rec(embedding=64, n_blocks=2, n_heads=2, n_epochs=10, batch_size=256, learning_rate=0.001, dropout=0.1, mask_prob=0.2,
             max_len=50, seed=42, session_key='SessionId', item_key='ItemId', time_key='Time')

    Bidirectional self-attentive sequential recommender in the style of BERT4Rec (Sun et al., CIKM 2019), trained on the device by
    the cloze objective with full-catalogue cross-entropy and Adam.  This is this project's definition (DESIGN §3x); no parity with
    another framework is claimed.  The defaults follow the paper's architecture (embedding 64, 2 blocks of 2 heads, dropout 0.1,
    max_len 50); the paper's training budget (about 400k steps at learning rate 1e-4), its weight decay and its learning-rate
    schedule are not reproduced, and the defaults were not checked against the paper's experiments.

    One item table E [(n_items + 1) x embedding], whose last row is the mask token, is the input embedding and the output item
    side.  For inputs x_0 .. x_(n-1), some of them the mask token: h = drop(LN0(E[x_t] + Pe[t])); n_blocks post-LN Transformer
    blocks, a = LN1(h + drop(A Wo + bo)) with A multi-head softmax attention over all n positions, h = LN2(a + drop(gelu(a W1 +
    b1) W2 + b2)); the head q_t = LNp(gelu(h_t Wp + bp)), and item i scores E[i] . q_t + bO[i].  Training cuts each session (events
    by time_key, ties by row order) into pieces of at most max_len events overlapping by one; each epoch masks every entry with
    probability mask_prob (a piece with none gets its last entry masked, see bert4rec_masks), replaces the masked entries by the
    mask token and, per mini-batch of batch_size pieces, takes one Adam step on the mean cross-entropy over the masked positions,
    with dropout on h0 and on both residual branches of every block.  A prefix is scored from its last max_len - 1 inputs followed
    by the mask token, q the head's output at the mask.  The parameters are float32 and drawn, like the epochs' piece orders and
    masks, from np.random.RandomState(seed).  fit prints the epoch's mean loss; `fit_stats` holds per epoch (mean loss, device ms,
    per-step losses).  predict_next computes the scores on the host in float64 from the float32 parameters.
    '''
    _kind = 'bert4rec'

    def __init__(self, embedding=64, n_blocks=2, n_heads=2, n_epochs=10, batch_size=256, learning_rate=0.001, dropout=0.1, mask_prob=0.2,
                 max_len=50, seed=42, session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.embedding = embedding
        self.n_blocks = n_blocks
        self.n_heads = n_heads
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.learning_rate = learning_rate
        self.dropout = dropout
        self.mask_prob = mask_prob
        self.max_len = max_len
        self.seed = seed
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.current_session = None

    def _n_keep(self):
        return self.embedding

    def _check(self):
        self._integer('embedding', 1, 1024)
        self._integer('n_heads', 1, self.embedding)
        if self.embedding % self.n_heads:
            raise ValueError('n_heads must divide embedding, not %r into %r' % (self.n_heads, self.embedding))
        self._integer('n_blocks', 1, 8)
        self._integer('n_epochs', 0, 1 << 30)
        self._integer('batch_size', 1, 1 << 20)
        self._integer('max_len', 2, 512)
        if (self.n_blocks + 1) * self.batch_size * self.max_len * self.embedding >= 1 << 32:
            raise ValueError('(n_blocks + 1) * batch_size * max_len * embedding must stay below 2^32 (dropout indices)')
        if not 0.0 < float(self.learning_rate) < np.inf:
            raise ValueError('learning_rate must be finite and > 0, not %r' % (self.learning_rate,))
        if not 0.0 <= float(self.dropout) < 1.0:
            raise ValueError('dropout must be in [0, 1), not %r' % (self.dropout,))
        if not 0.0 <= float(self.mask_prob) <= 1.0:
            raise ValueError('mask_prob must be in [0, 1], not %r' % (self.mask_prob,))

    def pieces(self, data):
        """(piece offsets, piece items) of the training data, after the item index (_index): pieces of at most max_len events, all
        of them inputs"""
        idx, _, offsets, o = self._sessions(data, 'time')
        return narm_pieces(offsets, idx[o], self.max_len)

    def fit(self, data):
        self._check()
        poff, pitems = self.pieces(data)
        if len(poff) < 2:
            raise ValueError('BERT4Rec needs a training session of at least 2 events')
        rs = np.random.RandomState(self.seed)
        params = bert4rec_init(self.n_items, self.embedding, self.n_blocks, self.max_len, rs)
        self._drop_caches()
        dev = _lib.Baselines(self._kind, self.n_items, self.embedding)
        dev.bert4rec_begin(self.n_blocks, self.n_heads, self.max_len, self.batch_size, poff, pitems, params)
        self.fit_stats = []
        for epoch in range(self.n_epochs):
            order = rs.permutation(len(poff) - 1)
            masks = bert4rec_masks(poff, self.mask_prob, rs)
            losses, ms = dev.bert4rec_epoch(order, masks, self.seed, self.learning_rate, self.dropout)
            mean = float(np.mean(losses.astype(np.float64)))
            self.fit_stats.append((mean, ms, losses))
            print(epoch, mean)
        self.params = dev.bert4rec_export()
        self._upload(dev)                        # ends the fit: the scratch leaves the device
        self.current_session = None
        self._dev = dev

    def _upload(self, dev):
        dev.bert4rec_import(self.n_blocks, self.n_heads, self.max_len, self.params)

    def params64(self):
        """name -> float64 copy of each parameter"""
        p = self.__dict__.get('_p64')
        if p is None:
            p = self._p64 = {k: v.astype(np.float64) for k, v in
                             bert4rec_unpack(self.params, self.n_items, self.embedding, self.n_blocks, self.max_len).items()}
        return p

    def score_prefix(self, prefix):
        """float64 scores [n_items] after the session's input item indices so far `prefix` (the current input last)"""
        p = self.params64()
        return p['E'][:self.n_items] @ bert4rec_encode(p, list(prefix)[-(self.max_len - 1):], self.n_heads) + p['bO']

    def predict_next(self, session_id, input_item_id, predict_for_item_ids):
        score = self.score_prefix(self._prefix(session_id, self.itemidmap[input_item_id]))
        return pd.Series(data=score[self.itemidmap[predict_for_item_ids].values], index=predict_for_item_ids)
