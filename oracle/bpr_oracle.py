"""float64 NumPy restatement of BPR-MF (the reference's baselines.py:303-418) as the device computes it (DESIGN §3k): the fit with
the reference's random draws and update formulas, its dot products in the device's order (lane-strided sequential sums, then a
fixed shuffle tree); the longest chain of dependent updates; the session vectors, scores and per-event counts of the evaluation in
the device's pinned k-order.  Test infrastructure: the device (g4r_bpr.cuh) is compared against it, and it is compared against
the reference's recorded runs (tests/golden/baselines/bpr_*.npz)."""
import numpy as np

from baselines_oracle import tie_noise, MODES  # noqa: F401

LANES = 32


def iteration_draws(n_rows, n_items):
    """one iteration's draws from the global np.random state, vectorised: the permutation of the rows, then one randint(n_items)
    per event (a row index; the negative item is that row's item)"""
    perm = np.random.permutation(n_rows)
    return perm, np.random.randint(n_items, size=n_rows)


def iteration_draws_loop(n_rows, n_items):
    """the same draws as the reference's loop takes them (baselines.py:381-384)"""
    perm = np.random.permutation(n_rows)
    return perm, np.array([np.random.randint(n_items) for _ in perm], dtype=np.int64)


def warp_dot(a, b):
    """sum(a * b) as k_bpr_sgd forms it: lane l adds the products of f = l, l + 32, ... in order, then a butterfly over the lanes"""
    F = len(a)
    prod = a * b
    v = np.zeros(LANES)
    for c in range(0, F, LANES):
        w = min(LANES, F - c)
        v[:w] = v[:w] + prod[c:c + w]
    lane = np.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        v = v + v[lane ^ o]
    return v[0]


def fit(row_session, row_item, U, I, bI, draws, learning_rate, lambda_session, lambda_item):
    """the reference's SGD (baselines.py:349-358) over the iterations' (perm, negrow) draws, in place on copies of U and I.
    Returns (U, I, per-iteration np.mean(log sigm) as the reference prints it, per-iteration longest chain of dependent updates)"""
    U, I = np.array(U, dtype=np.float64), np.array(I, dtype=np.float64)
    lr, ls, li = learning_rate, lambda_session, lambda_item
    means, levels = [], []
    for perm, negrow in draws:
        c_list = []
        lastU, lastI = {}, {}
        top = 0
        for t, e in enumerate(perm):
            u, p, n = row_session[e], row_item[e], row_item[negrow[t]]
            uF, iF1, iF2 = U[u].copy(), I[p].copy(), I[n].copy()
            x = ((warp_dot(iF1, uF) - warp_dot(iF2, uF)) + bI[p]) - bI[n]
            sigm = 1.0 / (1.0 + np.exp(-x))
            c = 1.0 - sigm
            U[u] += lr * (c * (iF1 - iF2) - ls * uF)
            I[p] += lr * (c * uF - li * iF1)
            I[n] += lr * (-c * uF - li * iF2)
            c_list.append(np.log(sigm))
            lv = 1 + max(lastU.get(u, 0), lastI.get(p, 0), lastI.get(n, 0))
            lastU[u] = lastI[p] = lastI[n] = lv
            top = max(top, lv)
        means.append(np.mean(c_list))
        levels.append(top)
    return U, I, means, levels


def session_vector(I, prefix):
    """mean of the prefix's item rows: the sequential row sum over the prefix divided by its length"""
    acc = np.zeros(I.shape[1])
    for x in prefix:
        acc = acc + I[x]
    return acc / len(prefix)


def scores(I, bI, uF):
    """every item's score: the products I[j, f] * uF[f] summed over f in order, then + bI[j]"""
    s = np.zeros(I.shape[0])
    for f in range(I.shape[1]):
        s = s + I[:, f] * uF[f]
    return s + bI


def rank_events(I, bI, items, offsets, n_history=None, mode='standard', cand=None, exclude_seen=False, k=0):
    """baselines_oracle.rank_events for BPR: per counted event (data order) counts int64 [n, 2] ((-1, -1) for an exclude_seen
    miss), and with k > 0 the lists (items [n, k], -1 past the eligible ones; scores [n, k] float64, NaN there)"""
    n_items = I.shape[0]
    items = np.asarray(items, dtype=np.int64)
    w0 = np.ones(n_items, np.int64) if cand is None else np.bincount(np.asarray(cand, dtype=np.int64), minlength=n_items)
    counts, li, ls = [], [], []
    e = 0
    for s in range(len(offsets) - 1):
        st, en = int(offsets[s]), int(offsets[s + 1])
        h = 0 if n_history is None else int(n_history[s])
        acc = np.zeros(I.shape[1])
        for p in range(st, en - 1):
            acc = acc + I[items[p]]
            if p < st + max(h, 1) - 1:
                continue
            y = items[p + 1]
            prefix = items[st:p + 1]
            sc = scores(I, bI, acc / (p - st + 1))
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
