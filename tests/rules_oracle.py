"""The rule-based baselines restated with explicit loops (DESIGN §3q): sequential rules (SR) and association rules (AR).  Counts are
Python integers, the weight is float(W) / L in float64 (each step correctly rounded, as the device's __ull2double_rn and
__ddiv_rn), and each row keeps its `pruning` largest weights by (weight desc, index asc).  The rows have the layout of
baselines_oracle.knn_rows, so baselines_oracle.rank_events('itemknn', (n_items, rows), ...) ranks them.  Test infrastructure."""
import numpy as np


def scale(steps, weighting):
    """L = lcm(1 .. steps) for SR 'div', 1 for SR 'same' and for AR (steps None)"""
    L = 1
    if steps is not None and weighting == 'div':
        for d in range(2, steps + 1):
            a, b = L, d
            while b:
                a, b = b, a % b
            L = L * d // a
    return L


def sequences(sessions, items, times):
    """(session offsets, items) of the training events: sessions in order of first appearance, each one's events by time with
    ties by row order"""
    first, seqs = {}, []
    for r, s in enumerate(sessions):
        if s not in first:
            first[s] = len(seqs)
            seqs.append([])
        seqs[first[s]].append((times[r], r, int(items[r])))
    off, flat = [0], []
    for q in seqs:
        flat += [x for _, _, x in sorted(q, key=lambda e: (e[0], e[1]))]
        off.append(len(flat))
    return np.array(off, np.int64), np.array(flat, np.int64)


def counts(offsets, items, n_items, steps=None, weighting=None):
    """W as one dict per row {j: int}: SR (steps 1 .. 20) sums L * f(q - p) over position pairs p < q <= p + steps with
    x_p = i != j = x_q, f(d) = 1 / d ('div') or 1 ('same'); AR (steps None) counts every ordered pair of distinct positions holding
    i != j, which is occ_s(i) * occ_s(j) per session"""
    L = scale(steps, weighting)
    W = [dict() for _ in range(n_items)]
    for s in range(len(offsets) - 1):
        x = [int(v) for v in items[offsets[s]:offsets[s + 1]]]
        n = len(x)
        for p in range(n):
            qs = range(n) if steps is None else range(p + 1, min(p + steps, n - 1) + 1)
            for q in qs:
                i, j = x[p], x[q]
                if i == j:
                    continue
                add = 1 if (steps is None or weighting == 'same') else L // (q - p)
                W[i][j] = W[i].get(j, 0) + add
    return W


def rows(offsets, items, n_items, pruning, steps=None, weighting=None):
    """{item index: (kept indices int64, kept weights float64)} by (weight desc, index asc)"""
    L = float(scale(steps, weighting))
    out = {}
    for i, row in enumerate(counts(offsets, items, n_items, steps, weighting)):
        j = np.array(sorted(row), np.int64)
        w = np.array([float(row[c]) / L for c in j.tolist()], np.float64)
        o = np.lexsort((j, -w))[:pruning]
        out[i] = (j[o], w[o])
    return out


def dense(rows_, n_items, pruning):
    """the rows in g4r_bl_rows_export's layout: idx [n_items, pruning] (-1 past len), w (0 past len), len"""
    idx = np.full((n_items, pruning), -1, np.int32)
    w = np.zeros((n_items, pruning))
    ln = np.zeros(n_items, np.int32)
    for i, (j, v) in rows_.items():
        idx[i, :len(j)] = j
        w[i, :len(j)] = v
        ln[i] = len(j)
    return idx, w, ln
