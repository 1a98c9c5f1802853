"""The SR-GNN case table shared by tests/test_gpu_srgnn.py and, without a GPU, tests/test_host_srgnn_shapes.py, which checks that
the table reaches every branch of g4r_srgnn.cuh's kernels (constants read from the header)."""
import os
import re

import numpy as np

import srgnn_oracle as so

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gru4rec_b200', 'csrc', 'g4r_srgnn.cuh')


def constants():
    """the SG_* integer constants of g4r_srgnn.cuh"""
    with open(HEADER) as f:
        src = f.read()
    return {k: int(v) for k, v in re.findall(r'\b(SG_[A-Z_]+) = (\d+)', src)}


def _rsc15(rs, n, NI, max_len):
    """RSC15-like sessions: lengths 2 .. with mean about 3.5, some items repeated (and so self-loops and revisits)"""
    out = []
    for _ in range(n):
        k = 2 + rs.geometric(0.6)
        pool = rs.randint(0, NI, max(1, k // 2 + rs.randint(0, 3)))
        s = [int(pool[rs.randint(len(pool))]) if rs.rand() < 0.35 else int(rs.randint(NI)) for _ in range(k)]
        out.append(s)
    return out


def _special(rs, NI, max_len):
    """sessions whose samples hit the graph's corners: a full-length prefix (and one cut to the last max_len inputs), a self-loop,
    a single node repeated, a revisit of every node, one input"""
    a, b, c = (int(v) for v in rs.randint(0, NI, 3))
    longs = [list(rs.randint(0, NI, max_len + 1)), list(rs.randint(0, max(2, NI // 50), max_len + 3))]
    return longs + [[a, a, b, a], [c, c, c, c], [a, b, c, a, b, c, a], [b, c]]


def _case(id, NI, d, step, max_len, bs, seed, scale=1.0, repeat=False):
    return dict(id=id, NI=NI, d=d, step=step, max_len=max_len, bs=bs, seed=seed, scale=scale, repeat=repeat)


GRAD_CASES = [
    _case('shipped', 37483, 100, 1, 50, 100, 1),
    _case('step3', 3000, 32, 3, 50, 64, 2),
    _case('step8', 500, 8, 8, 20, 32, 3),
    _case('trained_scale', 5000, 64, 1, 50, 100, 4, scale=8.0),
    _case('items172k', 172000, 100, 1, 50, 100, 5),
    _case('max_len512', 3000, 16, 1, 512, 12, 6),
    _case('d1024', 2000, 1024, 1, 20, 24, 7),
    _case('d1', 200, 1, 2, 10, 40, 8),
    _case('repeated_sample', 1000, 24, 2, 30, 40, 9, repeat=True),
]


def grad_batch(case):
    """(sessions, sample order of one batch, batch_size, rs): batch_size samples with the special sessions' corner samples first,
    a repeated case with its first sample twice"""
    rs = np.random.RandomState(case['seed'])
    L = case['max_len']
    sessions = _special(rs, case['NI'], L) + _rsc15(rs, 400, case['NI'], L)
    if L >= 512:
        sessions = [list(rs.randint(0, case['NI'], 520)), list(rs.randint(0, 40, 300))] + sessions
    smp = so.samples(sessions, L)
    n_special = sum(len(s) - 1 for s in sessions[:len(sessions) - 400])
    lens = np.array([len(x) for x, _ in smp])
    first = [int(np.argmax(lens))] + list(range(n_special))[::max(1, n_special // (case['bs'] // 2))]
    rest = [k for k in rs.permutation(len(smp)) if k not in set(first)]
    order = (first + rest)[:case['bs']]
    if case['repeat']:
        order[1] = order[0]
        order = order[:case['bs']]
    return sessions, np.array(order, np.int32), case['bs'], rs


EVAL_CASES = [
    dict(id='shipped', NI=5000, d=100, step=1, max_len=50, seed=11, n=3500),
    dict(id='step3_len512', NI=2000, d=16, step=3, max_len=512, seed=12, n=600),
]


def eval_sessions(case):
    """(items, offsets, n_history) of an evaluation case: RSC15-like sessions plus long ones past max_len, history on some"""
    rs = np.random.RandomState(case['seed'])
    L = case['max_len']
    sessions = _rsc15(rs, case['n'], case['NI'], L)
    for k in rs.choice(len(sessions), 12, replace=False):
        sessions[k] = list(rs.randint(0, case['NI'], L + 2 + rs.randint(0, 60)))
    lens = np.array([len(s) for s in sessions])
    nh = np.where(rs.rand(len(sessions)) < 0.3, rs.randint(0, 4, len(sessions)), 0).astype(np.int32)
    nh = np.minimum(nh, lens).astype(np.int32)
    return np.concatenate(sessions).astype(np.int32), np.r_[0, np.cumsum(lens)].astype(np.int64), nh


def eval_positions(offsets, n_history, max_len):
    """per counted event (evaluate's order) its sample's inputs, as the device plans them"""
    out = []
    for s in range(len(offsets) - 1):
        i0 = max(int(n_history[s]) if n_history is not None else 0, 1) - 1
        out += [min(i + 1, max_len) for i in range(i0, int(offsets[s + 1] - offsets[s]) - 1)]
    return np.array(out)


def eval_chunks(offsets, n_history, max_len, cap):
    """the chunk of every counted event under the device's planner: positions up to cap per chunk"""
    out, P, c = [], 0, 0
    for n in eval_positions(offsets, n_history, max_len):
        if P + n > cap:
            c, P = c + 1, 0
        out.append(c)
        P += n
    return np.array(out)
