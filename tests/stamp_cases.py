"""The STAMP case table shared by tests/test_gpu_stamp.py and, without a GPU, tests/test_host_stamp_shapes.py, which checks that
the table reaches every branch of g4r_stamp.cuh's kernels (constants read from the header)."""
import os
import re

import numpy as np

import stamp_oracle as sto

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gru4rec_b200', 'csrc', 'g4r_stamp.cuh')


def constants():
    """the ST_* integer constants of g4r_stamp.cuh"""
    with open(HEADER) as f:
        src = f.read()
    return {k: int(v) for k, v in re.findall(r'\b(ST_[A-Z_]+) = (\d+)', src)}


def _rsc15(rs, n, NI):
    """RSC15-like sessions: lengths 2 .. with mean about 3.5, some items repeated"""
    out = []
    for _ in range(n):
        k = 2 + rs.geometric(0.6)
        pool = rs.randint(0, NI, max(1, k // 2 + rs.randint(0, 3)))
        out.append([int(pool[rs.randint(len(pool))]) if rs.rand() < 0.35 else int(rs.randint(NI)) for _ in range(k)])
    return out


def _special(rs, NI, max_len):
    """sessions whose samples hit the kernels' corners: a full-length prefix and one cut to its last max_len inputs (two longer
    sessions), repeated items, a target that is also an input, one item repeated"""
    a, b, c = (int(v) for v in rs.randint(0, NI, 3))
    longs = [list(rs.randint(0, NI, max_len + 1)), list(rs.randint(0, max(2, NI // 50), max_len + 3))]
    return longs + [[a, a, b, a], [c, c, c, c], [a, b, c, a, b, c, a], [b, c, b]]


def _case(id, NI, d, max_len, bs, seed, scale=1.0, repeat=False):
    return dict(id=id, NI=NI, d=d, max_len=max_len, bs=bs, seed=seed, scale=scale, repeat=repeat)


INIT_STD = 0.05
GRAD_CASES = [
    _case('shipped', 37483, 100, 50, 512, 1),
    _case('items172k', 172000, 100, 50, 64, 2),
    _case('trained_scale', 5000, 64, 50, 100, 3, scale=16.0),
    _case('max_len512', 3000, 16, 512, 12, 4),
    _case('d1024', 2000, 1024, 20, 24, 5),
    _case('d1', 200, 1, 10, 40, 6),
    _case('d37', 1000, 37, 30, 40, 7),
    _case('batch1', 500, 24, 50, 1, 8),
    _case('repeated_sample', 1000, 24, 30, 40, 9, repeat=True),
]


def grad_batch(case):
    """(sessions, sample order of one batch, batch_size, rs): batch_size samples, the longest one first, then the special sessions'
    corner samples, a repeated case with its first sample twice"""
    rs = np.random.RandomState(case['seed'])
    L = case['max_len']
    sessions = _special(rs, case['NI'], L) + _rsc15(rs, 400, case['NI'])
    if L >= 512:
        sessions = [list(rs.randint(0, case['NI'], 520)), list(rs.randint(0, 40, 300))] + sessions
    smp = sto.samples(sessions, L)
    n_special = sum(len(s) - 1 for s in sessions[:len(sessions) - 400])
    lens = np.array([len(x) for x, _ in smp])
    first = [int(np.argmax(lens))] + list(range(n_special))[::max(1, n_special // max(1, case['bs'] // 2))]
    rest = [k for k in rs.permutation(len(smp)) if k not in set(first)]
    order = (first + rest)[:case['bs']]
    if case['repeat']:
        order[1] = order[0]
    return sessions, np.array(order, np.int32), case['bs'], rs


def case_params(case, rs):
    """float32 flat parameters of a case: the init, or at a trained model's scale E x scale and every other parameter x 4, the
    biases drawn at that scale too"""
    th = sto.init(case['NI'], case['d'], INIT_STD, rs)
    if case['scale'] != 1.0:
        p = sto.unpack(th, case['NI'], case['d'])
        p = {k: (rs.normal(0.0, 4 * INIT_STD, size=v.shape) if k in sto.BIASES else v * (case['scale'] if k == 'E' else 4.0)) for k, v in p.items()}
        th = sto.pack(p).astype(np.float32)
    return th


EVAL_CASES = [
    dict(id='shipped', NI=5000, d=100, max_len=50, seed=11, n=6000),
    dict(id='len512', NI=2000, d=16, max_len=512, seed=12, n=5000),
]


def eval_sessions(case):
    """(items, offsets, n_history) of an evaluation case: RSC15-like sessions plus long ones past max_len, history on some"""
    rs = np.random.RandomState(case['seed'])
    L = case['max_len']
    sessions = _rsc15(rs, case['n'], case['NI'])
    for k in rs.choice(len(sessions), 12, replace=False):
        sessions[k] = list(rs.randint(0, case['NI'], L + 2 + rs.randint(0, 60)))
    lens = np.array([len(s) for s in sessions])
    nh = np.where(rs.rand(len(sessions)) < 0.3, rs.randint(0, 4, len(sessions)), 0).astype(np.int32)
    nh = np.minimum(nh, lens).astype(np.int32)
    return np.concatenate(sessions).astype(np.int32), np.r_[0, np.cumsum(lens)].astype(np.int64), nh


def eval_chunks(offsets, n_history, max_len, cap):
    """the chunk of every counted event under NARM's evaluation planner: per session one piece from its start for the prefixes of
    at most max_len inputs and a window of the last max_len inputs for each longer one, up to cap positions and pieces per chunk"""
    out, P, npc, c = [], 0, 0, 0

    def piece(n):
        nonlocal P, npc, c
        if P + n > cap or npc >= cap:
            c, P, npc = c + 1, 0, 0
        P += n
        npc += 1

    for s in range(len(offsets) - 1):
        i0 = max(int(n_history[s]) if n_history is not None else 0, 1) - 1
        last = int(offsets[s + 1] - offsets[s]) - 2
        if last < i0:
            continue
        if i0 < max_len:
            n = min(last + 1, max_len)
            piece(n)
            out += [c] * (n - i0)
        for _ in range(max(i0, max_len), last + 1):
            piece(max_len)
            out.append(c)
    return np.array(out)
