"""The NextItNet test shapes (DESIGN §3w), shared by tests/test_gpu_nextitnet.py (the device against the float64 oracle) and
tests/test_host_nextitnet_shapes.py (which checks, without a GPU, that the table reaches every branch of g4r_nextitnet.cuh's
gather and gather-sum kernels, the model's limits, nm_gemm's split rule at these shapes and several evaluation chunks).

GRAD_CASES are one training mini-batch each: the pieces (lists of item indices, max_len + 1 events at most) as the fit holds them,
the batch (indices into the pieces, in slot order; a piece may appear twice), the batch_size the fit is begun with and a parameter
scale.  EVAL_CASES are one nextitnet_encode call each.  Everything is drawn from seeded RandomStates.  The evaluation's piece and
chunk planner and nm_gemm's split rule are NARM's (narm_cases restates them)."""
import os
import re

import numpy as np

import narm_cases as nc

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gru4rec_b200', 'csrc', 'g4r_nextitnet.cuh')
SHIPPED_DIL = (1, 2, 1, 2, 1, 2)


def constants():
    """NI_D_MAX, NI_K_MAX, NI_BLOCKS_MAX, NI_DIL_MAX, NI_LEN_MAX, NI_EVAL_PAIRS as g4r_nextitnet.cuh defines them"""
    with open(HEADER) as f:
        src = f.read()
    return {name: int(re.search(r'\b%s\s*=\s*(\d+)' % name, src).group(1))
            for name in ('NI_D_MAX', 'NI_K_MAX', 'NI_BLOCKS_MAX', 'NI_DIL_MAX', 'NI_LEN_MAX', 'NI_EVAL_PAIRS')}


def products(P, NI, d, K):
    """ni_grad's products: name -> (role, M, N, K) (every block's convolution products have the same shape)"""
    return {'conv': ('encoder', P, d, K * d), 'S': ('catalogue', P, NI, d), 'dQ': ('catalogue', P, d, NI), 'dW': ('catalogue', NI, d, P),
            'dbW': ('backward', 1, NI, P), 'dC': ('backward', K * d, d, P), 'db': ('backward', 1, d, P), 'dCOL': ('backward', P, K * d, d)}


def eval_plan(offsets, n_history, max_len):
    return nc.eval_plan(offsets, n_history, max_len, constants()['NI_EVAL_PAIRS'])


def receptive_field(dilations, K):
    """how far back q_t reaches: block b's two convolutions see (K - 1) l and (K - 1) 2 l positions back"""
    return (K - 1) * sum(3 * l for l in dilations)


def _shipped(rs, NI, max_len=50, n=128, n_full=4):
    """n pieces cut from RSC15-like sessions of Zipf items, n_full of them full (max_len inputs), in a shuffled order"""
    lens = nc.rsc15_lengths(rs, 4 * n)
    items = rs.zipf(1.2, size=int(lens.sum())) % NI
    sessions = np.split(items, np.cumsum(lens)[:-1])
    pieces = [p for p in nc.cut(sessions, max_len + 1) if len(p) <= max_len][:n - n_full]
    pieces += [list(rs.zipf(1.2, size=max_len + 1) % NI) for _ in range(n_full)]
    return [pieces[k] for k in rs.permutation(len(pieces))]


def _inputs(rs, NI, inputs):
    return [list(rs.randint(0, NI, k + 1)) for k in inputs]


def _uniform(rs, n, NI, max_len):
    """one 1-input piece, one max_len piece, the rest uniform"""
    return _inputs(rs, NI, np.r_[1, max_len, rs.randint(1, max_len + 1, n - 2)])


def _tile(rs, NI, inputs):
    """a batch of exactly sum(inputs) positions, P_max of the fit, whose first piece is repeated in slot 1; the fit also holds an
    unused piece as long as the first, so that the batch_size longest distinct pieces cover the batch exactly"""
    pieces = _inputs(rs, NI, [inputs[0]] + list(inputs[1:]) + [inputs[0]])
    return pieces, [0, 0] + list(range(1, len(inputs)))


def _case(id, NI, d, dil, K, max_len, build, seed, scale=1.0):
    """build(rs) -> pieces or (pieces, batch); the parameters are drawn after the pieces from the same RandomState"""
    return dict(id=id, NI=NI, d=d, dil=tuple(dil), K=K, max_len=max_len, build=build, seed=seed, scale=scale)


def grad_batch(case):
    """(pieces, batch, batch_size, rs): rs positioned for the parameters' draw"""
    rs = np.random.RandomState(case['seed'])
    out = case['build'](rs)
    pieces, batch = out if isinstance(out, tuple) else (out, list(range(len(out))))
    return pieces, np.asarray(batch), len(batch), rs


GRAD_CASES = [
    # the shipped shape: scripts/nextitnet_bench.py's training step
    _case('shipped', 37483, 100, SHIPPED_DIL, 3, 50, lambda rs: _shipped(rs, 37483), 1),
    # trained-model scale: E and W x scale, the kernels x 2, random gains and biases (the test asserts a logit spread >= 30)
    _case('trained-scale', 5000, 48, (1, 2, 4), 3, 20, lambda rs: _uniform(rs, 40, 5000, 20), 2, scale=16.0),
    _case('kernel-1', 2000, 32, (1, 2), 1, 20, lambda rs: _uniform(rs, 24, 2000, 20), 3),
    _case('kernel-5', 2000, 24, (1, 3, 2), 5, 30, lambda rs: _uniform(rs, 24, 2000, 30), 4),
    # every shifted tap of both convolutions lies before the start of every piece (dilation 64 > max_len 20)
    _case('taps-before-start', 1500, 16, (64, 1), 3, 20, lambda rs: _uniform(rs, 16, 1500, 20), 5),
    # a piece of exactly max_len = 512 inputs; the widest dilation reaches across most of it
    _case('length-512', 3000, 32, (1, 16, 128), 3, 512, lambda rs: _inputs(rs, 3000, [512, 300, 129, 1]), 6),
    _case('d-1024', 1000, 1024, (1, 2), 3, 8, lambda rs: _uniform(rs, 5, 1000, 8), 7),
    _case('catalogue-172000', 172000, 64, SHIPPED_DIL, 3, 50, lambda rs: _inputs(rs, 172000, np.r_[1, 50, rs.randint(1, 11, 10)]), 8),
    _case('blocks-16', 1000, 16, (1, 2, 4, 8) * 4, 3, 40, lambda rs: _uniform(rs, 12, 1000, 40), 9),
    _case('d-1', 500, 1, (1,), 3, 1, lambda rs: _inputs(rs, 500, [1] * 9), 10),
    _case('pmax', 129, 12, (1, 2), 2, 24, lambda rs: _tile(rs, 129, [2, 11, 13, 17, 19, 1]), 11),
]


def eval_sessions(case):
    """(items int32, offsets int64, n_history int32) of an evaluation case"""
    rs = np.random.RandomState(case['seed'])
    lens = case['lengths'](rs)
    items = rs.zipf(1.2, size=int(lens.sum())) % case['NI']
    nh = np.where(rs.rand(len(lens)) < 0.2, rs.randint(0, 8, len(lens)), 0)
    nh = np.minimum(nh, lens)
    return items.astype(np.int32), np.r_[0, np.cumsum(lens)].astype(np.int64), nh.astype(np.int32)


def _rsc15_with_long(rs, n_events, n_long, long_len):
    lens = nc.rsc15_lengths(rs, n_events)
    at = rs.choice(len(lens), n_long, replace=False)
    lens[at] = long_len
    return lens


EVAL_CASES = [
    # the shipped shape: RSC15-like sessions, a few of 120 events (windows), history counts on about a fifth of the sessions
    dict(id='shipped', NI=37483, d=100, dil=SHIPPED_DIL, K=3, max_len=50, seed=31, lengths=lambda rs: _rsc15_with_long(rs, 30000, 8, 120)),
    # long windows: sessions past max_len = 512, a receptive field wider than the window
    dict(id='len-512', NI=3000, d=32, dil=(1, 32, 128), K=3, max_len=512, seed=32,
         lengths=lambda rs: np.r_[560, 2, 1, rs.randint(2, 40, 30), 530, 512, 513, 300, rs.randint(400, 520, 40)]),
]
