"""The BERT4Rec test shapes (DESIGN §3x), shared by tests/test_gpu_bert4rec.py (the device against the float64 oracle) and
tests/test_host_bert4rec_shapes.py (which checks, without a GPU, that the table reaches every branch of g4r_bert4rec.cuh's attention
kernels, nm_gemm's split rule at these shapes, several evaluation chunks and a batch at exactly P_max).

GRAD_CASES are one training mini-batch each: the pieces (lists of item indices, 2 .. max_len events, all inputs) as the fit holds
them, the batch (indices into the pieces, in slot order; a piece may appear twice), the cloze masks of every piece, the batch_size
the fit is begun with, dropout and a parameter scale.  EVAL_CASES are one bert4rec_encode call each.  Everything is drawn from
seeded RandomStates.  nm_gemm's split rule is NARM's (narm_cases restates it)."""
import os
import re

import numpy as np

import bert4rec_oracle as bo
import narm_cases as nc

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gru4rec_b200', 'csrc', 'g4r_bert4rec.cuh')


def constants():
    """B4_ATT_THREADS, B4_EVAL_POS, B4_LEN_MAX, B4_D_MAX, B4_BLOCKS_MAX as g4r_bert4rec.cuh defines them"""
    with open(HEADER) as f:
        src = f.read()
    return {name: int(re.search(r'\b%s\s*=\s*(\d+)' % name, src).group(1))
            for name in ('B4_ATT_THREADS', 'B4_EVAL_POS', 'B4_LEN_MAX', 'B4_D_MAX', 'B4_BLOCKS_MAX')}


def products(P, Pm, NI, d):
    """b4_grad's products after the encoder: name -> (role, M, N, K)"""
    return {'S': ('catalogue', Pm, NI, d), 'dQ': ('catalogue', Pm, d, NI), 'dE': ('catalogue', NI, d, Pm), 'dbO': ('backward', 1, NI, Pm),
            'dW': ('backward', d, d, P), 'dW1': ('backward', d, 4 * d, P), 'dW2': ('backward', 4 * d, d, P), 'db': ('backward', 1, d, P),
            'dX': ('backward', P, d, d), 'dX1': ('backward', P, d, 4 * d), 'dX2': ('backward', P, 4 * d, d)}


def eval_plan(offsets, n_history, max_len):
    """b4_encode_events' plan: per counted event a window of min(p, max_len - 1) inputs and the mask, in chunks of at most
    B4_EVAL_POS positions.  Returns (chunks: per chunk its (session, last input index, window length), where: per counted event
    (chunk, slot))"""
    cap = constants()['B4_EVAL_POS']
    chunks, where, cur, P = [], [], [], 0
    for s in range(len(offsets) - 1):
        n = int(offsets[s + 1] - offsets[s])
        i0 = max(int(n_history[s]) if n_history is not None else 0, 1) - 1
        for i in range(i0, n - 1):
            w = min(i + 1, max_len - 1) + 1
            if P + w > cap:
                chunks.append(cur)
                cur, P = [], 0
            where.append((len(chunks), len(cur)))
            cur.append((s, i, w))
            P += w
    if cur:
        chunks.append(cur)
    return chunks, where


def _shipped(rs, NI, max_len=50, n=256, n_full=4):
    """n pieces cut from RSC15-like sessions of Zipf items, n_full of them full (max_len events), in a shuffled order"""
    lens = nc.rsc15_lengths(rs, 8 * n)
    items = rs.zipf(1.2, size=int(lens.sum())) % NI
    sessions = np.split(items, np.cumsum(lens)[:-1])
    pieces = [p for p in bo.pieces(sessions, max_len) if len(p) < max_len][:n - n_full]
    pieces += [list(rs.zipf(1.2, size=max_len) % NI) for _ in range(n_full)]
    return [pieces[k] for k in rs.permutation(len(pieces))]


def _lens(rs, NI, lens):
    return [list(rs.randint(0, NI, k)) for k in lens]


def _uniform(rs, n, NI, max_len):
    """one 2-event piece, one max_len piece, the rest uniform"""
    return _lens(rs, NI, np.r_[2, max_len, rs.randint(2, max_len + 1, n - 2)])


def _tile(rs, NI, lens):
    """a batch of exactly sum(lens) positions whose first piece is repeated in slot 1; the fit also holds an unused piece as long
    as the first, so that the batch_size longest distinct pieces cover the batch"""
    pieces = _lens(rs, NI, [lens[0]] + list(lens[1:]) + [lens[0]])
    return pieces, [0, 0] + list(range(1, len(lens)))


def _pmax(rs, NI, lens):
    """a batch of the batch_size longest distinct pieces: P = P_max"""
    pieces = _lens(rs, NI, list(lens) + [2, 3])
    return pieces, list(range(len(lens)))


def _case(id, NI, d, heads, blocks, max_len, drop, mask_prob, build, seed, scale=1.0):
    """build(rs) -> pieces or (pieces, batch); the masks, then the parameters, are drawn after the pieces from the same RandomState"""
    return dict(id=id, NI=NI, d=d, heads=heads, blocks=blocks, max_len=max_len, drop=drop, mask_prob=mask_prob, build=build, seed=seed,
                scale=scale)


def grad_batch(case):
    """(pieces, batch, masks (per piece), batch_size, rs): rs positioned for the parameters' draw"""
    rs = np.random.RandomState(case['seed'])
    out = case['build'](rs)
    pieces, batch = out if isinstance(out, tuple) else (out, list(range(len(out))))
    masks = bo.cloze([len(p) for p in pieces], case['mask_prob'], rs)
    return pieces, np.asarray(batch), masks, len(batch), rs


GRAD_CASES = [
    # the shipped shape: scripts/bert4rec_bench.py's training step
    _case('shipped', 37483, 64, 2, 2, 50, 0.1, 0.2, lambda rs: _shipped(rs, 37483), 1),
    _case('shipped-nodrop', 37483, 64, 2, 2, 50, 0.0, 0.2, lambda rs: _shipped(rs, 37483), 2),
    _case('heads-4-d-64', 2000, 64, 4, 2, 20, 0.1, 0.2, lambda rs: _uniform(rs, 32, 2000, 20), 3),
    # trained-model scale: E and Pe x 10, gp x 4, the other matrices x 2, random gains and biases (the test asserts a logit spread >= 30)
    _case('trained-scale', 5000, 64, 2, 2, 20, 0.1, 0.2, lambda rs: _uniform(rs, 40, 5000, 20), 4, scale=10.0),
    _case('catalogue-172000', 172000, 64, 2, 2, 50, 0.0, 0.2, lambda rs: _lens(rs, 172000, np.r_[2, 50, rs.randint(2, 12, 10)]), 5),
    # a 512-event piece: more keys and queries than an attention CTA has threads
    _case('length-512', 3000, 32, 2, 1, 512, 0.1, 0.2, lambda rs: _lens(rs, 3000, [512, 300, 129, 2]), 6),
    # one head of 1024 columns: wider than an attention CTA
    _case('d-1024', 1000, 1024, 1, 1, 8, 0.0, 0.2, lambda rs: _uniform(rs, 5, 1000, 8), 7),
    _case('blocks-8', 1000, 16, 2, 8, 10, 0.1, 0.2, lambda rs: _uniform(rs, 16, 1000, 10), 8),
    _case('mask-0.9', 1500, 32, 2, 2, 16, 0.1, 0.9, lambda rs: _uniform(rs, 20, 1500, 16), 9),
    # so rare that every piece has only its forced last entry masked
    _case('mask-0.01', 1500, 32, 2, 2, 16, 0.1, 0.01, lambda rs: _uniform(rs, 20, 1500, 16), 14),
    _case('tile-64', 128, 12, 3, 2, 24, 0.0, 0.3, lambda rs: _tile(rs, 128, [3, 11, 13, 17, 17]), 11),
    _case('tile-65', 129, 65, 5, 1, 24, 0.1, 0.3, lambda rs: _tile(rs, 129, [3, 11, 13, 17, 16, 2]), 12),
    _case('p-max', 700, 24, 2, 2, 30, 0.1, 0.2, lambda rs: _pmax(rs, 700, [30, 25, 9, 30, 4]), 13),
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
    dict(id='shipped', NI=37483, d=64, heads=2, blocks=2, max_len=50, seed=31, lengths=lambda rs: _rsc15_with_long(rs, 6000, 8, 120)),
    # long windows and several heads: sessions past max_len = 512
    dict(id='heads-4-len-512', NI=3000, d=32, heads=4, blocks=2, max_len=512, seed=32, lengths=lambda rs: np.r_[560, 2, 1, rs.randint(2, 40, 30), 530]),
]
