"""The NARM test shapes (DESIGN §3s), shared by tests/test_gpu_narm.py (the device against the float64 oracle) and
tests/test_host_narm_shapes.py (which checks, without a GPU, that the table reaches every branch of g4r_narm.cuh).

GRAD_CASES are one training mini-batch each: the pieces (lists of item indices) as the fit holds them, the batch (indices into the
pieces, in slot order; a piece may appear twice), the batch_size the fit is begun with, dropout and a parameter scale.
EVAL_CASES are one narm_encode call each: sessions, history counts and the model's shape.  Everything is drawn from seeded
RandomStates, so both files see the same data.  Also here: the constants of g4r_narm.cuh read from the source, and nm_gemm's k
split and nm_encode_events' piece and chunk planner restated in Python."""
import os
import re

import numpy as np

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gru4rec_b200', 'csrc', 'g4r_narm.cuh')


def constants():
    """NM_BM, NM_BN, NM_BK, NM_KCHUNK, NM_SPLIT_TILES, NM_PART_CAP, NM_EVAL_PAIRS as g4r_narm.cuh defines them"""
    with open(HEADER) as f:
        src = f.read()
    out = {}
    for name in ('NM_BM', 'NM_BN', 'NM_BK', 'NM_KCHUNK', 'NM_SPLIT_TILES', 'NM_EVAL_PAIRS'):
        out[name] = int(re.search(r'\b%s\s*=\s*(\d+)' % name, src).group(1))
    m = re.search(r'\bNM_PART_CAP\s*=\s*\(size_t\)(\d+)\s*<<\s*(\d+)', src)
    out['NM_PART_CAP'] = int(m.group(1)) << int(m.group(2))
    return out


def splits(role, M, N, K, c=None):
    """nm_gemm's number of k ranges for a product of M x N outputs over K (role 'encoder', 'catalogue' or 'backward')"""
    c = c or constants()
    tiles = -(-M // c['NM_BM']) * -(-N // c['NM_BN'])
    s = 1
    if role != 'encoder' and tiles < c['NM_SPLIT_TILES']:
        s = max(1, min(64, -(-K // c['NM_KCHUNK']), c['NM_PART_CAP'] // (M * N)))
    kc = -(-K // s)
    kc = max(c['NM_BK'], -(-kc // c['NM_BK']) * c['NM_BK'])
    return max(1, -(-K // kc))


def products(P, NI, d, H):
    """nm_grad's products after the encoder: name -> (role, M, N, K)"""
    return {'S': ('catalogue', P, NI, d), 'dQ': ('catalogue', P, d, NI), 'dE': ('catalogue', NI, d, P),
            'dB': ('backward', d, 2 * H, P), 'dC': ('backward', P, 2 * H, d), 'T1': ('backward', P, H, H), 'T2': ('backward', P, H, H),
            'dA1': ('backward', H, H, P), 'dA2': ('backward', H, H, P), 'dv': ('backward', 1, H, P), 'dWh': ('backward', H, H, P),
            'dWrz': ('backward', H, 2 * H, P), 'dWx': ('backward', d, 3 * H, P), 'dBh': ('backward', 1, 3 * H, P),
            'dEMB': ('backward', P, d, 3 * H)}


def eval_plan(offsets, n_history, max_len, pairs=None):
    """nm_encode_events' plan: a list of chunks, each a list of pieces (session, first input index, inputs); and per counted
    event (evaluate's order) its (chunk, position in the chunk)"""
    pairs = pairs or constants()['NM_EVAL_PAIRS']
    chunks, cur, P, where = [], [], 0, []

    def piece(s, i, n):
        nonlocal cur, P
        if P + n > pairs or len(cur) >= pairs:
            chunks.append(cur)
            cur, P = [], 0
        cur.append((s, i, n))
        P += n
        return P - n

    for s in range(len(offsets) - 1):
        length = int(offsets[s + 1] - offsets[s])
        i0 = max(0 if n_history is None else int(n_history[s]), 1) - 1
        last = length - 2
        if last < i0:
            continue
        if i0 < max_len:
            n = min(last + 1, max_len)
            p0 = piece(s, 0, n)
            where += [(len(chunks), p0 + i) for i in range(i0, n)]
        for i in range(max(i0, max_len), last + 1):
            p0 = piece(s, i - max_len + 1, max_len)
            where.append((len(chunks), p0 + max_len - 1))
    if cur:
        chunks.append(cur)
    return chunks, where


def rsc15_lengths(rs, n_events):
    """RSC15-like session lengths (scripts/narm_bench.session_lengths): 1 + geometric (mean about 3.5 events), a tail to 200"""
    lens = np.minimum(1 + rs.geometric(0.4, size=n_events // 2), 200)
    return lens[np.cumsum(lens) <= n_events]


def cut(sessions, max_len):
    """training pieces of sessions (lists in time order): at most max_len events, consecutive pieces sharing one event"""
    out = []
    for s in sessions:
        a = 0
        while len(s) >= 2:
            b = min(a + max_len, len(s))
            out.append(list(s[a:b]))
            if b == len(s):
                break
            a = b - 1
    return out


def uniform_pieces(rs, n, NI, max_len):
    """the original draw: one 2-event piece, one max_len piece, the rest uniform in 2 .. max_len"""
    lens = np.r_[2, max_len, rs.randint(2, max_len + 1, n - 2)]
    return [list(rs.randint(0, NI, k)) for k in lens]


def _shipped(rs, NI, max_len=50, n=512, n_full=8):
    """n pieces cut from RSC15-like sessions of Zipf items, n_full of them full max_len-event pieces, in a shuffled order"""
    lens = rsc15_lengths(rs, 4 * n)
    items = rs.zipf(1.2, size=int(lens.sum())) % NI
    sessions = np.split(items, np.cumsum(lens)[:-1])
    pieces = [p for p in cut(sessions, max_len) if len(p) < max_len][:n - n_full]
    pieces += [list(rs.zipf(1.2, size=max_len) % NI) for _ in range(n_full)]
    return [pieces[k] for k in rs.permutation(len(pieces))]


def _lengths(rs, NI, lens):
    return [list(rs.randint(0, NI, k)) for k in lens]


def _tile(rs, NI, inputs):
    """a batch of exactly sum(inputs) positions whose first piece (2 inputs) is repeated in slot 1; the fit also holds an unused
    piece of 3 inputs, so that the batch_size longest distinct pieces cover the batch"""
    pieces = _lengths(rs, NI, [2 + 1] + [k + 1 for k in inputs[1:]] + [3 + 1])
    return pieces, [0, 0] + list(range(1, len(inputs)))


def _case(id, NI, d, H, max_len, drop, build, seed, scale=1.0):
    """build(rs) -> pieces or (pieces, batch); the parameters are drawn after the pieces from the same RandomState"""
    return dict(id=id, NI=NI, d=d, H=H, max_len=max_len, drop=drop, build=build, seed=seed, scale=scale)


def grad_batch(case):
    """(pieces, batch, batch_size, rs): rs positioned for the parameters' draw"""
    rs = np.random.RandomState(case['seed'])
    out = case['build'](rs)
    pieces, batch = out if isinstance(out, tuple) else (out, list(range(len(out))))
    return pieces, np.asarray(batch), len(batch), rs


GRAD_CASES = [
    # the original rows: pieces of 2 .. 12 events, batches of 33 .. 45 (ids kept)
    _case('1000-16-24-37-drop0', 1000, 16, 24, 12, (0.0, 0.0), lambda rs: uniform_pieces(rs, 37, 1000, 12), 1037),
    _case('1000-16-24-37-drop1', 1000, 16, 24, 12, (0.25, 0.5), lambda rs: uniform_pieces(rs, 37, 1000, 12), 1037),
    _case('2345-50-100-45-drop2', 2345, 50, 100, 12, (0.25, 0.5), lambda rs: uniform_pieces(rs, 45, 2345, 12), 2390),
    _case('37483-50-100-33-drop3', 37483, 50, 100, 12, (0.0, 0.0), lambda rs: uniform_pieces(rs, 33, 37483, 12), 37516),
    _case('37483-50-100-33-drop4', 37483, 50, 100, 12, (0.25, 0.5), lambda rs: uniform_pieces(rs, 33, 37483, 12), 37516),
    # the shipped shape: scripts/narm_bench.py's training step
    _case('shipped', 37483, 50, 100, 50, (0.25, 0.5), lambda rs: _shipped(rs, 37483), 11),
    # trained-model scale: init x 3 and a random Bh (the test asserts a logit spread >= 30)
    _case('shipped-trained', 37483, 50, 100, 50, (0.25, 0.5), lambda rs: _shipped(rs, 37483), 12, scale=3.0),
    _case('catalogue-172000', 172000, 50, 100, 50, (0.0, 0.0),
          lambda rs: _lengths(rs, 172000, np.r_[2, 50, rs.randint(2, 21, 22)]), 13),
    _case('hidden-300', 3000, 37, 300, 20, (0.25, 0.5), lambda rs: uniform_pieces(rs, 24, 3000, 20), 14),
    _case('hidden-1024', 2000, 24, 1024, 8, (0.0, 0.0), lambda rs: uniform_pieces(rs, 6, 2000, 8), 15),
    _case('length-512', 3000, 10, 16, 512, (0.25, 0.5), lambda rs: _lengths(rs, 3000, [512, 300, 2]), 16),
    _case('embedding-130', 700, 130, 24, 10, (0.25, 0.5), lambda rs: uniform_pieces(rs, 19, 700, 10), 17),
    _case('embedding-1024', 1024, 1024, 16, 6, (0.0, 0.0), lambda rs: uniform_pieces(rs, 15, 1024, 6), 18),
    _case('tiny', 5, 1, 1, 2, (0.0, 0.0), lambda rs: _lengths(rs, 5, [2] * 9), 19),
    _case('tile-64', 128, 12, 20, 24, (0.0, 0.0), lambda rs: _tile(rs, 128, [2, 11, 13, 17, 19]), 20),
    _case('tile-65', 129, 12, 20, 24, (0.25, 0.5), lambda rs: _tile(rs, 129, [2, 11, 13, 17, 19, 1]), 21),
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
    lens = rsc15_lengths(rs, n_events)
    at = rs.choice(len(lens), n_long, replace=False)
    lens[at] = long_len
    return lens


EVAL_CASES = [
    # the shipped shape: RSC15-like sessions, a few of 120 events (windows), history counts on about a fifth of the sessions
    dict(id='shipped', NI=37483, d=50, H=100, max_len=50, seed=31, lengths=lambda rs: _rsc15_with_long(rs, 60000, 12, 120)),
    # long windows at a wide hidden layer: sessions past max_len = 512
    dict(id='hidden-300-len-512', NI=3000, d=37, H=300, max_len=512, seed=32,
         lengths=lambda rs: np.r_[600, 2, 1, rs.randint(2, 40, 30), 530, 512, 513, 300]),
]
