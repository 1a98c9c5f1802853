"""Without a GPU: the NARM test shapes (tests/narm_cases.py) reach every branch of g4r_narm.cuh that tests/test_gpu_narm.py is
meant to exercise, under the constants the header defines today, so that a change of a constant or a case cannot quietly drop
coverage: backward products split three or more ways and dL/dq 64 ways, attention triangles past one pass of 256 threads, a
512-event piece, hidden sizes past 256 and at 1024, embeddings past one 64-wide tile and at 1024, positions and catalogues at
64k and 64k + 1, a piece repeated in a batch, a long input-embedding scatter run, and evaluation over several chunks with
sessions across a chunk boundary and window pieces."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, 'oracle'), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import narm_cases as nc  # noqa: E402
import narm_oracle as no  # noqa: E402


@pytest.fixture(scope='module')
def grad_rows():
    """per gradient case: (case, batch's pieces, P, the fit's P_max, split count per product)"""
    c = nc.constants()
    rows = []
    for case in nc.GRAD_CASES:
        pieces, order, bs, _ = nc.grad_batch(case)
        P = sum(len(pieces[k]) - 1 for k in order)
        Pmax = sum(sorted((len(p) - 1 for p in pieces), reverse=True)[:bs])
        sp = {k: nc.splits(*v, c=c) for k, v in nc.products(P, case['NI'], case['d'], case['H']).items()}
        rows.append((case, [pieces[k] for k in order], P, Pmax, sp))
    return rows


def test_the_constants_are_read_from_the_header():
    c = nc.constants()
    assert set(c) == {'NM_BM', 'NM_BN', 'NM_BK', 'NM_KCHUNK', 'NM_SPLIT_TILES', 'NM_PART_CAP', 'NM_EVAL_PAIRS'}
    assert all(v > 0 for v in c.values())


def test_the_split_rule_on_known_shapes():
    # K of 37,483 over one tile column: ranges of 592 (37,483 / 64 rounded up to 16), 64 of them; encoder products never split
    assert nc.splits('catalogue', 300, 50, 37483) == 64
    assert nc.splits('encoder', 300, 50, 37483) == 1
    assert nc.splits('backward', 50, 200, 1024) == 2 and nc.splits('backward', 50, 200, 1025) == 3
    assert nc.splits('backward', 64 * 264, 64, 5000) == 1                 # enough output tiles: no split


def test_every_case_is_admissible_and_its_float64_logits_are_bounded(grad_rows):
    for case, batch, P, Pmax, _ in grad_rows:
        assert P <= Pmax, case['id']                                      # narm_grads would refuse the batch
        assert all(2 <= len(b) <= case['max_len'] for b in batch), case['id']
        assert all(0 <= x < case['NI'] for b in batch for x in b), case['id']
        assert len(batch) * case['max_len'] * max(case['d'], 2 * case['H']) < 2 ** 32
        assert P * case['NI'] * 8 <= 0.5e9, case['id']                    # the oracle's float64 logits


def test_the_gradient_cases_reach_every_product_branch(grad_rows):
    c = nc.constants()
    back = [max(v for k, v in sp.items() if nc.products(1, 1, 1, 1)[k][0] == 'backward') for _, _, _, _, sp in grad_rows]
    assert max(back) >= 3                                                 # k_nm_gsum past its second partial
    assert any(sp['dQ'] == 64 for *_, sp in grad_rows)
    assert any(sp['dQ'] > 1 and sp['dB'] > 1 for *_, sp in grad_rows)
    Ps = {P for _, _, P, _, _ in grad_rows}
    NIs = {case['NI'] for case, *_ in grad_rows}
    for vals in (Ps, NIs):
        assert any(v % c['NM_BM'] == 0 for v in vals) and any(v % c['NM_BM'] == 1 and v > 1 for v in vals)
    ds = {case['d'] for case, *_ in grad_rows}
    assert max(ds) == 1024 and any(c['NM_BN'] < d < 1024 for d in ds)    # more than one column tile of Q, dL/dq, dEMB


def test_the_gradient_cases_reach_every_encoder_branch(grad_rows):
    Hs = {case['H'] for case, *_ in grad_rows}
    assert max(Hs) == 1024 and any(256 < H < 1024 for H in Hs)          # per-thread arrays past q = 0; q = 3
    n = [max(len(b) - 1 for b in batch) for _, batch, _, _, _ in grad_rows]
    assert max(n) ** 2 > 256                                              # the attention triangle past one pass of 256 threads
    assert any(case['max_len'] == 512 and any(len(b) == 512 for b in batch) for case, batch, *_ in grad_rows)
    assert any(case['max_len'] == 2 and case['d'] == 1 and case['H'] == 1 for case, *_ in grad_rows)
    assert any(case['scale'] != 1.0 for case, *_ in grad_rows)


def test_the_gradient_cases_repeat_a_piece_and_run_a_long_scatter(grad_rows):
    assert any(len(set(map(tuple, batch))) < len(batch) for _, batch, *_ in grad_rows)
    assert any(any(len(a) > 1 for a in _indices(nc.grad_batch(case)[1])) for case, *_ in grad_rows)
    # the input-embedding scatter: one item heads a run of >= 100 positions (sorted by (input item, position))
    runs = [np.bincount(np.concatenate([b[:-1] for b in batch])).max() for _, batch, *_ in grad_rows]
    assert max(runs) >= 100


def _indices(order):
    """the slots of each piece index in a batch"""
    out = {}
    for slot, k in enumerate(order):
        out.setdefault(int(k), []).append(slot)
    return list(out.values())


def test_the_shipped_case_is_the_benchmark_shape(grad_rows):
    case, batch, P, _, _ = next(r for r in grad_rows if r[0]['id'] == 'shipped')
    assert (case['NI'], case['d'], case['H'], case['max_len'], len(batch), case['drop']) == (37483, 50, 100, 50, 512, (0.25, 0.5))
    assert sum(len(b) == 50 for b in batch) >= 8 and P > 1024


@pytest.mark.parametrize('case', [pytest.param(c, id=c['id']) for c in nc.EVAL_CASES])
def test_the_eval_cases_reach_several_chunks(case):
    items, off, nh = nc.eval_sessions(case)
    L = case['max_len']
    chunks, where = nc.eval_plan(off, nh, L)
    pairs = nc.constants()['NM_EVAL_PAIRS']
    assert len(chunks) >= 2 and all(sum(n for _, _, n in ch) <= pairs for ch in chunks)
    seen = {}
    for c, ch in enumerate(chunks):
        for s, _, _ in ch:
            seen.setdefault(s, set()).add(c)
    assert any(len(cs) > 1 for cs in seen.values())                     # a session's pieces on both sides of a boundary
    assert any(n == L and i > 0 for ch in chunks for _, i, n in ch)       # window pieces (prefixes longer than max_len)
    assert (nh > 1).any() and len(where) == int(np.maximum(0, np.diff(off) - np.maximum(nh, 1)).sum())
    assert case['H'] * 24 * pairs * 4 < 1.5e9                             # the chunk scratch stays a small share of the card
    if case['id'] == 'shipped':
        assert (case['NI'], case['d'], case['H'], L) == (37483, 50, 100, 50)
        assert sum(n for ch in chunks for _, _, n in ch) >= 70000 and (np.diff(off) >= 120).any()
    else:
        assert L == 512 and case['H'] > 256


def test_the_planner_places_every_event_as_the_oracle_prefixes_it():
    # on a small case: each counted event's chunk position holds the last input of its prefix, within its last max_len inputs
    rs = np.random.RandomState(3)
    lens = rs.randint(1, 14, 60)
    off = np.r_[0, np.cumsum(lens)]
    nh = np.minimum(rs.randint(0, 6, 60), lens)
    items = np.arange(off[-1])
    chunks, where = nc.eval_plan(off, nh, 4, pairs=40)
    assert len(chunks) > 3
    flat = []
    for ch in chunks:
        flat.append([x for s, i, n in ch for x in items[off[s] + i:off[s] + i + n]])
    got = [flat[c][p] for c, p in where]
    want = [items[off[s] + i] for s in range(60) for i in range(max(int(nh[s]), 1) - 1, int(lens[s]) - 1)]
    assert got == want
    p = no.unpack(no.init(5, 2, 3, rs), 5, 2, 3)
    assert no.encode(p, [1, 2, 3, 4, 0], 4).shape == (2,)
