"""Without a GPU: the SASRec case table (tests/sasrec_cases.py) reaches every branch of g4r_sasrec.cuh's attention kernels (pieces
of at most and of more keys than an attention CTA's threads, one head and several, a head wider than the CTA), the model's limits
(d = 1 at max_len 1, n_blocks 8, max_len 512, d 1024), nm_gemm's split rule at these shapes (backward products split, dL/dq split
64 ways, encoder products whole), P at the tile edges with a piece repeated in a batch, and evaluation across several chunks."""
import numpy as np

import narm_cases as nc
import sasrec_cases as sc


def _batches():
    out = []
    for case in sc.GRAD_CASES:
        pieces, batch, bs, _ = sc.grad_batch(case)
        inputs = [len(pieces[k]) - 1 for k in batch]
        assert all(1 <= n <= case['max_len'] for n in inputs), case['id']
        out.append((case, pieces, batch, inputs))
    return out


def test_the_constants_are_what_the_table_is_built_around():
    c = sc.constants()
    assert c['SA_ATT_THREADS'] == 128 and c['SA_LEN_MAX'] == 512 and c['SA_D_MAX'] == 1024 and c['SA_BLOCKS_MAX'] == 8
    assert c['SA_EVAL_PAIRS'] >= c['SA_LEN_MAX']                  # a chunk holds a whole window


def test_the_table_reaches_every_attention_branch():
    T = sc.constants()['SA_ATT_THREADS']
    b = _batches()
    assert any(max(inp) > T for _, _, _, inp in b)               # more keys (and queries after a key) than threads
    assert any(max(inp) <= T for _, _, _, inp in b)
    assert any(c['heads'] == 1 for c, _, _, _ in b) and any(c['heads'] >= 4 for c, _, _, _ in b)
    assert any(c['d'] // c['heads'] > T for c, _, _, _ in b)      # a head wider than the CTA: columns loop per thread
    assert any(c['d'] // c['heads'] == c['d'] == 1024 for c, _, _, _ in b)
    assert any(c['d'] == 1 and c['max_len'] == 1 for c, _, _, _ in b)
    assert any(c['blocks'] == 8 for c, _, _, _ in b) and any(c['max_len'] == 512 and 512 in inp for c, _, _, inp in b)
    assert any(c['NI'] == 172000 for c, _, _, _ in b) and any(c['scale'] != 1.0 for c, _, _, _ in b)
    assert any(c['drop'] > 0 for c, _, _, _ in b) and any(c['drop'] == 0 for c, _, _, _ in b)


def test_the_split_rule_at_these_shapes():
    got = {}
    for case, _, _, inputs in _batches():
        P = sum(inputs)
        for name, (role, M, N, K) in sc.products(P, case['NI'], case['d']).items():
            got.setdefault(name, set()).add(nc.splits(role, M, N, K))
        # the encoder's products never split k, so an event's q does not depend on its chunk
        assert nc.splits('encoder', P, case['d'], case['d']) == 1
    shipped = next(x for x in _batches() if x[0]['id'] == 'shipped')
    P = sum(shipped[3])
    assert nc.splits('backward', shipped[0]['d'], shipped[0]['d'], P) >= 2    # weight gradients over the positions split
    assert nc.splits('catalogue', P, 50, 37483) == 64                         # dL/dq over the catalogue: 64 partials
    assert max(got['dW']) >= 2 and min(got['dW']) == 1 and max(got['dQ']) == 64


def test_tile_edges_and_a_repeated_piece():
    sizes = {c['id']: (sum(inp), len(set(batch.tolist())) < len(batch)) for c, _, batch, inp in _batches()}
    assert sizes['tile-64'] == (64, True) and sizes['tile-65'] == (65, True)
    for cid in ('tile-64', 'tile-65'):
        case, pieces, batch, inputs = next(x for x in _batches() if x[0]['id'] == cid)
        longest = sorted((len(p) - 1 for p in pieces), reverse=True)[:len(batch)]
        assert sum(inputs) <= sum(longest)                       # within the scratch the fit sizes (P_max)


def test_evaluation_spans_several_chunks_with_windows():
    for case in sc.EVAL_CASES:
        items, off, nh = sc.eval_sessions(case)
        chunks, where = sc.eval_plan(off, nh, case['max_len'])
        assert len(chunks) >= 2, case['id']
        assert np.diff(off).max() > case['max_len'] + 1          # windows of the last max_len inputs
        assert len(where) == int(np.maximum(0, np.diff(off) - np.maximum(nh, 1)).sum())
