"""Without a GPU: the BERT4Rec case table (tests/bert4rec_cases.py) reaches every branch of g4r_bert4rec.cuh's attention kernels
(pieces of at most and of more positions than an attention CTA's threads, one head and several, a head wider than the CTA), the
model's limits (n_blocks 8, max_len 512, d 1024, 172,000 items), the cloze masks' extremes (mask_prob 0.9, and 0.01 with only the
forced last entries masked), nm_gemm's split rule at these shapes (backward products split, dL/dq split 64 ways, encoder products
whole), P at the tile edges with a piece repeated in a batch, a batch at exactly P_max, and evaluation across several chunks."""
import numpy as np

import bert4rec_cases as bc
import narm_cases as nc


def _batches():
    out = []
    for case in bc.GRAD_CASES:
        pieces, batch, masks, bs, _ = bc.grad_batch(case)
        lens = [len(pieces[k]) for k in batch]
        assert all(2 <= n <= case['max_len'] for n in lens), case['id']
        assert all(any(m) and len(m) == len(p) for m, p in zip(masks, pieces)), case['id']
        out.append((case, pieces, batch, masks, lens))
    return out


def test_the_constants_are_what_the_table_is_built_around():
    c = bc.constants()
    assert c['B4_ATT_THREADS'] == 128 and c['B4_LEN_MAX'] == 512 and c['B4_D_MAX'] == 1024 and c['B4_BLOCKS_MAX'] == 8
    assert c['B4_EVAL_POS'] >= c['B4_LEN_MAX']                    # a chunk holds a whole window


def test_the_table_reaches_every_attention_branch():
    T = bc.constants()['B4_ATT_THREADS']
    b = _batches()
    assert any(max(n) > T for _, _, _, _, n in b)                  # more keys (and queries per key) than threads
    assert any(max(n) <= T for _, _, _, _, n in b)
    assert any(c['heads'] == 1 for c, *_ in b) and any(c['heads'] >= 4 for c, *_ in b)
    assert any(c['d'] // c['heads'] > T for c, *_ in b)            # a head wider than the CTA: columns loop per thread
    assert any(c['d'] // c['heads'] == c['d'] == 1024 for c, *_ in b)
    assert any(c['blocks'] == 8 for c, *_ in b) and any(c['max_len'] == 512 and 512 in n for c, _, _, _, n in b)
    assert any(c['NI'] == 172000 for c, *_ in b) and any(c['scale'] != 1.0 for c, *_ in b)
    assert any(c['drop'] > 0 for c, *_ in b) and any(c['drop'] == 0 for c, *_ in b)


def test_the_cloze_masks_reach_both_extremes():
    b = {c['id']: (pieces, batch, masks) for c, pieces, batch, masks, _ in _batches()}
    pieces, batch, masks = b['mask-0.9']
    rate = np.mean([v for k in batch for v in masks[k]])
    assert rate > 0.8 and any(sum(masks[k]) >= 5 for k in batch)
    pieces, batch, masks = b['mask-0.01']
    assert all(masks[k][-1] and sum(masks[k]) == 1 for k in batch)      # only the forced last entries
    pieces, batch, masks = b['shipped']
    assert any(sum(masks[k]) >= 2 for k in batch) and any(not masks[k][-1] for k in batch)


def test_the_split_rule_at_these_shapes():
    got = {}
    for case, pieces, batch, masks, lens in _batches():
        P, Pm = sum(lens), sum(sum(masks[k]) for k in batch)
        for name, (role, M, N, K) in bc.products(P, Pm, case['NI'], case['d']).items():
            got.setdefault(name, set()).add(nc.splits(role, M, N, K))
        # the encoder's products never split k, so an event's q does not depend on its chunk
        assert nc.splits('encoder', P, 4 * case['d'], case['d']) == 1 and nc.splits('encoder', P, case['d'], 4 * case['d']) == 1
    shipped = next(x for x in _batches() if x[0]['id'] == 'shipped')
    P = sum(shipped[4])
    assert len(shipped[2]) == 256
    assert nc.splits('backward', 64, 64, P) >= 2                                 # weight gradients over the positions split
    Pm = sum(sum(shipped[3][k]) for k in shipped[2])
    assert nc.splits('catalogue', Pm, 64, 37483) == 64                           # dL/dq over the catalogue: 64 partials
    assert max(got['dW']) >= 2 and min(got['dW']) == 1 and max(got['dQ']) == 64


def test_tile_edges_p_max_and_a_repeated_piece():
    sizes = {c['id']: (sum(n), len(set(batch.tolist())) < len(batch)) for c, _, batch, _, n in _batches()}
    assert sizes['tile-64'] == (64, True) and sizes['tile-65'] == (65, True)
    for cid in ('tile-64', 'tile-65', 'p-max'):
        case, pieces, batch, masks, lens = next(x for x in _batches() if x[0]['id'] == cid)
        longest = sorted((len(p) for p in pieces), reverse=True)[:len(batch)]
        assert sum(lens) <= sum(longest)                         # within the scratch the fit sizes (P_max)
        if cid == 'p-max':
            assert sum(lens) == sum(longest)


def test_evaluation_spans_several_chunks_with_windows():
    for case in bc.EVAL_CASES:
        items, off, nh = bc.eval_sessions(case)
        chunks, where = bc.eval_plan(off, nh, case['max_len'])
        assert len(chunks) >= 2, case['id']
        assert np.diff(off).max() > case['max_len'], case['id']        # windows of the last max_len - 1 inputs
        assert len(where) == int(np.maximum(0, np.diff(off) - np.maximum(nh, 1)).sum())
        starts = {}
        for c, ch in enumerate(chunks):
            for s, _, _ in ch:
                starts.setdefault(s, set()).add(c)
        assert any(len(v) > 1 for v in starts.values()), case['id']    # a session's events across chunks
