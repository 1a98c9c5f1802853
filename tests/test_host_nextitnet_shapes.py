"""Without a GPU: the NextItNet case table (tests/nextitnet_cases.py) reaches every branch of g4r_nextitnet.cuh's gather and
gather-sum (a tap inside the piece and one before its start, a gather-sum term inside and one past its end, the one-tap kernel,
pieces whose every shifted tap lies before their start), the model's limits (kernel_size 1 and 5, d = 1 at max_len 1, 16 blocks,
a full piece at max_len 512, d 1024, 172,000 items), nm_gemm's split rule at these shapes (backward products split, dL/dq split 64
ways, encoder products whole), P = P_max with a piece repeated in a batch, and evaluation across several chunks."""
import numpy as np

import narm_cases as nc
import nextitnet_cases as nic


def _batches():
    out = []
    for case in nic.GRAD_CASES:
        pieces, batch, bs, _ = nic.grad_batch(case)
        inputs = [len(pieces[k]) - 1 for k in batch]
        assert all(1 <= n <= case['max_len'] for n in inputs), case['id']
        out.append((case, pieces, batch, inputs))
    return out


def _taps(case, inputs):
    """per convolution of the case (dilations l, 2 l) the numbers of (inside, before the start) taps over the batch's positions;
    the gather-sum's (inside, past the end) terms are the same counts"""
    out = []
    for l in case['dil']:
        for dl in (l, 2 * l):
            inside = before = 0
            for n in inputs:
                for k in range(case['K']):
                    back = (case['K'] - 1 - k) * dl
                    inside += max(0, n - back)
                    before += min(n, back)
            out.append((inside, before))
    return out


def test_the_constants_are_what_the_table_is_built_around():
    c = nic.constants()
    assert c['NI_D_MAX'] == 1024 and c['NI_K_MAX'] == 8 and c['NI_BLOCKS_MAX'] == 16 and c['NI_DIL_MAX'] == 256 and c['NI_LEN_MAX'] == 512
    assert c['NI_EVAL_PAIRS'] >= c['NI_LEN_MAX']                  # a chunk holds a whole window


def test_the_table_reaches_every_gather_branch():
    b = _batches()
    taps = {c['id']: _taps(c, inp) for c, _, _, inp in b}
    assert all(i > 0 for t in taps.values() for i, _ in t)
    assert any(bf > 0 for t in taps.values() for _, bf in t)
    # the one-tap kernel: no tap is ever shifted, nothing lies before the start
    assert all(bf == 0 for _, bf in taps['kernel-1'])
    # every shifted tap of the first block lies before the start of every piece: only the last tap reads inside
    case, _, _, inp = next(x for x in b if x[0]['id'] == 'taps-before-start')
    assert case['dil'][0] * (case['K'] - 1) >= max(inp) and taps['taps-before-start'][0][0] == sum(inp)
    assert any(c['K'] == 1 for c, _, _, _ in b) and any(c['K'] == 5 for c, _, _, _ in b)
    assert any(c['d'] == 1 and c['max_len'] == 1 for c, _, _, _ in b)
    assert any(len(c['dil']) == nic.constants()['NI_BLOCKS_MAX'] for c, _, _, _ in b)
    assert any(c['max_len'] == 512 and 512 in inp for c, _, _, inp in b)
    assert any(c['d'] == 1024 for c, _, _, _ in b) and any(c['NI'] == 172000 for c, _, _, _ in b)
    assert any(c['scale'] != 1.0 for c, _, _, _ in b)


def test_the_split_rule_at_these_shapes():
    got = {}
    for case, _, _, inputs in _batches():
        P = sum(inputs)
        for name, (role, M, N, K) in nic.products(P, case['NI'], case['d'], case['K']).items():
            got.setdefault(name, set()).add(nc.splits(role, M, N, K))
        # the encoder's products never split k, so an event's q does not depend on its chunk
        assert nc.splits('encoder', P, case['d'], case['K'] * case['d']) == 1
    shipped = next(x for x in _batches() if x[0]['id'] == 'shipped')
    P = sum(shipped[3])
    assert nc.splits('backward', 3 * 100, 100, P) >= 2                       # kernel gradients over the positions split
    assert nc.splits('catalogue', P, 100, 37483) == 64                       # dL/dq over the catalogue: 64 partials
    assert max(got['dC']) >= 2 and min(got['dC']) == 1 and max(got['dQ']) == 64 and got['conv'] == {1}


def test_p_max_with_a_repeated_piece():
    case, pieces, batch, inputs = next(x for x in _batches() if x[0]['id'] == 'pmax')
    assert len(set(batch.tolist())) < len(batch)
    longest = sorted((len(p) - 1 for p in pieces), reverse=True)[:len(batch)]
    assert sum(inputs) == sum(longest)                           # exactly the scratch the fit sizes (P_max)


def test_evaluation_spans_several_chunks_with_windows():
    for case in nic.EVAL_CASES:
        items, off, nh = nic.eval_sessions(case)
        chunks, where = nic.eval_plan(off, nh, case['max_len'])
        assert len(chunks) >= 2, case['id']
        assert np.diff(off).max() > case['max_len'] + 1          # windows of the last max_len inputs
        assert len(where) == int(np.maximum(0, np.diff(off) - np.maximum(nh, 1)).sum())
