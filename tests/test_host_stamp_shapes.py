"""Without a GPU: the STAMP case table (tests/stamp_cases.py) reaches every branch of g4r_stamp.cuh's kernels, with the constants
read from the header: samples of more positions than an attention CTA has warps and of max_len 512, widths past a CTA's threads
(d 1024), below a warp (d 1) and not a multiple of 32, one input (m_s = m_t = x_1), prefixes cut to their last max_len inputs,
repeated items, a target that is also an input, a sample repeated in a batch, a batch of one, 172,000 items, a trained model's
scale, and evaluation across several chunks with windows of the last max_len inputs."""
import numpy as np

import stamp_cases as stc
import stamp_oracle as sto


def _batches():
    out = []
    for case in stc.GRAD_CASES:
        sessions, order, bs, _ = stc.grad_batch(case)
        smp = sto.samples(sessions, case['max_len'])
        batch = [smp[k] for k in order]
        assert len(batch) == bs and all(1 <= len(x) <= case['max_len'] for x, _ in batch), case['id']
        out.append((case, sessions, order, batch))
    return out


def test_the_constants_are_what_the_table_is_built_around():
    c = stc.constants()
    assert c['ST_THREADS'] == 256 and c['ST_LEN_MAX'] == 512 and c['ST_D_MAX'] == 1024
    assert c['ST_EVAL_POS'] >= c['ST_LEN_MAX']                    # a chunk holds a whole window


def test_the_table_reaches_every_kernel_branch():
    T = stc.constants()['ST_THREADS']
    b = _batches()
    lens = [max(len(x) for x, _ in batch) for _, _, _, batch in b]
    assert any(n > T // 32 for n in lens) and any(n == 512 for n in lens)               # attention CTAs: positions loop per warp
    assert any(n * c['d'] > T for n, (c, _, _, _) in zip(lens, b))                      # gather / dx CTAs: elements loop per thread
    assert any(c['d'] > T and c['d'] == 1024 for c, _, _, _ in b)                       # units loop per thread
    assert any(c['d'] == 1 for c, _, _, _ in b) and any(c['d'] % 32 and c['d'] > 32 for c, _, _, _ in b)   # idle lanes, lanes loop
    assert any(c['NI'] == 172000 for c, _, _, _ in b) and any(c['scale'] != 1.0 for c, _, _, _ in b)
    assert any(len(set(o.tolist())) < len(o) for _, _, o, _ in b)                       # a sample repeated in a batch
    assert any(c['bs'] == 1 for c, _, _, _ in b)                                         # a batch of one
    for case, sessions, _, batch in b:
        if case['bs'] == 1:
            assert len(batch[0][0]) == case['max_len'], case['id']                          # the longest sample
            continue
        L = case['max_len']
        assert any(len(x) == 1 for x, _ in batch), case['id']                            # n = 1: m_s = m_t = x_1
        assert any(len(set(x)) < len(x) for x, _ in batch), case['id']                   # repeated items scatter into one row
        assert any(y in x for x, y in batch), case['id']                                 # a target that is also an input
        assert any(len(x) == L for x, _ in batch), case['id']                            # a full-length prefix
        cut = [(x, y) for x, y in sto.samples(sessions, L) if len(x) == L]
        assert any(s[:L + 1] != s[-(L + 1):] for s in sessions if len(s) > L + 1), case['id']   # prefixes cut to their last max_len
        assert cut, case['id']


def test_the_evaluation_cases_cross_chunks_and_windows():
    cap = stc.constants()['ST_EVAL_POS']
    for case in stc.EVAL_CASES:
        items, off, nh = stc.eval_sessions(case)
        chunk = stc.eval_chunks(off, nh, case['max_len'], cap)
        assert chunk.max() >= 1, case['id']
        assert (np.diff(off) > case['max_len'] + 1).any() and nh.max() >= 2, case['id']
        assert len(chunk) == int(np.maximum(0, np.diff(off) - np.maximum(nh, 1)).sum())
