"""Without a GPU: the SR-GNN case table (tests/srgnn_cases.py) reaches every branch of g4r_srgnn.cuh's kernels, with the constants
read from the header: samples of more inputs than a graph CTA's threads and of max_len 512, widths past a readout CTA's threads
(d 1024) and below a warp (d 1), one, three and eight propagation steps, repeated items, self-loops, single-node graphs and
nodes without in- or out-edges, a sample repeated in a batch, 172,000 items, a trained model's scale, and evaluation across
several chunks with windows of the last max_len inputs."""
import numpy as np

import srgnn_cases as sc
import srgnn_oracle as so


def _batches():
    out = []
    for case in sc.GRAD_CASES:
        sessions, order, bs, _ = sc.grad_batch(case)
        smp = so.samples(sessions, case['max_len'])
        batch = [smp[k] for k in order]
        assert len(batch) == bs and all(1 <= len(x) <= case['max_len'] for x, _ in batch), case['id']
        out.append((case, order, batch))
    return out


def test_the_constants_are_what_the_table_is_built_around():
    c = sc.constants()
    assert c['SG_THREADS'] == 256 and c['SG_LEN_MAX'] == 512 and c['SG_D_MAX'] == 1024 and c['SG_STEP_MAX'] == 8
    assert c['SG_EVAL_POS'] >= c['SG_LEN_MAX']                    # a chunk holds a whole window


def test_the_table_reaches_every_kernel_branch():
    T = sc.constants()['SG_THREADS']
    b = _batches()
    lens = [max(len(x) for x, _ in batch) for _, _, batch in b]
    assert any(n > T for n in lens) and any(n == 512 for n in lens)            # graph CTA: positions and edges loop per thread
    assert any(c['d'] > T and c['d'] == 1024 for c, _, _ in b)                 # readout CTAs: units loop per thread
    assert any(c['d'] == 1 for c, _, _ in b) and any(32 < c['d'] <= T for c, _, _ in b)   # warp reductions: idle lanes, lanes loop
    assert {1, 3, 8} <= {c['step'] for c, _, _ in b}
    assert any(c['NI'] == 172000 for c, _, _ in b) and any(c['scale'] != 1.0 for c, _, _ in b)
    assert any(len(set(o.tolist())) < len(o) for _, o, _ in b)                 # a sample repeated in a batch
    for case, _, batch in b:
        graphs = [so.graph(x) for x, _ in batch]
        assert any(len(g[0]) < len(x) for g, (x, _) in zip(graphs, batch)), case['id']            # repeated items merge
        assert any(np.diag(g[3]).any() for g in graphs), case['id']                               # a self-loop
        assert any(len(g[0]) == 1 for g in graphs), case['id']                                    # a single node
        assert any(not g[2][i].any() for g in graphs for i in range(len(g[0])) if len(g[0]) > 1), case['id']   # no in-edge
        assert any(len(x) == case['max_len'] for x, _ in batch), case['id']                       # a full-length prefix


def test_the_evaluation_cases_cross_chunks_and_windows():
    cap = sc.constants()['SG_EVAL_POS']
    for case in sc.EVAL_CASES:
        items, off, nh = sc.eval_sessions(case)
        chunk = sc.eval_chunks(off, nh, case['max_len'], cap)
        assert chunk.max() >= 1, case['id']
        assert (np.diff(off) > case['max_len'] + 1).any() and nh.max() >= 2, case['id']
        assert len(chunk) == len(sc.eval_positions(off, nh, case['max_len']))
