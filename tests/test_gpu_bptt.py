"""-m gpu: truncated backpropagation through time (bptt > 1, DESIGN §3l).

(a) every window is counted; (b) at learning_rate 0 the per-step costs and the final hidden state of an epoch equal a bptt = 1,
step_mode 0 run bit for bit, with sample-store refills inside windows and the shrinking tail; (c) windows against the float64
oracle's train_window (tests/bptt_oracle.py), started from the device's state before the window; (d) two runs are bitwise equal; (e) one call equals the
same range split at window multiples, and a misaligned range is refused without a change; (f) fit_resumable interrupted and
resumed equals the uninterrupted run, fit_more runs; (g) run.py; (h) a task that needs the gradient through time."""
import contextlib
import io
import os
import re
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import gru4rec_oracle as orc
import bptt_oracle as bo
from gru4rec_b200 import _lib
from gru4rec_b200.gru4rec import GRU4Rec
from gru4rec_b200.synth import make_sessions
from gpu_utils import make_cfg, push_weights, random_opt_state, oracle_f64, param_names, oracle_param, f64_errors, F64_REL, F64_RTOL

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mk(L, B, loss, fact, S=2048, **kw):
    mk = dict(layers=[L] if isinstance(L, int) else list(L), batch_size=B, n_sample=S, loss=loss, final_act=fact, adapt='adagrad',
              learning_rate=0.05, momentum=0.0, sample_alpha=0.75)
    mk.update(kw)
    return mk


def _sessions(n_items, B, seed, kind='mixed', pool=None, n_sess=None):
    """session CSR: 'mixed' lengths 2..11 with some sessions of one repeated item and some drawn from `pool` (targets among the
    samples); 'len2' every session has length 2 (every step resets every lane); 'repeat' every session repeats one item"""
    rs = np.random.RandomState(seed)
    n_sess = n_sess or 5 * B + 3            # the last round of sessions leaves the epoch's tail with M < B
    lens = np.full(n_sess, 2) if kind == 'len2' else rs.randint(2, 12, n_sess)
    sess = []
    for k, n in enumerate(lens):
        if kind == 'repeat' or (kind == 'mixed' and k % 5 == 0):
            sess.append(np.full(n, rs.randint(n_items)))
        elif kind == 'mixed' and k % 5 == 1 and pool is not None:
            sess.append(pool[rs.randint(0, len(pool), n)])
        else:
            sess.append(rs.randint(0, n_items, n))
    items = np.concatenate(sess).astype(np.int64)
    offset = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return items, offset, np.arange(n_sess, dtype=np.int64)


def _engine(mk, n_items, T, store_rows, seed, **cfgkw):
    """engine with random weights, hidden state, biases, logQ support, optimizer state and a fixed sample store whose rows share a
    small pool of items (duplicates within and across steps)"""
    rs = np.random.RandomState(seed)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    for h in m.H:
        h[:] = rs.randn(*h.shape).astype(np.float32) * 0.5
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    for b in m.Bh:
        b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    S = mk['n_sample']
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=store_rows * S, bptt=T, **cfgkw))
    push_weights(eng, m)
    pool = rs.choice(n_items, max(1, S // 16), replace=False)
    store = rs.randint(0, n_items, size=(store_rows, S)).astype(np.int64)
    store[:, :S // 4] = pool[rs.randint(0, len(pool), size=(store_rows, S // 4))]
    eng.set_sample_store(store)
    P0 = None
    if mk.get('logq', 0):
        P0 = rs.randint(1, 50, size=n_items).astype(np.float32)
        eng.set_logq_support(P0)
    if mk.get('adapt') is not None:
        random_opt_state(eng, m, np.random.RandomState(seed + 1))
    return eng, store, P0, pool


def _assert_state(eng, m, costs, ref_costs, tag):
    bad = []
    checks = [('cost', costs, ref_costs)] + [(n, eng.get(n), oracle_param(m, n)) for n in param_names(m)]
    checks += [('%s.%s' % k, eng.get('%s.%s' % k), v) for k, v in m.opt.items()]
    checks += [('H%d' % i, eng.get('H%d' % i), m.H[i]) for i in range(len(m.layers))]
    for name, dev, ref in checks:
        a, r = f64_errors(dev, ref)
        if not (a <= F64_REL and r <= F64_RTOL):
            bad.append('%s: %.3g / %.3g' % (name, a, r))
    assert not bad, '%s: %s' % (tag, '; '.join(bad))


# name -> (model keywords, n_items, T, session kind)
CASES = {
    'none_L100_B32_bprmax': (_mk(100, 32, 'bpr-max', 'elu-0.5', bpreg=1.95), 3000, 8, 'mixed'),
    'rsc15_shared_xe_logq': (_mk(100, 32, 'cross-entropy', 'softmax', constrained_embedding=True, logq=1.0, dropout_p_hidden=0.2, momentum=0.3), 3000, 4, 'mixed'),
    'embed64_96_100_drop_top1max': (_mk([96, 100], 32, 'top1-max', 'linear', embedding=64, dropout_p_hidden=0.2, dropout_p_embed=0.3), 3000, 5, 'mixed'),
    'three_layers_relu': (_mk([40, 40, 40], 24, 'bpr-max', 'elu-0.5', hidden_act='relu', S=256), 1000, 16, 'mixed'),
    'rees46_shared_L512_B240': (_mk(512, 240, 'bpr-max', 'elu-0.5', constrained_embedding=True), 4000, 16, 'mixed'),
    'adam': (_mk(48, 16, 'bpr-max', 'linear', S=128, adapt='adam', adapt_params=[0.9, 0.999], embedding=32), 500, 3, 'mixed'),
    'rmsprop_mom_l2': (_mk(48, 16, 'top1', 'tanh', S=128, adapt='rmsprop', adapt_params=[0.9], momentum=0.3, lmbd=1e-3), 500, 3, 'mixed'),
    'adadelta': (_mk(48, 16, 'bpr', 'linear', S=128, adapt='adadelta', adapt_params=[0.95], learning_rate=1.0), 500, 3, 'mixed'),
    'grad_cap_below': (_mk(48, 16, 'bpr-max', 'linear', S=128, grad_cap=1e-3), 500, 3, 'mixed'),
    'grad_cap_above': (_mk(48, 16, 'bpr-max', 'linear', S=128, grad_cap=1e3), 500, 3, 'mixed'),
    'xe_smoothing': (_mk(48, 16, 'cross-entropy', 'softmax', S=128, smoothing=0.2, embedding=24), 500, 3, 'mixed'),
    'sessions_of_two': (_mk(48, 16, 'bpr-max', 'linear', S=128), 500, 4, 'len2'),
    'repeated_item_shared': (_mk(48, 16, 'bpr-max', 'linear', S=128, constrained_embedding=True, momentum=0.2), 500, 4, 'repeat'),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_windows_match_float64(name):
    """(c) the first two windows of the epoch and the two that end it (the last one short where the step count allows, in the
    compacted tail), each against the float64 oracle started from the device's state before it"""
    mk, n_items, T, kind = CASES[name]
    B, S = mk['batch_size'], mk['n_sample']
    rows = 256
    eng, store, P0, pool = _engine(mk, n_items, T, rows, seed=7)
    items, offset, order = _sessions(n_items, B, 11, kind, pool=pool)
    sched = _lib.Schedule(items, offset, order, B, S, mode=0)
    steps = orc.build_train_schedule(items, offset, order, B, S)
    n = len(steps)
    assert n == sched.n_steps and n <= rows
    n_win = (n + T - 1) // T
    check = sorted({0, 1, n_win - 2, n_win - 1})
    assert steps[-1]['M'] < B
    w0 = eng.bptt_windows()
    for k in range(n_win):
        first, Tw = k * T, min(T, n - k * T)
        if k not in check:
            eng.train_steps(sched, first, Tw)
            continue
        m = oracle_f64(eng, mk, n_items, first, P0)
        win = [dict(X=st['X'], Y=st['Y'], R=st['R'], slots=st['slots'], samples=store[first + t] if S else None)
               for t, st in enumerate(steps[first:first + Tw])]
        costs = eng.train_steps(sched, first, Tw)
        ref = bo.train_window(m, win)
        _assert_state(eng, m, costs, ref, '%s window %d (steps %d..%d)' % (name, k, first, first + Tw - 1))
    assert eng.bptt_windows() - w0 == n_win       # (a)


def test_lr0_costs_equal_one_step_updates():
    """(b) learning_rate 0 without an adaptive scaler: no parameter moves, so a window path that aligns sample rows, dropout masks,
    slots and resets with the schedule reproduces the one-step path's costs and hidden state bit for bit -- through sample-store
    refills inside windows (7 rows, windows of 4) and the compacted tail"""
    mk = _mk(64, 32, 'bpr-max', 'elu-0.5', S=256, adapt=None, learning_rate=0.0, dropout_p_hidden=0.3, embedding=32, dropout_p_embed=0.2)
    n_items = 800
    items, offset, order = _sessions(n_items, 32, 3)
    rs = np.random.RandomState(5)
    P = np.cumsum(rs.rand(n_items)).astype(np.float32)
    P /= P[-1]
    out = []
    for T, step_mode in ((1, 0), (4, 0), (4, 2)):
        m = orc.OracleGRU4Rec(**mk)
        m.init(n_items)
        eng = _lib.Engine(make_cfg(n_items, mk, sample_store=7 * 256, bptt=T, step_mode=step_mode))
        push_weights(eng, m)
        eng.set_sampling_cdf(P)
        eng.generate_samples()
        sched = _lib.Schedule(items, offset, order, 32, 256, mode=0)
        costs = eng.train_steps(sched, 0, sched.n_steps)
        out.append((costs, [eng.get('H%d' % i) for i in range(len(mk['layers']))], eng.bptt_windows(), sched.n_steps))
    (c1, h1, w1, n), (c4, h4, w4, _), (c4b, h4b, _, _) = out
    assert n % 4 != 0 and w1 == 0 and w4 == (n + 3) // 4
    np.testing.assert_array_equal(c1, c4)
    np.testing.assert_array_equal(c4, c4b)           # step_mode has no effect with bptt > 1
    for a, b in zip(h1, h4):
        np.testing.assert_array_equal(a, b)


def _run_engine(T, split):
    mk = CASES['rsc15_shared_xe_logq'][0]
    eng, store, P0, pool = _engine(mk, 3000, T, 256, seed=3)
    items, offset, order = _sessions(3000, 32, 4, pool=pool)
    sched = _lib.Schedule(items, offset, order, 32, 2048, mode=0)
    n = sched.n_steps
    costs = []
    for a, b in zip([0] + split, split + [n]):
        costs.append(eng.train_steps(sched, a, b - a))
    names = ['Wx0', 'Wh0', 'Wrz0', 'Bh0', 'Wy', 'By', 'Wy.acc', 'Wy.vel', 'H0']
    return np.concatenate(costs), {k: eng.get(k) for k in names}, eng, sched


def test_runs_are_deterministic_and_splits_equal():
    """(d) two runs are bitwise equal; (e) one call equals the range split at window multiples; a misaligned call is refused
    and leaves the state as it was"""
    c1, s1, _, _ = _run_engine(4, [])
    c2, s2, eng, sched = _run_engine(4, [])
    c3, s3, _, _ = _run_engine(4, [8, 12, 24])
    for c, s in ((c2, s2), (c3, s3)):
        np.testing.assert_array_equal(c1, c)
        for k in s1:
            np.testing.assert_array_equal(s1[k], s[k], err_msg=k)
    before = {k: eng.get(k) for k in s1}
    ptr = eng.get_sample_pointer()
    for first, n in ((2, 4), (4, 3)):
        with pytest.raises(Exception):
            eng.train_steps(sched, first, n)
        with pytest.raises(Exception):
            eng.upload_steps(sched, first, n)
    with pytest.raises(Exception):
        eng.train_step(np.zeros(4, np.int32), np.ones(4, np.int32))
    assert eng.get_sample_pointer() == ptr
    for k in before:
        np.testing.assert_array_equal(before[k], eng.get(k), err_msg=k)


MK = dict(loss='bpr-max', final_act='elu-0.5', layers=[24], batch_size=16, n_epochs=2, n_sample=64, momentum=0.2, dropout_p_hidden=0.2)
LOSS_LINE = re.compile(r'Epoch\d+ --> loss: [0-9.]+')


def _quiet(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        fn()
    return buf.getvalue()


class _Stop(Exception):
    pass


def test_fit_resumable_and_fit_more(tmp_path):
    """(f) fit_resumable with bptt = 4, interrupted after its second checkpoint and called again, equals fit(); fit_more runs"""
    data = make_sessions(n_items=300, n_events=3000, seed=1)
    ref = GRU4Rec(**MK)
    ref.bptt = 4
    out_ref = _quiet(lambda: ref.fit(data.copy(), sample_store=64 * 23))
    assert ref._engine.bptt_windows() > 0
    path = str(tmp_path / 'run.npz')
    calls = []

    def stop(epoch, step):
        calls.append((epoch, step))
        if len(calls) == 2:
            raise _Stop()

    out = ''
    for attempt in range(2):
        gru = GRU4Rec(**MK)
        gru.set_params(bptt=4)
        try:
            out += _quiet(lambda: gru.fit_resumable(data.copy(), path, 24, sample_store=64 * 23, on_checkpoint=stop if attempt == 0 else None))
        except _Stop:
            pass
    assert 'Resuming from checkpoint' in out and calls[1][1] > 0
    assert LOSS_LINE.findall(out) == LOSS_LINE.findall(out_ref)
    names = gru._param_names() + gru._state_names()
    assert not [n for n in names if not np.array_equal(ref._engine.get(n), gru._engine.get(n))]
    assert GRU4Rec.load_checkpoint(path).bptt == 4
    w = gru._engine.bptt_windows()
    out = _quiet(lambda: gru.fit_more(data.copy(), n_epochs=1, sample_store=64 * 23))
    assert len(LOSS_LINE.findall(out)) == 1 and gru._engine.bptt_windows() > w


def test_run_py_trains_with_bptt(tmp_path):
    """(g) run.py train -ps ...,bptt=8 -t test --history H prints the epoch lines and the metrics"""
    data = make_sessions(n_items=300, n_events=20000, seed=4)
    cut = data.SessionId.max() * 3 // 5
    train, rest = data[data.SessionId <= cut], data[data.SessionId > cut]
    first = rest.groupby('SessionId').cumcount() == 0
    paths = [str(tmp_path / f) for f in ('train.tsv', 'test.tsv', 'history.tsv')]
    for frame, p in zip((train, rest[~first], rest[first]), paths):
        frame.to_csv(p, sep='\t', index=False)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'run.py'), paths[0], '-ps', 'layers=32,batch_size=16,n_epochs=2,n_sample=64,bptt=8',
                        '-t', paths[1], '--history', paths[2], '-m', '5', '10'], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert len(LOSS_LINE.findall(r.stdout)) == 2 and 'Recall@5' in r.stdout, r.stdout[-2000:]


def test_bptt_learns_what_one_step_updates_cannot():
    """(h) each session: its first item, four random distractors, then the first item again as the last target.  Predicting that
    target needs the state to keep the first item over four steps, which only a gradient through time asks the recurrent weights
    to do.  Recall@20 over those last events, from evaluate_events, with bptt = 6 against bptt = 1 after equal training."""
    from gru4rec_b200.evaluation import evaluate_events
    rs = np.random.RandomState(0)
    n_items, n_sess = 400, 6000
    rows = []
    for s in range(n_sess):
        a = rs.randint(n_items)
        seq = [a] + list(rs.randint(0, n_items, 4)) + [a]
        rows += [(s, it, s * 10 + k) for k, it in enumerate(seq)]
    df = pd.DataFrame(rows, columns=['SessionId', 'ItemId', 'Time'])
    train, test = df[df.SessionId < 5000], df[df.SessionId >= 5000]
    rec = {}
    for T in (1, 6):
        gru = GRU4Rec(loss='cross-entropy', final_act='softmax', layers=[64], batch_size=32, n_epochs=8, n_sample=0, learning_rate=0.05,
                      adapt='adagrad', dropout_p_hidden=0.0)
        gru.bptt = T
        _quiet(lambda: gru.fit(train.copy()))
        ev = evaluate_events(gru, test.copy(), cut_off=[20], batch_size=64)['events']
        last = ev[ev['Time'] % 10 == 5]
        assert len(last) == 1000
        rec[T] = float((last['rank'] <= 20).mean())
    print('Recall@20 on the repeated item: bptt=1 %.4f, bptt=6 %.4f' % (rec[1], rec[6]))
    assert rec[6] > rec[1], rec
