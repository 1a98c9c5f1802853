"""-m gpu: full-softmax training (full_softmax=True, DESIGN §3n) -- every step scores and updates the whole catalogue.

(a) step by step against the float64 restatement (tests/full_softmax_oracle.py), the oracle re-seeded from the device before every
step: the cost, y / H / dvec of every layer, dSx, and either every gradient recovered from a plain SGD update or the update of
every weight and every optimizer-state tensor (every Wy / By row changes); (b) the shipped shapes; (c) two runs, window sizes
1 and 16, and logq / n_sample / sample_alpha are bitwise irrelevant, and a sampled handle is unaffected by a full one; (d) the
counters; (e) fit_resumable interrupted and resumed equals fit(), fit() -> evaluate_gpu and run.py."""
import contextlib
import io
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import full_softmax_oracle as fso
from gru4rec_b200 import _lib
from gru4rec_b200.gru4rec import GRU4Rec
from gru4rec_b200.synth import make_sessions
from gpu_utils import make_cfg, push_weights, random_opt_state, oracle_f64, param_names, oracle_param, opt_slots, f64_failures
import gru4rec_oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mk(L, B, loss='cross-entropy', fact='softmax', **kw):
    mk = dict(layers=[L] if isinstance(L, int) else list(L), batch_size=B, n_sample=2048, loss=loss, final_act=fact, adapt=None,
              learning_rate=0.5, momentum=0.0)
    mk.update(kw)
    return mk


ADA = dict(adapt='adagrad', learning_rate=0.05, momentum=0.3, lmbd=1e-3)
# name -> (model keywords, n_items).  Catalogues that are not a multiple of the 64-item tile end in a padded last tile.
CASES = {
    'none_xe_sgd': (_mk(48, 16), 3001),
    'none_xelogit_adagrad': (_mk(40, 12, 'xe_logit', 'softmax_logit', **ADA), 2500),
    'embed_xe_adagrad_drop': (_mk(40, 16, embedding=24, dropout_p_hidden=0.3, dropout_p_embed=0.2, **ADA), 2049),
    'embed_xelogit_sgd': (_mk(36, 8, 'xe_logit', 'softmax_logit', embedding=20), 1000),
    'shared_xe_adagrad_drop': (_mk(64, 32, constrained_embedding=True, dropout_p_hidden=0.3, dropout_p_embed=0.2, logq=1.0, **ADA), 5000),
    'shared_xelogit_sgd': (_mk(32, 16, 'xe_logit', 'softmax_logit', constrained_embedding=True), 1999),
    'two_layer_none_xe': (_mk([32, 40], 8, **ADA), 1000),
    'two_layer_shared_sgd': (_mk([24, 28], 8, constrained_embedding=True, dropout_p_hidden=0.2), 1500),
    'B1_shared_xe': (_mk(16, 1, constrained_embedding=True, **ADA), 777),
    'adam_embed_xe': (_mk(32, 16, embedding=16, adapt='adam', adapt_params=[0.9, 0.999], learning_rate=0.01), 1200),
    'rmsprop_none_xelogit': (_mk(32, 16, 'xe_logit', 'softmax_logit', adapt='rmsprop', adapt_params=[0.9], learning_rate=0.01, momentum=0.2), 1300),
}
SHIPPED = {
    'rsc15_xe_shared': (_mk(100, 32, constrained_embedding=True, dropout_p_hidden=0.4, adapt='adagrad', learning_rate=0.2, momentum=0.2,
                            sample_alpha=0.5, bpreg=0.0, logq=1.0), 37483),
    'rees46_xe_shared': (_mk(512, 240, constrained_embedding=True, dropout_p_embed=0.45, adapt='adagrad', learning_rate=0.065,
                             sample_alpha=0.5, bpreg=0.0, logq=1.0), 172000),
}


def _engine(mk, n_items, seed=0, **cfgkw):
    """a full-softmax engine with random weights, hidden state, biases and optimizer state"""
    rs = np.random.RandomState(seed)
    m = orc.OracleGRU4Rec(**mk)
    m.init(n_items)
    for h in m.H:
        h[:] = rs.randn(*h.shape).astype(np.float32) * 0.5
    m.By[:] = rs.randn(*m.By.shape).astype(np.float32) * 0.1
    for b in m.Bh:
        b[:] = rs.randn(*b.shape).astype(np.float32) * 0.1
    eng = _lib.Engine(make_cfg(n_items, mk, full_softmax=True, **cfgkw))
    push_weights(eng, m)
    random_opt_state(eng, m, np.random.RandomState(seed + 2))
    return eng


def _steps(n_items, B, seed):
    """step 1: every lane, one reset; step 2: M < B (B > 1), a duplicated input and a target that is also an input"""
    rs = np.random.RandomState(seed)
    X = rs.randint(0, n_items, B); Y = rs.randint(0, n_items, B); R = rs.rand(B) < 0.2
    out = [(X, Y, R)]
    M = max(1, B - 3)
    X2 = rs.randint(0, n_items, M); Y2 = rs.randint(0, n_items, M); R2 = rs.rand(M) < 0.2
    if M > 2:
        X2[1] = X2[0]; Y2[2] = X2[0]
    return out + [(X2, Y2, R2)]


def _rows(C, G):
    """(table, rows, per-position gradient) of the row tables of a full step"""
    I = len(C['Y'])
    if C['mode'] == 'shared':
        out = [('Wy', C['Xc'], np.vstack([G['dSx'], G['dSy']]))]
    elif C['mode'] == 'embed':
        out = [('E', C['X'], G['dSx']), ('Wy', np.arange(I), G['dSy'])]
    else:
        out = [('Wx0', C['X'], G['dSx']), ('Wy', np.arange(I), G['dSy'])]
    return out + [('By', np.arange(I), G['dSBy'])]


def _wgmma(mk, n_items, eval_tc=None):
    """the score tiles a full step runs on: forced by eval_tc, else wgmma from 64 lanes and 2048 items (wgmma_tiles)"""
    return eval_tc if eval_tc is not None else (mk['batch_size'] >= 64 and n_items >= 2048)


def _launches(mk, tc):
    """kernel launches of one Engine.train_step: plan, [input flags], the graph's step, its launch"""
    mode = 2 if mk.get('constrained_embedding') else (1 if mk.get('embedding') else 0)
    step = (mode != 0) + 5 + (2 if tc else 0) + 1
    step += sum(5 + (1 if (i > 0 or mode != 0) else 0) for i in range(len(mk['layers'])))     # f1, f2, b1, b2, [b3], dense
    return 1 + (mode == 2) + step + 1


def _run_steps(eng, mk, n_items, steps, tc=False):
    """checks of every step against the float64 restatement re-seeded from the device (gpu_utils' bar); `tc`: the step must run
    the wgmma score tiles (two more launches: the operand splits)"""
    sgd = mk.get('adapt', 'adagrad') is None and not mk.get('momentum', 0) and not mk.get('lmbd', 0)
    lr = mk['learning_rate']
    f64 = lambda a: np.asarray(a, np.float64)
    ulp = lambda a, b: 2.0 ** -23 * (np.abs(a) + np.abs(b))
    checks, costs = [], []
    for k, (X, Y, R) in enumerate(steps):
        m = oracle_f64(eng, mk, n_items, k)
        names, slots = param_names(m), opt_slots(m)
        W0 = {n: eng.get(n) for n in names}
        S0 = {(n, s): eng.get('%s.%s' % (n, s)) for n in names for s in slots}
        n0, l0 = eng.full_steps(), eng.kernel_launches()
        cost = eng.train_step(X, Y, R)
        assert eng.full_steps() == n0 + 1 and eng.fast_windows() == (0, 0)
        assert eng.kernel_launches() - l0 == _launches(mk, tc), 'expected the %s score tiles' % ('wgmma' if tc else 'fp32')
        costs.append(cost)
        ref_cost = fso.train_step_full(m, X, Y, R)
        C, G = m.last_cache, m.last_grads
        M, tag = len(X), 'step %d (M=%d) ' % (k + 1, len(X))
        ys = [lc['inp'] for lc in C['layers'][1:]] + [C['y_last']]
        checks.append((tag + 'cost', np.float64(cost), ref_cost, 0.0))
        for i in range(len(m.layers)):
            checks += [(tag + 'y%d' % i, eng.get('y%d' % i)[:M], ys[i], 0.0), (tag + 'H%d' % i, eng.get('H%d' % i)[:M], C['H_new'][i], 0.0),
                       (tag + 'dvec%d' % i, eng.get('dvec%d' % i)[:M], G['dvec'][i], 0.0)]
        if C['mode'] != 'none':
            checks.append((tag + 'dSx', eng.get('dSx')[:M], G['dSx'], 0.0))
        W1 = {n: eng.get(n) for n in names}
        rows = {n: np.unique(idx, return_inverse=True, return_counts=True) for n, idx, _ in _rows(C, G)}
        assert (W1['Wy'] != W0['Wy']).any(axis=1).mean() > 0.99, tag + 'not every Wy row changed'
        if sgd:
            dense = [('Wx%d' % i, G['dWx'][i]) for i in range(len(m.layers)) if G['dWx'][i] is not None]
            dense += [(n % i, G[g][i]) for i in range(len(m.layers)) for n, g in (('Wh%d', 'dWh'), ('Wrz%d', 'dWrz'), ('Bh%d', 'dBh'))]
            for n, g in dense:
                w0, w1 = f64(W0[n]), f64(W1[n])
                checks.append((tag + 'd' + n, (w0 - w1).reshape(g.shape) / lr, g, ulp(w0, w1).reshape(g.shape) / lr))
            for n, idx, g in _rows(C, G):
                r, inv, cnt = rows[n]
                w0, w1 = f64(W0[n][r]), f64(W1[n][r])
                gref = np.zeros((len(r),) + W0[n].shape[1:])
                np.add.at(gref, inv.reshape(-1), g.reshape(len(idx), -1))
                checks.append((tag + 'd' + n + ' rows', (w0 - w1) / lr, gref, cnt[:, None] * ulp(w0, w1) / lr))
        else:
            for n in names:
                mult = rows[n][2][:, None] if n in rows else 1
                sel = rows[n][0] if n in rows else slice(None)
                pairs = [(n, W0[n], W1[n], oracle_param(m, n))] + [('%s.%s' % (n, s), S0[(n, s)], eng.get('%s.%s' % (n, s)), m.opt[(n, s)]) for s in slots]
                for what, a0, a1, r1 in pairs:
                    r1 = np.asarray(r1).reshape(a0.shape)[sel]
                    a0, a1 = f64(a0[sel]), f64(a1[sel])
                    checks.append((tag + what + ' update', a1 - a0, r1 - a0, mult * ulp(a0, a1)))
    return checks, costs


# (case, eval_tc): None = the automatic choice; True / False force the wgmma / fp32 score tiles where the shape picks the other
PARAMS = [(n, None) for n in sorted(CASES)] + [(n, True) for n in ('none_xe_sgd', 'embed_xelogit_sgd', 'shared_xe_adagrad_drop',
                                                                   'two_layer_none_xe', 'B1_shared_xe', 'adam_embed_xe')] + \
         [('wide_shared_xe', False), ('wide_none_xelogit', False)]
CASES.update({
    # 64 lanes or more and 2048 items or more: the automatic choice is wgmma
    'wide_shared_xe': (_mk(128, 96, constrained_embedding=True, dropout_p_embed=0.2, **ADA), 9000),
    'wide_none_xelogit': (_mk(64, 130, 'xe_logit', 'softmax_logit'), 4100),
})
PARAMS += [('wide_shared_xe', None), ('wide_none_xelogit', None)]


@pytest.mark.parametrize('name,eval_tc', PARAMS, ids=['%s-%s' % (n, {None: 'auto', True: 'wgmma', False: 'fp32'}[t]) for n, t in PARAMS])
def test_full_step_matches_float64(name, eval_tc):
    """(a) two steps of every case against float64 (bar of gpu_utils: 4e-5 of max |ref| / 1e-3 relative above 1 % of max), on
    the score tiles the shape picks and on the other kind forced"""
    mk, n_items = CASES[name]
    eng = _engine(mk, n_items, **({} if eval_tc is None else dict(eval_tc=eval_tc)))
    checks, _ = _run_steps(eng, mk, n_items, _steps(n_items, mk['batch_size'], 1), tc=_wgmma(mk, n_items, eval_tc))
    failed = f64_failures(checks)
    assert not failed, '\n'.join(failed)
    eng.close()


@pytest.mark.parametrize('name', sorted(SHIPPED))
def test_shipped_shapes_match_float64(name):
    """(b) the RSC15 XE-shared and the Rees46 shapes, two steps each"""
    mk, n_items = SHIPPED[name]
    eng = _engine(mk, n_items)
    checks, _ = _run_steps(eng, mk, n_items, _steps(n_items, mk['batch_size'], 2), tc=_wgmma(mk, n_items))
    failed = f64_failures(checks)
    assert not failed, '\n'.join(failed)
    eng.close()


def _schedule_run(mk, n_items, cfgkw=None, seed=3, steps=None):
    """an epoch schedule (resets, compacted tail) through train_steps; returns costs and every parameter and state tensor"""
    items, offset = _sessions(n_items, mk['batch_size'], seed)
    sched = _lib.Schedule(items, offset, np.arange(len(offset) - 1, dtype=np.int64), mk['batch_size'], mk.get('n_sample', 0), mode=0)
    eng = _engine(mk, n_items, **(cfgkw or {}))
    n = sched.n_steps if steps is None else steps
    costs = eng.train_steps(sched, 0, n)
    m = orc.OracleGRU4Rec(**mk)
    m.E = np.zeros(1) if (mk.get('embedding') and not mk.get('constrained_embedding')) else None
    names = param_names(m) + ['H%d' % i for i in range(len(mk['layers']))]
    names += ['%s.%s' % (p, s) for p in param_names(m) for s in opt_slots(m)]
    out = dict(costs=np.asarray(costs), **{k: eng.get(k) for k in names})
    assert eng.full_steps() == n
    eng.close()
    return out, n


def _sessions(n_items, B, seed):
    rs = np.random.RandomState(seed)
    lens = rs.randint(2, 12, 4 * B + 3)
    items = rs.randint(0, n_items, int(lens.sum())).astype(np.int64)
    return items, np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _same(a, b):
    bad = [k for k in a if not np.array_equal(a[k], b[k])]
    assert not bad, 'differ: %s' % bad


BIT_MK = _mk(32, 8, constrained_embedding=True, dropout_p_hidden=0.2, dropout_p_embed=0.1, **ADA)


@pytest.mark.parametrize('eval_tc', [False, True], ids=['fp32', 'wgmma'])
def test_bitwise_properties(eval_tc):
    """(c) on either score tile kind: two runs are identical; windows of 1 and 16 steps agree; logq, n_sample and sample_alpha
    change nothing; (d) the counter"""
    kw = dict(eval_tc=eval_tc)
    a, n = _schedule_run(BIT_MK, 3000, kw)
    assert n > 16
    b, _ = _schedule_run(BIT_MK, 3000, kw)
    _same(a, b)
    c, _ = _schedule_run(BIT_MK, 3000, dict(kw, max_resident_steps=1))
    _same(a, c)
    d, _ = _schedule_run(BIT_MK, 3000, dict(kw, max_resident_steps=16))
    _same(a, d)
    e, _ = _schedule_run(dict(BIT_MK, logq=1.0, n_sample=64, sample_alpha=0.3), 3000, dict(kw, sample_store=64 * 50))
    _same(a, e)


def test_sampled_handle_unaffected_by_a_full_one():
    """(c) a full_softmax=False run is the same before and after a full-softmax handle lived in the process"""
    mk = dict(BIT_MK, n_sample=32)

    def sampled():
        items, offset = _sessions(700, 8, 5)
        sched = _lib.Schedule(items, offset, np.arange(len(offset) - 1, dtype=np.int64), 8, 32, mode=0)
        eng = _lib.Engine(make_cfg(700, mk, sample_store=32 * 40))
        m = orc.OracleGRU4Rec(**mk); m.init(700)
        push_weights(eng, m)
        eng.set_sampling_cdf((np.arange(1, 701) / 700.0).astype(np.float32))
        eng.generate_samples()
        costs = eng.train_steps(sched, 0, sched.n_steps)
        out = dict(costs=np.asarray(costs), Wy=eng.get('Wy'), By=eng.get('By'), Wh0=eng.get('Wh0'))
        assert eng.full_steps() == 0
        eng.close()
        return out
    before = sampled()
    full, _ = _schedule_run(BIT_MK, 700)
    after = sampled()
    _same(before, after)


MK = dict(loss='cross-entropy', final_act='softmax', layers=[24], batch_size=16, n_epochs=2, n_sample=64, momentum=0.2,
          dropout_p_hidden=0.2, learning_rate=0.1)
LOSS_LINE = re.compile(r'Epoch\d+ --> loss: [0-9.]+')


def _quiet(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        fn()
    return buf.getvalue()


class _Stop(Exception):
    pass


def test_fit_resumable_fit_more_and_evaluate(tmp_path):
    """(e) fit_resumable with full_softmax, interrupted after its second checkpoint and called again, equals fit(); fit_more
    continues; evaluate_gpu ranks the trained model"""
    from gru4rec_b200 import evaluation
    data = make_sessions(n_items=300, n_events=3000, seed=1)
    ref = GRU4Rec(**MK)
    ref.full_softmax = True
    out_ref = _quiet(lambda: ref.fit(data.copy(), sample_store=64 * 23))
    assert 'Full softmax' in out_ref and 'sample store' not in out_ref
    assert ref._engine.full_steps() > 0
    path = str(tmp_path / 'run.npz')
    calls = []

    def stop(epoch, step):
        calls.append((epoch, step))
        if len(calls) == 2:
            raise _Stop()

    out = ''
    for attempt in range(2):
        gru = GRU4Rec(**MK)
        gru.set_params(full_softmax=True)
        try:
            out += _quiet(lambda: gru.fit_resumable(data.copy(), path, 24, sample_store=64 * 23, on_checkpoint=stop if attempt == 0 else None))
        except _Stop:
            pass
    assert 'Resuming from checkpoint' in out and calls[1][1] > 0
    assert LOSS_LINE.findall(out) == LOSS_LINE.findall(out_ref)
    names = gru._param_names() + gru._state_names()
    assert not [n for n in names if not np.array_equal(ref._engine.get(n), gru._engine.get(n))]
    assert GRU4Rec.load_checkpoint(path).full_softmax is True
    n = gru._engine.full_steps()
    out = _quiet(lambda: gru.fit_more(data.copy(), n_epochs=1, sample_store=64 * 23))
    assert len(LOSS_LINE.findall(out)) == 1 and gru._engine.full_steps() > n
    rec, mrr = evaluation.evaluate_gpu(gru, data.copy(), batch_size=50, cut_off=[20])
    assert 0.0 < rec[0] <= 1.0 and 0.0 < mrr[0] <= rec[0]


def test_run_py_trains_with_full_softmax(tmp_path):
    """(e) run.py train -ps ...,full_softmax=True -t test prints the set line, the epoch lines and the metrics"""
    data = make_sessions(n_items=300, n_events=20000, seed=4)
    cut = data.SessionId.max() * 3 // 5
    paths = [str(tmp_path / f) for f in ('train.tsv', 'test.tsv')]
    data[data.SessionId <= cut].to_csv(paths[0], sep='\t', index=False)
    data[data.SessionId > cut].to_csv(paths[1], sep='\t', index=False)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'run.py'), paths[0], '-ps',
                        'loss=cross-entropy,final_act=softmax,layers=32,batch_size=16,n_epochs=2,n_sample=64,full_softmax=True',
                        '-t', paths[1], '-m', '5', '10'], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert re.search(r'SET\s+full_softmax\s+TO\s+True', r.stdout), r.stdout[-2000:]
    assert len(LOSS_LINE.findall(r.stdout)) == 2 and 'Recall@5' in r.stdout, r.stdout[-2000:]
