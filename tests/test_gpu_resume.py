"""-m gpu: continuing a training run (DESIGN §3i).

1. A handle rebuilt from an export -- every named tensor, the sample store and the g4r_train_state_export blob -- continues the
   run of the handle it came from bit for bit, on every kind of training step, with the cut inside a window, at a refill of the
   device sample store and in the epoch's shrinking tail.
2. GRU4Rec.fit_resumable interrupted after a checkpoint and called again equals fit(): epoch loss lines, weights, optimizer
   state.
3. GRU4Rec.fit_more over the same frame with no new items equals fit() with the epochs added up, when the first run ends where
   the sample store would be refilled anyway.
4. g4r_copy_item_tables: old rows bit-identical, new rows as given / zero, padding zero; fit_more's new rows and a step on the
   grown model against the float64 oracle; rows of items absent from the new data untouched.
5. recommend_sessions across fit_more.
6. Refusals leave the handle as it was."""
import contextlib
import io
import re

import numpy as np
import pytest
import gru4rec_oracle as orc
from gru4rec_b200 import _lib
from gru4rec_b200.gru4rec import GRU4Rec
from gru4rec_b200.synth import make_sessions
from gpu_utils import make_cfg, push_weights, opt_slots, random_opt_state, f64_run_steps, f64_failures
from test_gpu_windows import CASES as WINDOW_CASES, _mk

pytestmark = pytest.mark.gpu

ROWS = 7            # rows of the device sample store: it is refilled every 7 steps

# name -> (model keywords, n_items, step_mode, kernel path)
CASES = {
    'headline_fast': WINDOW_CASES['headline'][:2] + (2, 'fast'),
    'rsc15_persistent': WINDOW_CASES['rsc15'][:2] + (1, 'persistent'),
    'embed_2layer_drop_phases': WINDOW_CASES['embed64_2layer_drop'][:2] + (0, 'phases'),
    'adam': WINDOW_CASES['adam_embed_2layer_mom_l2'][:2] + (0, 'phases'),
    'rmsprop_cap_smooth': WINDOW_CASES['rmsprop_cap_smooth'][:2] + (0, 'phases'),
    'adadelta': (_mk(64, 32, 'cross-entropy', 'softmax', adapt='adadelta', adapt_params=[0.95], learning_rate=1.0, embedding=32), 4000, 0, 'phases'),
    'tc_L160_B64': WINDOW_CASES['tc_auto_L160_B64'][:2] + (2, 'tc'),
}


def _epoch(n_items, B, S, seed):
    """a whole epoch's schedule: it ends in the shrinking tail (M < B)"""
    rs = np.random.RandomState(seed)
    lens = rs.randint(2, 10, 6 * B)
    items = rs.randint(0, n_items, lens.sum()).astype(np.int64)
    offset = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    sched = _lib.Schedule(items, offset, np.arange(len(lens), dtype=np.int64), B, S, mode=0)
    return sched, sched.batch_sizes()


def _fresh(mk, n_items, step_mode, seed, init=True):
    """a training handle with the settings that come from the data (sampling CDF, logQ support); with `init`, also the state
    the run starts from: random weights, hidden state, optimizer state"""
    rs = np.random.RandomState(seed)
    eng = _lib.Engine(make_cfg(n_items, mk, sample_store=ROWS * mk['n_sample'], step_mode=step_mode))
    pop = rs.randint(1, 50, n_items).astype(np.float64) ** 0.5
    cdf = pop.cumsum() / pop.sum()
    cdf[-1] = 1
    eng.set_sampling_cdf(cdf.astype(np.float32))
    if mk.get('logq', 0):
        eng.set_logq_support(rs.randint(1, 50, n_items).astype(np.float32))
    m = orc.OracleGRU4Rec(**mk)
    if init:
        m.init(n_items)
        for h in m.H:
            h[:] = rs.randn(*h.shape).astype(np.float32) * 0.5
        push_weights(eng, m)
        random_opt_state(eng, m, np.random.RandomState(seed + 1))
    return eng, m


def _tensor_names(m):
    """parameters, their optimizer state, the training hidden state"""
    names = [k % i for i in range(len(m.layers)) for k in ('Wx%d', 'Wh%d', 'Wrz%d', 'Bh%d')] + ['Wy', 'By']
    if m.embedding and not m.constrained_embedding:
        names.append('E')
    return names + ['%s.%s' % (n, s) for n in names for s in opt_slots(m)] + ['H%d' % i for i in range(len(m.layers))]


def _export(eng, m):
    out = {n: eng.get(n) for n in _tensor_names(m)}
    out['store'], out['blob'] = eng.get_sample_store(), eng.train_state_export()
    out['pointer'] = np.array(eng.get_sample_pointer())
    return out


def _assert_path(eng, path, steps):
    launches, (fast, fallback) = eng.kernel_launches(), eng.fast_windows()
    assert eng.uses_tensor_cores() == (path == 'tc')
    if path == 'fast':
        assert fast > 0 and fallback == 0 and launches <= 2 * steps + 6, (launches, fast, fallback)
    elif path == 'persistent':
        assert fast == 0 and launches <= 2 * steps + 6, (launches, fast, fallback)
    else:
        assert fast == 0 and fallback == 0 and launches >= 8 * steps, (launches, fast, fallback)


@pytest.mark.parametrize('name', list(CASES))
def test_resumed_run_is_bit_identical(name):
    mk, n_items, step_mode, path = CASES[name]
    sched, M = _epoch(n_items, mk['batch_size'], mk['n_sample'], seed=11)
    N = sched.n_steps
    assert N > 3 * ROWS and M[N - 2] < mk['batch_size']
    eng, m = _fresh(mk, n_items, step_mode, seed=7)
    costs = eng.train_steps(sched, 0, N)
    _assert_path(eng, path, N)
    want = _export(eng, m)
    want['costs'] = costs
    assert np.isfinite(costs).all() and want['blob'].size > 64
    eng.close()
    # the cut: inside the first store, exactly where the store is used up (the next step refills it), in the shrinking tail
    for k in (3, 2 * ROWS, N - 2):
        eng, m = _fresh(mk, n_items, step_mode, seed=7)
        head = eng.train_steps(sched, 0, k)
        _assert_path(eng, path, k)
        saved = _export(eng, m)
        eng.close()
        eng, m = _fresh(mk, n_items, step_mode, seed=7, init=False)
        for n in _tensor_names(m):
            eng.set(n, saved[n])
        eng.set_sample_store(saved['store'])
        eng.train_state_import(saved['blob'])
        assert np.array_equal(eng.train_state_export(), saved['blob'])
        tail = eng.train_steps(sched, k, N - k)
        _assert_path(eng, path, N - k)
        got = _export(eng, m)
        got['costs'] = np.concatenate([head, tail])
        eng.close()
        differ = [n for n in want if not np.array_equal(want[n], got[n])]
        assert not differ, 'cut after step %d of %d: %s differ' % (k, N, differ)


# ---- the Python surface ----
MK = dict(loss='bpr-max', final_act='elu-0.5', layers=[24], batch_size=16, n_epochs=3, n_sample=64, momentum=0.2, dropout_p_hidden=0.2)
LOSS_LINE = re.compile(r'Epoch\d+ --> loss: [0-9.]+')


def _run(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        fn()
    return buf.getvalue()


def _model_state(gru):
    names = gru._param_names()
    return {n: gru._engine.get(n) for n in names + gru._state_names()}


class _Stop(Exception):
    pass


@pytest.mark.parametrize('extra,store_type', [({}, 'gpu'), (dict(train_random_order=True), 'gpu'), ({}, 'cpu')], ids=['plain', 'random_order', 'cpu_store'])
def test_fit_resumable_interrupted_equals_fit(tmp_path, extra, store_type):
    data = make_sessions(n_items=300, n_events=4000, seed=1)
    store = 64 * 23            # refilled many times per epoch, at steps that are no multiple of the checkpoint interval
    ref = GRU4Rec(**dict(MK, **extra))
    out_ref = _run(lambda: ref.fit(data.copy(), sample_store=store, store_type=store_type))
    path = str(tmp_path / 'run.npz')
    calls = []

    def stop_at_third(epoch, step):
        calls.append((epoch, step))
        if len(calls) == 3 or (epoch, step) == (2, 30):
            raise _Stop()

    out = ''
    for attempt in range(3):
        gru = GRU4Rec(**dict(MK, **extra))
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                gru.fit_resumable(data.copy(), path, 30, sample_store=store, store_type=store_type, on_checkpoint=stop_at_third if attempt < 2 else None)
        except _Stop:
            pass
        out += buf.getvalue()
    assert 'Resuming from checkpoint' in out and calls[2][1] > 0 and (2, 30) in calls, calls
    assert LOSS_LINE.findall(out) == LOSS_LINE.findall(out_ref) and len(LOSS_LINE.findall(out)) == 3
    a, b = _model_state(ref), _model_state(gru)
    assert not [n for n in a if not np.array_equal(a[n], b[n])]


def test_fit_more_without_new_items_equals_longer_fit():
    """Precondition of the equality: the first run ends exactly where the sample store is used up, so that the longer fit()
    refills it at the step at which fit_more() draws its new store -- the store holds one epoch's mini-batches."""
    data = make_sessions(n_items=300, n_events=4000, seed=2)
    probe = GRU4Rec(**dict(MK, n_epochs=1))
    _run(lambda: probe.fit(data.copy(), sample_store=64 * 100000))
    n_steps = probe._engine.get_sample_pointer()            # mini-batches of one epoch
    assert 100 < n_steps < 100000
    store = 64 * n_steps
    long = GRU4Rec(**dict(MK, n_epochs=3))
    out_long = _run(lambda: long.fit(data.copy(), sample_store=store))
    gru = GRU4Rec(**dict(MK, n_epochs=2))
    out = _run(lambda: gru.fit(data.copy(), sample_store=store))
    assert gru._engine.get_sample_pointer() == n_steps
    out += _run(lambda: gru.fit_more(data.copy(), n_epochs=1, sample_store=store))
    assert 'Optimizer state kept' in out
    assert [s.split(':')[1] for s in LOSS_LINE.findall(out)] == [s.split(':')[1] for s in LOSS_LINE.findall(out_long)]
    a, b = _model_state(long), _model_state(gru)
    assert not [n for n in a if not np.array_equal(a[n], b[n])]


@pytest.mark.parametrize('mode', ['none', 'embedding', 'constrained'])
@pytest.mark.parametrize('adapt', ['adam', 'adadelta'])
def test_copy_item_tables(mode, adapt):
    """L = 50: ldL = 52, two padding columns in every Wy row"""
    mk = _mk(50, 8, 'bpr-max', 'elu-0.5', S=32, adapt='adagrad' if mode == 'constrained' else adapt, adapt_params=[0.9, 0.999], momentum=0.3,
             embedding=20 if mode == 'embedding' else 0, constrained_embedding=mode == 'constrained')
    n_old, n_add = 211, 37
    src, m = _fresh(dict(mk), n_old, 0, seed=3)
    names = _tensor_names(m)
    before = {n: src.get(n) for n in names}
    dst = _lib.Engine(make_cfg(n_old + n_add, mk, sample_store=5 * 32, step_mode=0))
    junk = np.random.RandomState(0)
    for n in names:                    # whatever the destination held is overwritten, the new rows of the state included
        dst.set(n, junk.randn(*dst.shape(n)).astype(np.float32))
    rs = np.random.RandomState(1)
    new = dict(new_Wy=rs.randn(n_add, 50).astype(np.float32), new_By=rs.randn(n_add, 1).astype(np.float32))
    if mode != 'constrained':
        new['new_in'] = rs.randn(n_add, 20 if mode == 'embedding' else 150).astype(np.float32)
    v0 = dst.kernel_launches()
    dst.copy_item_tables(src, **new)
    assert dst.kernel_launches() > v0
    fills = {'Wy': new['new_Wy'], 'By': new['new_By'], ('E' if mode == 'embedding' else 'Wx0'): new.get('new_in')}
    tables = ('Wy', 'By') + (('E',) if mode == 'embedding' else ('Wx0',) if mode == 'none' else ())
    for n in names:
        got = dst.get(n)
        if n.split('.')[0] in tables:
            assert np.array_equal(got[:n_old], before[n]), n
            assert np.array_equal(got[n_old:], fills[n] if n in fills else np.zeros_like(got[n_old:])), n
        else:
            assert np.array_equal(got, before[n]), n
    assert all(np.array_equal(src.get(n), before[n]) for n in names)
    # the padding columns of the grown table are zero: a scoring pass over the grown catalogue reads whole rows
    X = np.arange(8, dtype=np.int32) + n_old
    assert np.isfinite(dst.predict(X)).all()
    src.close(); dst.close()


def _grown_pair(tmp_path, extra=None):
    """a trained model, and the frame it is grown with: 40 unseen items, and only half of the old catalogue"""
    mk = dict(MK, n_epochs=1, dropout_p_hidden=0.0, **(extra or {}))
    data = make_sessions(n_items=300, n_events=4000, seed=3)
    gru = GRU4Rec(**mk)
    _run(lambda: gru.fit(data.copy(), sample_store=64 * 50))
    more = make_sessions(n_items=190, n_events=3000, seed=4)
    old_ids = gru.itemidmap.index.values
    remap = np.concatenate([old_ids[:150], np.arange(10 ** 6, 10 ** 6 + 40)])
    more['ItemId'] = remap[more['ItemId'].values.astype(np.int64) % len(remap)]
    more['SessionId'] += 10 ** 6
    return gru, mk, data, more


@pytest.mark.parametrize('extra', [{}, dict(embedding=16), dict(constrained_embedding=True)], ids=['none', 'embedding', 'constrained'])
def test_fit_more_grows_the_catalogue(tmp_path, extra):
    gru, mk, data, more = _grown_pair(tmp_path, extra)
    n_old = gru.n_items
    old_ids = gru.itemidmap.index.values.copy()
    before = _model_state(gru)
    out = _run(lambda: gru.fit_more(more.copy(), n_epochs=0, sample_store=64 * 50))
    assert 'Optimizer state kept' in out and 'Added' in out
    first_seen = more['ItemId'].values[np.sort(np.unique(more['ItemId'].values, return_index=True)[1])]
    new_ids = np.array([i for i in first_seen if i >= 10 ** 6])
    n_add = len(new_ids)
    assert n_add > 0 and gru.n_items == n_old + n_add
    assert np.array_equal(gru.itemidmap.index.values[:n_old], old_ids) and np.array_equal(gru.itemidmap.index.values[n_old:], new_ids)
    # zero epochs: the grown model as fit_more() builds it -- old rows as they were, new rows by init_matrix's rule
    grown = _model_state(gru)
    rs = np.random.RandomState(42 + n_old)
    want = {}
    if extra.get('embedding'):
        want['E'] = gru._init_rows(rs, (n_add, 16))
    elif not extra:
        want['Wx0'] = np.hstack([gru._init_rows(rs, (n_add, 24)) for _ in range(3)])
    want['Wy'] = gru._init_rows(rs, (n_add, 24))
    want['By'] = np.zeros((n_add, 1), np.float32)
    for n, a in before.items():
        if n.split('.')[0] in want:
            assert np.array_equal(grown[n][:n_old], a), n
            assert np.array_equal(grown[n][n_old:], want[n] if n in want else np.zeros_like(grown[n][n_old:])), n
        elif not n.startswith('H'):
            assert np.array_equal(grown[n], a), n
    # two steps on the grown model, new items among inputs, targets and samples, each against the float64 oracle
    eng = gru._engine
    okw = {k: v for k, v in mk.items() if k != 'n_epochs'}
    rs = np.random.RandomState(5)
    store = eng.get_sample_store()
    store[:2, :8] = rs.randint(n_old, gru.n_items, (2, 8))
    eng.set_sample_store(store)
    steps = []
    for _ in range(2):
        X, Y = rs.randint(0, gru.n_items, 16), rs.randint(0, gru.n_items, 16)
        X[:4], Y[4:8] = rs.randint(n_old, gru.n_items, 4), rs.randint(n_old, gru.n_items, 4)
        steps.append((X, Y, np.zeros(16, bool)))
    g0 = int(eng.train_state_export().view(np.uint32)[10])        # the global step (dropout is off in this model)
    assert g0 > 0
    checks, _, _ = f64_run_steps(eng, okw, gru.n_items, store, steps, None, None, require_dsy=False)
    failed = f64_failures(checks)
    assert not failed, '\n'.join(failed)
    # one epoch on the new frame: rows of items absent from it stay as they were, optimizer state included
    absent = np.setdiff1d(np.arange(gru.n_items), gru.itemidmap[more['ItemId'].unique()].values)
    assert len(absent) > 100
    prev = _model_state(gru)
    out = _run(lambda: gru.fit_more(more.copy(), n_epochs=1, sample_store=64 * 50))
    assert len(LOSS_LINE.findall(out)) == 1 and 'Added' not in out
    after = _model_state(gru)
    tables = [n for n in prev if n.split('.')[0] in ('Wy', 'By', 'E') or (n.split('.')[0] == 'Wx0' and not extra)]
    for n in tables:
        assert np.array_equal(prev[n][absent], after[n][absent]), n
    assert any(not np.array_equal(prev[n], after[n]) for n in tables)


def test_sessions_survive_growth_and_new_items_are_served(tmp_path):
    gru, mk, data, more = _grown_pair(tmp_path)
    twin, _, _, _ = _grown_pair(tmp_path)
    a, b = gru.itemidmap.index.values[3], gru.itemidmap.index.values[17]
    gru.recommend_sessions([901], [a], k=5)
    _run(lambda: gru.fit_more(more.copy(), n_epochs=0, sample_store=64 * 50))
    _run(lambda: twin.fit_more(more.copy(), n_epochs=0, sample_store=64 * 50))
    twin.recommend_sessions([901], [a], k=5)
    ids1, sc1 = gru.recommend_sessions([901], [b], k=5)
    ids2, sc2 = twin.recommend_sessions([901], [b], k=5)
    assert np.array_equal(ids1, ids2) and np.array_equal(sc1, sc2)
    new_a, new_b = gru.itemidmap.index.values[-2:]
    assert new_a >= 10 ** 6 and new_b >= 10 ** 6
    ids, sc = gru.recommend_sessions([901], [new_a], k=1, items=[new_a, new_b], exclude_seen=True)
    assert ids[0, 0] == new_b and np.isfinite(sc).all()


def test_refusals_leave_the_handle_untouched():
    mk = _mk(24, 8, 'bpr-max', 'elu-0.5', S=32, adapt='adagrad')
    eng, m = _fresh(mk, 200, 0, seed=1)
    eng.generate_samples()
    blob = eng.train_state_export()
    other = _lib.Engine(make_cfg(200, mk, sample_store=(ROWS + 1) * 32, step_mode=0))      # another store size
    other_blob = other.train_state_export()
    wrong_version = blob.copy(); wrong_version.view(np.uint32)[1] += 1
    wrong_magic = blob.copy(); wrong_magic[0] ^= 0xff
    wrong_sample = blob.copy(); wrong_sample.view(np.int32)[4] += 1
    for bad in (blob[:-8], blob[:16], wrong_version, wrong_magic, wrong_sample, other_blob):
        with pytest.raises(NotImplementedError):
            eng.train_state_import(bad)
        assert np.array_equal(eng.train_state_export(), blob)
    eng.train_state_import(blob)
    # copy_item_tables: another layer width, fewer items, another optimizer
    before = {n: other.get(n) for n in _tensor_names(m)}
    for mk2, n_items in ((dict(mk, layers=[28]), 200), (mk, 150), (dict(mk, adapt='adam', adapt_params=[0.9, 0.999]), 200)):
        src = _lib.Engine(make_cfg(n_items, mk2, sample_store=ROWS * 32, step_mode=0))
        with pytest.raises(NotImplementedError):
            (other if n_items == 200 else src).copy_item_tables(src if n_items == 200 else other)
        src.close()
    assert all(np.array_equal(other.get(n), before[n]) for n in before)
    eng.close(); other.close()
