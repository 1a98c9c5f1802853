"""CPU tests of the host logic of continued training (GRU4Rec.save_checkpoint / load_checkpoint / fit_resumable / fit_more and
run.py's flags for them; DESIGN §3i) on the engine double, extended here with what the library adds for it: optimizer state and
the training hidden state by name, Engine.train_state_export / train_state_import (the oracle's step counter, the sample
pointer and the MRG stream states, refused for another n_sample / store size) and Engine.copy_item_tables, all on the oracle's
own arrays.  The device side is tested in test_gpu_resume.py."""
import contextlib
import io
import os
import re
import sys

import numpy as np
import pytest

from gru4rec_b200 import _lib
from gru4rec_b200.gru4rec import GRU4Rec
from gru4rec_b200.synth import make_sessions
import oracle_engine
from gpu_utils import oracle_param, OPT_SLOTS
from test_host_sessions import SessionOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITEM_TABLES = ('Wy', 'By', 'E')


class ResumeOracleEngine(SessionOracleEngine):
    def _param2d(self, name):
        p = np.asarray(oracle_param(self.m, name))
        return p.reshape(1, -1) if name.startswith('Bh') else p.reshape(p.shape[0], -1)

    def get(self, name):
        if '.' in name:
            p, slot = name.split('.')
            like = self._param2d(p)
            return np.array(self.m.opt.get((p, slot), np.zeros_like(like)), np.float32).reshape(like.shape)
        if name[0] == 'H' and name[1:].isdigit():
            return self.m.H[int(name[1:])].copy()
        return super().get(name)

    def set(self, name, arr):
        if '.' in name:
            p, slot = name.split('.')
            self.m.opt[(p, slot)] = np.array(arr, np.float32).reshape(np.asarray(oracle_param(self.m, p)).shape)
        elif name[0] == 'H' and name[1:].isdigit():
            self.m.H[int(name[1:])][:] = arr
        else:
            super().set(name, arr)

    def get_sample_store(self):
        return np.zeros((self.gen_len, self.S), np.int64) if self.store is None else np.array(self.store, np.int64)

    def _fingerprint(self):
        return [self.S, self.gen_len]

    def train_state_export(self):
        streams = np.zeros(0, np.int64) if self.mrg_state is None else np.asarray(self.mrg_state, np.int64).reshape(-1)
        head = np.array(self._fingerprint() + [self.m.step_count, self.ptr, streams.size], np.int64)
        return np.concatenate([head, streams]).view(np.uint8).copy()

    def train_state_import(self, blob):
        blob = np.ascontiguousarray(blob, np.uint8)
        if blob.size < 40 or blob.size % 8:
            raise NotImplementedError('truncated blob')
        a = blob.view(np.int64)
        if list(a[:2]) != self._fingerprint() or a.size != 5 + a[4]:
            raise NotImplementedError('the blob was exported with another n_sample / sample-store size')
        self.m.step_count, self.ptr = int(a[2]), int(a[3])
        if a[4]:
            import gru4rec_oracle as orc
            self.mrg = orc.MRGStreams(12345)
            self.mrg_state = a[5:].reshape(-1, 6).copy()

    def copy_item_tables(self, src, new_Wy=None, new_By=None, new_in=None):
        mode_in = 'E' if self.m.E is not None else ('Wx0' if not self.m.constrained_embedding else None)
        fills = {'Wy': new_Wy, 'By': new_By, mode_in: new_in}
        names = src_names = [n for n in ['Wx%d' % i for i in range(self.n_layers)] + ['Wh%d' % i for i in range(self.n_layers)] +
                             ['Wrz%d' % i for i in range(self.n_layers)] + ['Bh%d' % i for i in range(self.n_layers)] + ['Wy', 'By'] +
                             (['E'] if self.m.E is not None else [])]
        slots = OPT_SLOTS[self.m.adapt] + (('vel',) if self.m.momentum > 0 else ())
        for n in names:
            for full in [n] + ['%s.%s' % (n, s) for s in slots]:
                a = src.get(full)
                if n in ITEM_TABLES or n == mode_in:
                    add = int(self.cfg.n_items) - a.shape[0]
                    fill = fills.get(full)
                    a = np.vstack([a, np.zeros((add, a.shape[1]), np.float32) if fill is None else np.asarray(fill, np.float32).reshape(add, -1)])
                self.set(full, a)
        for i in range(self.n_layers):
            self.set('H%d' % i, src.get('H%d' % i))
        assert src_names


def _install(monkeypatch, made=None):
    """every engine a GRU4Rec builds is the double (it takes the model keywords from the configuration's owner)"""
    made = [] if made is None else made
    owner = []

    def make(cfg, device=0):
        eng = ResumeOracleEngine(cfg, oracle_engine.model_kwargs_of(owner[-1]), device)
        made.append(eng)
        return eng
    monkeypatch.setattr(_lib, 'Engine', make)
    real = GRU4Rec._make_config

    def make_config(self, *a, **k):
        owner.append(self)
        return real(self, *a, **k)
    monkeypatch.setattr(GRU4Rec, '_make_config', make_config)
    return made


MK = dict(loss='bpr-max', final_act='elu-0.5', layers=[10], batch_size=8, n_epochs=2, n_sample=16, momentum=0.1, dropout_p_hidden=0.2)
LOSS_LINE = re.compile(r'Epoch\d+ --> loss: [0-9.]+')
STORE = 16 * 9


def _run(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        fn()
    return buf.getvalue()


def _state(gru):
    return {n: gru._engine.get(n) for n in gru._param_names() + gru._state_names()}


def _data(seed=1, n_items=60, n_events=500):
    return make_sessions(n_items=n_items, n_events=n_events, seed=seed)


class _Stop(Exception):
    pass


@pytest.mark.parametrize('extra,store_type', [({}, 'gpu'), (dict(train_random_order=True), 'gpu'), ({}, 'cpu')], ids=['plain', 'random_order', 'cpu_store'])
def test_fit_resumable_equals_fit(monkeypatch, tmp_path, extra, store_type):
    _install(monkeypatch)
    data = _data()
    ref = GRU4Rec(**dict(MK, **extra))
    out_ref = _run(lambda: ref.fit(data.copy(), sample_store=STORE, store_type=store_type))
    path = str(tmp_path / 'run.npz')
    replaced = []
    real_replace = os.replace
    monkeypatch.setattr(os, 'replace', lambda a, b: (replaced.append((a, b)), real_replace(a, b))[1])
    calls = []

    def stop(epoch, step):
        calls.append((epoch, step))
        assert os.path.exists(path) and os.listdir(str(tmp_path)) == ['run.npz']        # in place, no temporary file left
        if len(calls) == 2 or (epoch, step) == (1, 14):
            raise _Stop()

    out = ''
    for attempt in range(3):
        gru = GRU4Rec(**dict(MK, **extra))
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                gru.fit_resumable(data.copy(), path, 7, sample_store=STORE, store_type=store_type, on_checkpoint=stop if attempt < 2 else None)
        except _Stop:
            pass
        out += buf.getvalue()
    assert calls[1] == (0, 14) and (1, 14) in calls and out.count('Resuming from checkpoint') == 2
    assert all(b == path and a != path and os.path.dirname(a) == str(tmp_path) for a, b in replaced) and len(replaced) >= len(calls)
    assert LOSS_LINE.findall(out) == LOSS_LINE.findall(out_ref) and len(LOSS_LINE.findall(out)) == 2
    a, b = _state(ref), _state(gru)
    assert not [n for n in a if not np.array_equal(a[n], b[n])]
    # a finished run's checkpoint: nothing left to do
    again = GRU4Rec(**dict(MK, **extra))
    assert not LOSS_LINE.findall(_run(lambda: again.fit_resumable(data.copy(), path, 7, sample_store=STORE, store_type=store_type)))


def test_checkpoint_of_other_data_starts_anew(monkeypatch, tmp_path):
    _install(monkeypatch)
    path = str(tmp_path / 'run.npz')
    data = _data()
    _run(lambda: GRU4Rec(**MK).fit_resumable(data.copy(), path, 50, sample_store=STORE))
    for frame, mk, store in ((_data(seed=2), MK, STORE), (data, dict(MK, learning_rate=0.05), STORE), (data, MK, 16 * 5)):
        ref = GRU4Rec(**mk)
        out_ref = _run(lambda: ref.fit(frame.copy(), sample_store=store))
        gru = GRU4Rec(**mk)
        out = _run(lambda: gru.fit_resumable(frame.copy(), path, 50, sample_store=store))
        assert 'WARNING: checkpoint' in out and 'starting a new run' in out and 'Resuming' not in out
        assert LOSS_LINE.findall(out) == LOSS_LINE.findall(out_ref)
        os.remove(path)
        _run(lambda: GRU4Rec(**MK).fit_resumable(data.copy(), path, 50, sample_store=STORE))


def test_checkpoint_round_trip_and_pickles_unchanged(monkeypatch, tmp_path):
    _install(monkeypatch)
    data = _data()
    data['ItemId'] = data['ItemId'].astype(str)
    gru = GRU4Rec(**dict(MK, adapt='adam', adapt_params=[0.9, 0.999]))
    _run(lambda: gru.fit(data.copy(), sample_store=STORE))
    p1, p2, ck = str(tmp_path / 'a.pickle'), str(tmp_path / 'b.pickle'), str(tmp_path / 'm.npz')
    gru.savemodel(p1)
    before = _state(gru)
    blob, store = gru._engine.train_state_export(), gru._engine.get_sample_store()
    gru.save_checkpoint(ck)
    with np.load(ck, allow_pickle=False) as z:            # arrays and one JSON string: loads with pickle switched off
        assert 'meta' in z.files and 'state/Wy.countt' in z.files and 'param/Wy' in z.files
    back = GRU4Rec.load_checkpoint(ck)
    assert back.itemidmap.index.dtype == gru.itemidmap.index.dtype and list(back.itemidmap.index) == list(gru.itemidmap.index)
    assert back.layers == gru.layers and back.adapt == 'adam' and back.adapt_params == [0.9, 0.999]
    for n in gru._param_names():
        assert np.array_equal(np.asarray(back._host[n]).reshape(before[n].shape), before[n])
    gru.savemodel(p2)                 # the same model after the checkpoint round trip: the same bytes
    assert open(p1, 'rb').read() == open(p2, 'rb').read()
    # the loaded model continues from the saved state
    out = _run(lambda: back.fit_more(data.copy(), n_epochs=0, sample_store=STORE))
    assert 'Optimizer state kept' in out and 'Added' not in out
    after = _state(back)
    assert not [n for n in before if not np.array_equal(before[n], after[n])]
    assert back._engine.m.step_count == gru._engine.m.step_count > 0
    assert np.array_equal(back._engine.train_state_export()[:24], blob[:24]) and store.shape == back._engine.get_sample_store().shape
    # a pickle holds weights only
    loaded = GRU4Rec.loadmodel(p1)
    out = _run(lambda: loaded.fit_more(data.copy(), n_epochs=0, sample_store=STORE))
    assert 'No optimizer state to keep' in out
    assert not np.any(loaded._engine.get('Wy.acc')) and np.array_equal(loaded._engine.get('Wy'), before['Wy'])


@pytest.mark.parametrize('extra', [dict(logq=1.0, loss='cross-entropy', final_act='softmax'), dict(embedding=6), dict(constrained_embedding=True, sigma=0.3, init_as_normal=True)],
                         ids=['none_logq', 'embedding', 'constrained_normal'])
def test_fit_more_grows_the_catalogue(monkeypatch, tmp_path, extra):
    made = _install(monkeypatch)
    mk = dict(MK, n_epochs=1, **extra)
    gru = GRU4Rec(**mk)
    _run(lambda: gru.fit(_data(), sample_store=STORE))
    n_old = gru.n_items
    old_ids = gru.itemidmap.index.values.copy()
    before = _state(gru)
    gru.recommend_sessions([5], [old_ids[2]], k=3)                 # a session opened before the growth
    more = _data(seed=3, n_items=40, n_events=300)
    ids = np.concatenate([old_ids[:25], np.arange(10 ** 6, 10 ** 6 + 15)])
    more['ItemId'] = ids[more['ItemId'].values.astype(np.int64) % len(ids)]
    first_seen = more['ItemId'].values[np.sort(np.unique(more['ItemId'].values, return_index=True)[1])]
    new_ids = first_seen[first_seen >= 10 ** 6]
    n_add = len(new_ids)
    out = _run(lambda: gru.fit_more(more, n_epochs=0, sample_store=STORE))
    # recommend_sessions replaced the training engine by a scoring engine: the state is gone, and fit_more says so
    assert 'No optimizer state to keep' in out and 'Added %d new items' % n_add in out
    assert np.array_equal(gru.itemidmap.index.values, np.concatenate([old_ids, new_ids])) and gru.n_items == n_old + n_add
    assert np.array_equal(more['ItemIdx'].values, gru.itemidmap[more['ItemId'].values].values)
    eng = gru._engine
    rs = np.random.RandomState(42 + n_old)

    def rule(shape):
        sigma = extra.get('sigma') or np.sqrt(6.0 / (shape[0] + shape[1]))
        return (rs.randn(*shape) * sigma if extra.get('init_as_normal') else rs.rand(*shape) * sigma * 2 - sigma).astype(np.float32)
    if extra.get('embedding'):
        assert np.array_equal(eng.get('E')[n_old:], rule((n_add, 6)))
    elif not extra.get('constrained_embedding'):
        assert np.array_equal(eng.get('Wx0')[n_old:], np.hstack([rule((n_add, 10)) for _ in range(3)]))
    assert np.array_equal(eng.get('Wy')[n_old:], rule((n_add, 10))) and not np.any(eng.get('By')[n_old:])
    for n in gru._param_names():
        assert np.array_equal(eng.get(n)[:before[n].shape[0]], before[n]), n
    # sampling CDF and logQ support over the grown catalogue: items absent from the new frame have no mass
    counts = np.bincount(more['ItemIdx'].values, minlength=gru.n_items)
    cdf = np.cumsum(counts ** gru.sample_alpha) / np.sum(counts ** gru.sample_alpha)
    cdf[-1] = 1
    assert np.array_equal(eng.P, cdf.astype(np.float32)) and len(eng.P) == gru.n_items
    absent = counts == 0
    assert absent[:n_old].sum() >= 30 and not np.isin(eng.store, np.flatnonzero(absent)).any()
    if extra.get('logq'):
        assert np.array_equal(eng.m.P0, np.where(absent, 1.0, counts).astype(np.float32))
    # the session continues, old indices serve the same ids, a new item can be recommended
    assert gru.export_sessions()[0].tolist() == [5] and gru.export_sessions()[2][0].tolist() == [old_ids[2]]
    rec, _ = gru.recommend_sessions([5], [new_ids[0]], k=1, items=list(new_ids[:2]), exclude_seen=True)
    assert rec[0, 0] == new_ids[1]
    # training goes on over the grown catalogue, and the state it builds is kept by the next call
    out = _run(lambda: gru.fit_more(more, n_epochs=1, sample_store=STORE))
    assert len(LOSS_LINE.findall(out)) == 1
    out = _run(lambda: gru.fit_more(more, sample_store=STORE))
    assert 'Optimizer state kept' in out and len(LOSS_LINE.findall(out)) == 1
    assert all(e.closed for e in made[:-1]) and not made[-1].closed


def test_run_py_flags(monkeypatch, tmp_path, capsys):
    _install(monkeypatch)
    sys.path.insert(0, ROOT)
    import run
    train, more, ck, ck2 = (str(tmp_path / n) for n in ('train.tsv', 'more.tsv', 'm.npz', 'm2.npz'))
    d = _data()
    d.to_csv(train, sep='\t', index=False)
    d2 = _data(seed=4)
    d2['ItemId'] += 30
    d2.to_csv(more, sep='\t', index=False)
    ps = 'layers=10,batch_size=8,n_epochs=1,n_sample=16,loss=bpr-max,final_act=elu-0.5'
    run.main([train, '-ps', ps, '-ss', str(STORE), '--save_checkpoint', ck])
    out = capsys.readouterr().out
    assert 'Saving checkpoint to: ' + ck in out and os.path.exists(ck)
    run.main([more, '--load_checkpoint', ck, '--fit_more', '-ss', str(STORE), '--save_checkpoint', ck2])
    out = capsys.readouterr().out
    assert 'Loading checkpoint from file: ' + ck in out and 'Optimizer state kept' in out and 'Added' in out
    assert GRU4Rec.load_checkpoint(ck2).n_items > GRU4Rec.load_checkpoint(ck).n_items
    with pytest.raises(SystemExit):
        run.main([more, '--fit_more', '-ps', ps])
    with pytest.raises(SystemExit):
        run.main([more, '--load_checkpoint', ck, '-ps', ps])
