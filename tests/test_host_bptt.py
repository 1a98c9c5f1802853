"""CPU: truncated backpropagation through time (bptt > 1, DESIGN §3l) -- the float64 window oracle (tests/bptt_oracle.py) (one step is train_step; the
window gradient against torch.autograd of an independent restatement) and the Python surface of the option (set_params, pickles,
checkpoints, refusals before any engine is built, window-aligned ranges handed to the engine)."""
import json
import pickle

import numpy as np
import pytest
import torch

import gru4rec_oracle as orc
import bptt_oracle as bo
import oracle_engine
from gru4rec_b200 import _lib
from gru4rec_b200.gru4rec import GRU4Rec
from test_host_resume import ResumeOracleEngine, MK, STORE, _data, _run


# ---------------------------------------------------------------------------------------------------------------- the oracle
def _window(kind, B=4, T=6, n_items=40, S=7, seed=0):
    """a window of the epoch's schedule that ends in its compacted tail and holds a reset before its last step"""
    while True:             # the first seed from `seed` on whose schedule has both
        rs = np.random.RandomState(seed)
        lens = rs.randint(2, 7, 4 * B + 1)
        items = rs.randint(0, n_items, int(lens.sum())).astype(np.int64)
        offset = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        win = orc.build_train_schedule(items, offset, np.arange(len(lens)), B, S)[-T:]
        if not np.array_equal(win[-1]['slots'], np.arange(win[-1]['M'])) and (T == 1 or any(st['R'].any() for st in win[:-1])):
            break
        seed += 1
    for st in win:
        st['samples'] = rs.randint(0, n_items, S)
    return win


MODES = {
    'none_bprmax_elu': dict(loss='bpr-max', final_act='elu-0.5', layers=[6], bpreg=1.5),
    'embed_2layer_drop': dict(loss='top1-max', final_act='linear', layers=[6, 5], embedding=4, dropout_p_hidden=0.3, dropout_p_embed=0.25),
    'shared_xe_logq': dict(loss='cross-entropy', final_act='softmax', layers=[6], constrained_embedding=True, logq=1.0),
}


def _oracle(kw, n_items=40, B=4, S=7, dtype=np.float64):
    m = orc.OracleGRU4Rec(batch_size=B, n_sample=S, learning_rate=0.05, dtype=dtype, **kw)
    m.init(n_items)
    rs = np.random.RandomState(3)
    for h in m.H:
        h[:] = rs.randn(*h.shape) * 0.5
    m.By[:] = rs.randn(*m.By.shape) * 0.1
    m.P0 = rs.randint(1, 20, n_items).astype(dtype)
    return m


@pytest.mark.parametrize('mode', sorted(MODES))
def test_window_of_one_step_is_train_step(mode):
    win = _window(mode, T=1)
    for dtype in (np.float64, np.float32):
        a, b = _oracle(MODES[mode], dtype=dtype), _oracle(MODES[mode], dtype=dtype)
        st = win[0]
        c1 = a.train_step(st['X'], st['Y'], st['R'], samples=st['samples'], slots=st['slots'])
        c2 = bo.train_window(b, [st])
        assert c1 == c2[0]
        for name in ('Wy', 'By', 'E'):
            if getattr(a, name) is not None:
                np.testing.assert_array_equal(getattr(a, name), getattr(b, name))
        for name in ('Wx', 'Wh', 'Wrz', 'Bh', 'H'):
            for x, y in zip(getattr(a, name), getattr(b, name)):
                np.testing.assert_array_equal(x, y)
        for k in a.opt:
            np.testing.assert_array_equal(a.opt[k], b.opt[k])


def _act(name, x):
    if name == 'linear':
        return x
    if name == 'tanh':
        return torch.tanh(x)
    if name.startswith('elu-'):
        return torch.where(x >= 0, x, float(name.split('-')[1]) * (torch.exp(torch.clamp(x, max=0)) - 1))
    if name == 'softmax':
        return torch.softmax(x, dim=1)
    raise NotImplementedError(name)


def _loss(m, yhat):
    M = yhat.shape[0]
    ar = torch.arange(M)
    diag = yhat[ar, ar]
    if m.loss == 'cross-entropy':
        return (-torch.log(diag + 1e-24)).sum()
    hm = 1.0 - torch.eye(M, yhat.shape[1], dtype=yhat.dtype)
    Xh = yhat * hm
    e = torch.exp(Xh - Xh.max(dim=1, keepdim=True).values) * hm
    s = e / e.sum(dim=1, keepdim=True)
    if m.loss == 'bpr-max':
        A = (torch.sigmoid(diag[:, None] - yhat) * s).sum(1)
        return (-torch.log(A + 1e-24) + m.bpreg * (yhat * yhat * s).sum(1)).sum()
    if m.loss == 'top1-max':
        return (s * (torch.sigmoid(yhat - diag[:, None]) + torch.sigmoid(yhat * yhat))).sum()
    raise NotImplementedError(m.loss)


def _torch_window_grads(m, win):
    """the window's objective (sum of the step costs) restated in torch float64 from the model's weights and the steps' masks;
    gradients by autograd with the entering hidden state a constant"""
    P = {}
    nl = len(m.layers)
    for i in range(nl):
        for k in ('Wx', 'Wh', 'Wrz', 'Bh'):
            P['%s%d' % (k, i)] = torch.tensor(getattr(m, k)[i], requires_grad=True)
    P['Wy'] = torch.tensor(m.Wy, requires_grad=True)
    P['By'] = torch.tensor(m.By, requires_grad=True)
    if m.E is not None:
        P['E'] = torch.tensor(m.E, requires_grad=True)
    H = [torch.tensor(h) for h in m.H]
    step = m.step_count
    total = 0.0
    for st in win:
        M = len(st['X'])
        m.step_count = step
        masks = m.make_masks(M)
        step += 1
        X, Yc = torch.tensor(st['X']), torch.tensor(np.concatenate([st['Y'], st['samples']]))
        slots = torch.tensor(st['slots'])
        first = 0
        if m.constrained_embedding or m.embedding:
            x = (P['Wy'] if m.constrained_embedding else P['E'])[X]
            if 'e' in masks:
                x = x * torch.tensor(masks['e'])
        else:
            x, first = None, 1
        for i in range(nl):
            L = m.layers[i]
            vec = (P['Wx0'][X] + P['Bh0']) if i == 0 and first else x @ P['Wx%d' % i] + P['Bh%d' % i]
            Hs = H[i][slots]
            rz = torch.sigmoid(vec[:, L:] + Hs @ P['Wrz%d' % i])
            r, z = rz[:, :L], rz[:, L:]
            ht = _act(m.hidden_act, (Hs * r) @ P['Wh%d' % i] + vec[:, :L])
            h = (1 - z) * Hs + z * ht
            if ('h', i) in masks:
                h = h * torch.tensor(masks[('h', i)])
            H[i] = H[i].index_put((slots,), torch.where(torch.tensor(st['R'])[:, None], torch.zeros_like(h), h))
            x = h
        o = x @ P['Wy'][Yc].T + P['By'][Yc].reshape(-1)
        if m.logq:
            o = o - m.logq * torch.log(torch.tensor(np.concatenate([m.P0[st['Y']], m.P0[st['samples']] ** m.sample_alpha])))
        total = total + _loss(m, _act(m.final_act, o)) / m.batch_size
    names = sorted(P)
    return dict(zip(names, torch.autograd.grad(total, [P[n] for n in names])))


@pytest.mark.parametrize('mode', sorted(MODES))
def test_window_gradient_matches_autograd(mode):
    win = _window(mode)
    m = _oracle(MODES[mode])
    ref = _torch_window_grads(_oracle(MODES[mode]), win)
    bo.train_window(m, win)
    Cm, Gm = m.last_window
    nl = len(m.layers)
    got = {}
    for i in range(nl):
        for k in ('Wx', 'Wh', 'Wrz', 'Bh'):
            if Gm['d' + k][i] is not None:
                got['%s%d' % (k, i)] = Gm['d' + k][i]
    tables = {'Wy': np.zeros_like(m.Wy), 'By': np.zeros_like(m.By)}
    if Cm['mode'] == 'shared':
        np.add.at(tables['Wy'], Cm['Xc'], Gm['dSx'])
    else:
        in_name = 'E' if Cm['mode'] == 'embed' else 'Wx0'
        tables[in_name] = np.zeros_like(m.E if in_name == 'E' else m.Wx[0])
        np.add.at(tables[in_name], Cm['X'], Gm['dSx'])
        np.add.at(tables['Wy'], Cm['Y'], Gm['dSy'])
    np.add.at(tables['By'], Cm['Y'], Gm['dSBy'])
    got.update(tables)
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    for name, g in got.items():
        r = ref[name].numpy().reshape(np.shape(g))
        err = np.abs(g - r).max() / max(np.abs(r).max(), 1e-300)
        assert err <= 1e-10, '%s: %.3g' % (name, err)
    # the through-time terms are there: the same window without them (windows of one step) has other dense gradients
    m1 = _oracle(MODES[mode])
    m1.learning_rate = 0.0                        # the weights stay those the window started from
    acc = None
    for st in win:
        bo.train_window(m1, [st])
        g = m1.last_window[1]['dWh'][nl - 1]
        acc = g if acc is None else acc + g
    assert np.abs(acc - got['Wh%d' % (nl - 1)]).max() > 1e-6 * np.abs(acc).max()


# -------------------------------------------------------------------------------------------------------------- the surface
class _RangeEngine(ResumeOracleEngine):
    ranges = []

    def train_steps(self, sched, first=0, n=None):
        _RangeEngine.ranges.append((first, n, sched.n_steps))
        return super().train_steps(sched, first, n)


def _install(monkeypatch):
    made = []
    owner = []

    def make(cfg, device=0):
        assert int(cfg.bptt) == int(owner[-1].bptt)
        eng = _RangeEngine(cfg, oracle_engine.model_kwargs_of(owner[-1]), device)
        made.append(eng)
        return eng
    monkeypatch.setattr(_lib, 'Engine', make)
    real = GRU4Rec._make_config

    def make_config(self, *a, **k):
        owner.append(self)
        return real(self, *a, **k)
    monkeypatch.setattr(GRU4Rec, '_make_config', make_config)
    return made


def test_set_params_pickle_and_checkpoint_keep_bptt(monkeypatch, tmp_path):
    gru = GRU4Rec(**MK)
    assert gru.bptt == 1
    _run(lambda: gru.set_params(bptt='8'))
    assert gru.bptt == 8 and type(gru.bptt) is int
    _install(monkeypatch)
    gru.bptt = 4
    _run(lambda: gru.fit(_data(), sample_store=STORE))
    assert pickle.loads(pickle.dumps(gru)).bptt == 4
    old = pickle.loads(pickle.dumps(gru))
    del old.__dict__['bptt']                      # a pickle written before the option existed
    assert pickle.loads(pickle.dumps(old)).bptt == 1
    path = str(tmp_path / 'c.npz')
    gru.save_checkpoint(path)
    assert GRU4Rec.load_checkpoint(path).bptt == 4
    with np.load(path, allow_pickle=False) as z:
        arrays = {k: z[k] for k in z.files}
    meta = json.loads(str(arrays['meta']))
    del meta['engine']['bptt']
    arrays['meta'] = np.array(json.dumps(meta))
    old_path = str(tmp_path / 'old.npz')
    np.savez(old_path, **arrays)
    assert GRU4Rec.load_checkpoint(old_path).bptt == 1


@pytest.mark.parametrize('case', ['range', 'cpu_store', 'world'])
def test_refusals_come_before_any_engine(monkeypatch, case):
    made = _install(monkeypatch)
    gru = GRU4Rec(**MK)
    gru.bptt = 65 if case == 'range' else 4
    if case == 'world':
        monkeypatch.setattr(GRU4Rec, '_world', staticmethod(lambda: (2, 0)))
    with pytest.raises(ValueError if case == 'range' else NotImplementedError):
        _run(lambda: gru.fit(_data(), sample_store=STORE, store_type='cpu' if case == 'cpu_store' else 'gpu'))
    assert made == []


def test_fit_hands_the_engine_window_aligned_ranges(monkeypatch, tmp_path):
    _install(monkeypatch)
    _RangeEngine.ranges = []
    gru = GRU4Rec(**MK)
    gru.bptt = 4
    _run(lambda: gru.fit(_data(), sample_store=STORE))
    gru2 = GRU4Rec(**MK)
    gru2.bptt = 4
    _run(lambda: gru2.fit_resumable(_data(), str(tmp_path / 'r.npz'), 8, sample_store=STORE))
    assert len(_RangeEngine.ranges) > 4
    for first, n, total in _RangeEngine.ranges:
        assert first % 4 == 0 and (n % 4 == 0 or first + n == total), (first, n, total)


def test_fit_resumable_rejects_a_misaligned_interval(monkeypatch, tmp_path):
    made = _install(monkeypatch)
    gru = GRU4Rec(**MK)
    gru.bptt = 4
    with pytest.raises(ValueError):
        gru.fit_resumable(_data(), str(tmp_path / 'r.npz'), 6, sample_store=STORE)
    assert made == []
