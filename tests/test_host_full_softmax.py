"""CPU: full-softmax training (full_softmax=True, DESIGN §3n) -- the float64 restatement (tests/full_softmax_oracle.py) against
central finite differences and scipy's logsumexp, and the surface of the option: set_params, pickles, checkpoints, refusals before
any engine is built (and at the C ABI), the engine configuration fit() asks for, and the C99 caller of the new field."""
import ctypes
import json
import os
import pickle
import shutil
import subprocess

import numpy as np
import pytest
from scipy.special import logsumexp

import gru4rec_oracle as orc
import full_softmax_oracle as fso
import oracle_engine
from gru4rec_b200 import _lib
from gru4rec_b200.gru4rec import GRU4Rec
from test_host_resume import ResumeOracleEngine, STORE, _data, _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODES = {
    'none': dict(layers=[5]),
    'embed_2layer': dict(layers=[5, 4], embedding=3),
    'shared': dict(layers=[5], constrained_embedding=True),
}
LOSSES = {'xe': ('cross-entropy', 'softmax'), 'xe_logit': ('xe_logit', 'softmax_logit')}


def _oracle(mode, loss, n_items=13, B=4, drop=True):
    kw = dict(MODES[mode])
    if drop:
        kw.update(dropout_p_hidden=0.3, dropout_p_embed=0.25 if mode != 'none' else 0.0)
    m = orc.OracleGRU4Rec(loss=LOSSES[loss][0], final_act=LOSSES[loss][1], batch_size=B, n_sample=7, logq=1.0, dtype=np.float64, **kw)
    m.init(n_items)
    rs = np.random.RandomState(3)
    for h in m.H:
        h[:] = rs.randn(*h.shape)
    m.By[:] = rs.randn(*m.By.shape) * 0.3
    m.Wy *= 3.0
    m.P0 = rs.randint(1, 20, n_items).astype(np.float64)
    return m


def _params(m):
    out = [('Wx%d' % i, m.Wx[i]) for i in range(len(m.layers))] + [('Wh%d' % i, m.Wh[i]) for i in range(len(m.layers))]
    out += [('Wrz%d' % i, m.Wrz[i]) for i in range(len(m.layers))] + [('Bh%d' % i, m.Bh[i]) for i in range(len(m.layers))]
    out += [('Wy', m.Wy), ('By', m.By)] + ([('E', m.E)] if m.E is not None else [])
    return out


def _full_grads(m, C, G):
    """the gradient of the cost wrt every parameter as a dense array (row gradients scattered onto their tables)"""
    nl = len(m.layers)
    g = {}
    for i in range(nl):
        g['Wh%d' % i], g['Wrz%d' % i], g['Bh%d' % i] = G['dWh'][i], G['dWrz'][i], G['dBh'][i]
        g['Wx%d' % i] = G['dWx'][i] if G['dWx'][i] is not None else np.zeros_like(m.Wx[i])
    g['Wy'] = G['dSy'].copy()
    g['By'] = G['dSBy'].copy()
    if C['mode'] == 'shared':
        np.add.at(g['Wy'], C['X'], G['dSx'])
    elif C['mode'] == 'embed':
        g['E'] = np.zeros_like(m.E)
        np.add.at(g['E'], C['X'], G['dSx'])
    else:
        np.add.at(g['Wx0'], C['X'], G['dSx'])
    return g


@pytest.mark.parametrize('loss', sorted(LOSSES))
@pytest.mark.parametrize('mode', sorted(MODES))
def test_gradients_against_finite_differences(mode, loss):
    """backward_full's gradient of every parameter element against float64 central differences of the cost, with dropout,
    a reset lane and a compacted tail (M = 3 lanes at physical slots 3, 0, 2 of B = 4), a duplicated input and an input that is
    also a target"""
    m = _oracle(mode, loss)
    X, Y, R = np.array([4, 4, 11]), np.array([7, 4, 0]), np.array([False, True, False])
    slots = np.array([3, 0, 2])
    M = len(X)
    masks = m.make_masks(M)
    H = [h[slots] for h in m.H]

    def cost():
        _, C = fso.forward_full(m, X, M, R=R, masks=masks, H=H)
        return fso.backward_full(m, C, M, Y)[0]
    _, C = fso.forward_full(m, X, M, R=R, masks=masks, H=H)
    c0, G = fso.backward_full(m, C, M, Y)
    grads = _full_grads(m, C, G)
    eps = 1e-6
    for name, p in _params(m):
        fd = np.zeros(p.shape)
        for idx in np.ndindex(p.shape):
            old = p[idx]
            p[idx] = old + eps; cp = cost()
            p[idx] = old - eps; cm = cost()
            p[idx] = old
            fd[idx] = (cp - cm) / (2 * eps)
        np.testing.assert_allclose(grads[name].reshape(p.shape), fd, rtol=1e-5, atol=1e-8, err_msg=name)
    assert abs(cost() - c0) == 0.0


@pytest.mark.parametrize('loss', sorted(LOSSES))
def test_cost_against_logsumexp(loss):
    """the cost is the mean over batch_size of logsumexp(o_b) - o_b[Y_b] over the catalogue; logq is not applied"""
    m = _oracle('shared', loss, n_items=50, B=6, drop=False)
    X, Y = np.array([1, 2, 3, 4, 5]), np.array([9, 2, 40, 0, 49])
    _, C = fso.forward_full(m, X, len(X), masks={}, H=[h[:len(X)] for h in m.H])
    c, _ = fso.backward_full(m, C, len(X), Y)
    o = C['y_last'] @ m.Wy.T + m.By.reshape(-1)
    ref = np.sum(logsumexp(o, axis=1) - o[np.arange(len(X)), Y]) / m.batch_size
    assert abs(c - ref) <= 1e-12 * abs(ref)


def test_train_step_full_updates_every_row_and_ignores_logq():
    """every Wy / By row moves; logq, n_sample and sample_alpha make no difference"""
    a = _oracle('shared', 'xe')
    b = _oracle('shared', 'xe')
    b.logq, b.n_sample, b.sample_alpha = 0.0, 2048, 0.1
    Wy0 = a.Wy.copy()
    X, Y, R = np.array([1, 2, 1]), np.array([3, 1, 12]), np.array([False, False, True])
    ca = fso.train_step_full(a, X, Y, R)
    cb = fso.train_step_full(b, X, Y, R)
    assert ca == cb and np.array_equal(a.Wy, b.Wy) and np.array_equal(a.By, b.By)
    assert (a.Wy != Wy0).any(axis=1).all()


# -------------------------------------------------------------------------------------------------------------- the surface
MK = dict(loss='cross-entropy', final_act='softmax', layers=[10], batch_size=8, n_epochs=2, n_sample=16, momentum=0.1, dropout_p_hidden=0.2)


class _FullOracleEngine(ResumeOracleEngine):
    """the engine double, training every step of a full_softmax configuration with the restatement"""
    def train_steps(self, sched, first=0, n=None):
        if not int(self.cfg.full_softmax):
            return super().train_steps(sched, first, n)
        e = self._export(sched)
        n = sched.n_steps - first if n is None else n
        costs = np.empty(n, dtype=np.float32)
        for j, k in enumerate(range(first, first + n)):
            M = int(e['M'][k])
            costs[j] = fso.train_step_full(self.m, e['X'][k, :M], e['Y'][k, :M], (e['F'][k, :M] & 1).astype(bool),
                                           slots=e['slots'][k, :M].astype(np.int64))
        return costs


def _install(monkeypatch):
    made, owner = [], []

    def make(cfg, device=0):
        assert int(cfg.full_softmax) == int(owner[-1].full_softmax)
        made.append(cfg)
        return _FullOracleEngine(cfg, oracle_engine.model_kwargs_of(owner[-1]), device)
    monkeypatch.setattr(_lib, 'Engine', make)
    real = GRU4Rec._make_config

    def make_config(self, *a, **k):
        owner.append(self)
        return real(self, *a, **k)
    monkeypatch.setattr(GRU4Rec, '_make_config', make_config)
    return made


def test_set_params_pickle_and_checkpoint_keep_full_softmax(monkeypatch, tmp_path):
    gru = GRU4Rec(**MK)
    assert gru.full_softmax is False
    out = _run(lambda: gru.set_params(full_softmax='True'))
    assert gru.full_softmax is True and 'full_softmax' in out
    _run(lambda: gru.set_params(full_softmax='0'))
    assert gru.full_softmax is False
    made = _install(monkeypatch)
    gru.full_softmax = True
    out = _run(lambda: gru.fit(_data(), sample_store=STORE))
    assert out.count('Full softmax') == 1 and 'sample store' not in out
    assert made and all(int(c.full_softmax) == 1 and int(c.sample_store) == 0 for c in made)
    assert pickle.loads(pickle.dumps(gru)).full_softmax is True
    old = pickle.loads(pickle.dumps(gru))
    del old.__dict__['full_softmax']              # a pickle written before the option existed
    assert pickle.loads(pickle.dumps(old)).full_softmax is False
    path = str(tmp_path / 'c.npz')
    gru.save_checkpoint(path)
    assert GRU4Rec.load_checkpoint(path).full_softmax is True
    with np.load(path, allow_pickle=False) as z:
        arrays = {k: z[k] for k in z.files}
    meta = json.loads(str(arrays['meta']))
    del meta['engine']['full_softmax']
    arrays['meta'] = np.array(json.dumps(meta))
    old_path = str(tmp_path / 'old.npz')
    np.savez(old_path, **arrays)
    assert GRU4Rec.load_checkpoint(old_path).full_softmax is False


def test_scoring_engine_is_not_full(monkeypatch):
    """the scoring engine a trained model builds for evaluate_gpu / predict_next_batch trains nothing: full_softmax stays 0"""
    gru = GRU4Rec(**MK)
    gru.full_softmax = True
    gru.n_items = 30
    assert int(gru._make_config(0, 16, training=False, single=True).full_softmax) == 0
    assert int(gru._make_config(0, 0, training=True, single=True).full_softmax) == 1


@pytest.mark.parametrize('case', ['bpr_max', 'xe_with_linear', 'smoothing', 'grad_cap', 'bptt', 'world'])
def test_refusals_come_before_any_engine(monkeypatch, case):
    made = _install(monkeypatch)
    gru = GRU4Rec(**MK)
    gru.full_softmax = True
    if case == 'bpr_max':
        gru.loss, gru.final_act = 'bpr-max', 'elu-0.5'
    elif case == 'xe_with_linear':
        gru.final_act = 'linear'
    elif case == 'smoothing':
        gru.smoothing = 0.1
    elif case == 'grad_cap':
        gru.grad_cap = 1.0
    elif case == 'bptt':
        gru.bptt = 4
    else:
        monkeypatch.setattr(GRU4Rec, '_world', staticmethod(lambda: (2, 0)))
    with pytest.raises(NotImplementedError):
        _run(lambda: gru.fit(_data(), sample_store=STORE))
    assert made == []


def _cfg(**kw):
    mk = dict(loss='cross-entropy', final_act='softmax', layers=[16], batch_size=8, n_sample=32)
    mk.update({k: v for k, v in kw.items() if k in ('loss', 'final_act', 'smoothing', 'grad_cap')})
    cfg = _lib.make_config(500, mk, sample_store=32 * 10, full_softmax=True, bptt=kw.get('bptt', 1))
    cfg.world_size = kw.get('world_size', 1)
    return cfg


def _workspace(cfg):
    lib = _lib.load()
    n = ctypes.c_size_t()
    return lib.g4r_workspace_bytes(ctypes.byref(cfg), ctypes.byref(n)), n.value


@pytest.mark.parametrize('kw', [dict(loss='bpr-max', final_act='elu-0.5'), dict(smoothing=0.1), dict(grad_cap=1.0), dict(bptt=4),
                                dict(world_size=2)], ids=['bpr_max', 'smoothing', 'grad_cap', 'bptt', 'world'])
def test_abi_refuses_what_full_softmax_does_not_cover(kw):
    assert _workspace(_cfg(**kw))[0] == _lib.G4R_ERR_INVALID


def test_abi_workspace_has_no_sample_store():
    """the sample store is not allocated, so its size makes no difference; the [n_items x lanes] dL/do buffer grows with the
    catalogue"""
    rc, full = _workspace(_cfg())
    assert rc == 0
    for store in (0, 32 * 1000):
        cfg = _cfg(); cfg.sample_store = store
        assert _workspace(cfg) == (0, full)
    cfg = _cfg(); cfg.n_items = 1500
    rc, bigger = _workspace(cfg)
    assert rc == 0 and bigger - full >= 1000 * 8 * 4


C_SRC = r'''
#include <stddef.h>
#include <stdio.h>
#include "g4r.h"

int main(void) {
  g4r_config c;
  int64_t (*steps)(const g4r_handle*) = g4r_full_steps;
  if (steps(NULL) != 0) return 1;
  printf("ok %d %d %d\n", (int)offsetof(g4r_config, bptt), (int)offsetof(g4r_config, full_softmax), (int)sizeof c);
  return 0;
}
'''


def test_c99_caller_and_struct_offset(tmp_path):
    """full_softmax is appended after bptt: a C99 caller builds, and its offsets agree with the ctypes mirror"""
    gcc = shutil.which('gcc') or shutil.which('cc')
    if gcc is None:
        pytest.skip('no C compiler')
    inc, libdir = os.path.join(ROOT, 'include'), os.path.join(ROOT, 'gru4rec_b200')
    src = tmp_path / 'caller.c'
    src.write_text(C_SRC)
    exe = str(tmp_path / 'caller')
    cuda_lib = '/usr/local/cuda/lib64'
    r = subprocess.run([gcc, '-std=c99', '-Wall', '-Wextra', '-pedantic', '-Werror', '-I' + inc, str(src), '-L' + libdir, '-lg4r',
                        '-Wl,-rpath,' + libdir, '-L' + cuda_lib, '-Wl,-rpath,' + cuda_lib, '-o', exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    _, bptt_off, full_off, size = r.stdout.split()
    assert int(bptt_off) == _lib.G4RConfig.bptt.offset and int(full_off) == _lib.G4RConfig.full_softmax.offset == int(bptt_off) + 4
    assert int(size) == ctypes.sizeof(_lib.G4RConfig)


def test_engine_refuses_a_workspace_that_does_not_fit(monkeypatch):
    """Engine() refuses a full-softmax workspace larger than the free device memory, naming the bytes it needs, before it
    allocates anything or creates a handle"""
    import torch
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda device=None: (1 << 20, 80 << 30))
    monkeypatch.setattr(torch, 'empty', lambda *a, **k: pytest.fail('allocated a workspace that does not fit'))
    cfg = _cfg()
    cfg.n_items = 172000
    rc, need = _workspace(cfg)
    assert rc == 0 and need > 1 << 20
    with pytest.raises(NotImplementedError, match='%d bytes' % need):
        _lib.Engine(cfg)
