"""CPU: the per-element float64 bound of a full-softmax step (full_softmax=True, DESIGN §3n; tests/full_softmax_oracle.py,
full_step_reference / row_update_bounds) can be met by float32 and has teeth.

At the RSC15 XE-shared shape (37,483 items, L 100, B 32, Adagrad + momentum) and at a 5,000-item shared Adagrad case with
dropout, each from random init (every lane's softmax nearly uniform) and at a trained-like spread (Wy / By scaled so that each
lane's scores spread over about 6-8):
- it can be met: the oracle itself at float32, and a float32 emulation of the device's step (3xTF32 scores from hi / lo splits,
  per 64-item tile max / sum-exp merged in order, dL/do as fac (p - [j = t]) / B), meet the bound on every element of every
  Wy / By row update and its optimizer state, and on dvec / dSx per lane;
- it has teeth: each planted error below misses it somewhere, and the report names the check that caught it."""
import copy

import numpy as np
import pytest

import gru4rec_oracle as orc
import full_softmax_oracle as fso


def _mk(L, B, **kw):
    mk = dict(layers=[L], batch_size=B, n_sample=2048, loss='cross-entropy', final_act='softmax', adapt=None, learning_rate=0.5,
              momentum=0.0)
    mk.update(kw)
    return mk


CASES = {
    'rsc15_xe_shared': (_mk(100, 32, constrained_embedding=True, dropout_p_hidden=0.4, adapt='adagrad', learning_rate=0.2,
                            momentum=0.2, bpreg=0.0), 37483),
    'shared_xe_adagrad_drop': (_mk(64, 32, constrained_embedding=True, dropout_p_hidden=0.3, dropout_p_embed=0.2, adapt='adagrad',
                                   learning_rate=0.05, momentum=0.3, lmbd=1e-3), 5000),
}
SPREADS = ('random', 'trained')
F32 = np.float32


def _f32_values(a):
    return np.asarray(a, F32).astype(np.float64)


def _with_dtype(m, dt):
    """a copy of oracle m with every array in dtype dt"""
    c = copy.deepcopy(m)
    c.dtype = dt
    for k, v in vars(c).items():
        if isinstance(v, np.ndarray) and v.dtype.kind == 'f':
            setattr(c, k, v.astype(dt))
        elif isinstance(v, list) and v and isinstance(v[0], np.ndarray):
            setattr(c, k, [a.astype(dt) for a in v])
    c.opt = {k: v.astype(dt) for k, v in c.opt.items()}
    return c


def _setup(name, spread):
    """float64 oracle holding float32 values (weights, hidden state, optimizer state in a trained model's range) and one step
    (X, Y, R) with a duplicated input and a target that is another lane's input"""
    mk, n = CASES[name]
    rs = np.random.RandomState(0)
    m = orc.OracleGRU4Rec(dtype=np.float64, **mk)
    m.init(n)
    for h in m.H:
        h[:] = rs.randn(*h.shape) * 0.5
    for b in m.Bh:
        b[:] = rs.randn(*b.shape) * 0.1
    m.By[:] = rs.randn(*m.By.shape) * 0.1
    B = mk['batch_size']
    X, Y, R = rs.randint(0, n, B), rs.randint(0, n, B), rs.rand(B) < 0.2
    X[1] = X[0]; Y[2] = X[3]
    if spread == 'trained':
        for _ in range(2):      # the input rows are Wy rows too: scale twice so that the lanes' score std settles near 1.5
            _, C = fso.forward_full(m, X, B, R=R, masks=m.make_masks(B), H=[h[:B] for h in m.H])
            f = 1.5 / C['o'].std(axis=1).mean()
            m.Wy *= f; m.By *= f
    m.init_opt_state()
    rs2 = np.random.RandomState(2)
    for pname in ['Wx0', 'Wh0', 'Wrz0', 'Bh0', 'Wy', 'By']:
        p = m.Wy if pname == 'Wy' else m.By if pname == 'By' else getattr(m, pname[:-1])[0]
        m.opt[(pname, 'acc')] = 10.0 ** rs2.uniform(-4, -2, p.shape)
        m.opt[(pname, 'vel')] = rs2.randn(*p.shape) * 1e-3
    for lst in (m.Wx, m.Wh, m.Wrz, m.Bh, m.H):
        for a in lst:
            a[:] = _f32_values(a)
    m.Wy, m.By = _f32_values(m.Wy), _f32_values(m.By)
    m.opt = {k: _f32_values(v) for k, v in m.opt.items()}
    return m, (X, Y, R)


def _tf32(x):
    """round to TF32 (10 explicit mantissa bits), to nearest"""
    u = np.ascontiguousarray(x, F32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(F32)


def _scores(y, Wy, By, kind):
    if kind == '3xtf32':
        yh, wh = _tf32(y), _tf32(Wy)
        yl, wl = _tf32(y - yh), _tf32(Wy - wh)
        return yh @ wh.T + (yh @ wl.T + yl @ wh.T) + By
    if kind == '1xtf32':
        return _tf32(y) @ _tf32(Wy).T + By
    return y @ Wy.T + By


def _device_do(m, o, Y, drop_tile=None, swap=False):
    """dL/do as the device forms it in float32: per 64-item tile max / sum-exp, the tiles merged in order, the target's
    probability, fac (p - [j = t]) / B"""
    M, I = o.shape
    T = -(-I // 64)
    op = np.full((M, T * 64), -np.inf, F32)
    op[:, :I] = o
    t = op.reshape(M, T, 64)
    mt = t.max(axis=2)
    Zt = np.exp(t - mt[:, :, None]).sum(axis=2, dtype=F32)
    if drop_tile is not None:
        Zt[:, drop_tile] = 0
    mx = mt.max(axis=1)
    Z = (Zt * np.exp(mt - mx[:, None])).sum(axis=1, dtype=F32)
    ar = np.arange(M)
    p = np.exp(o - mx[:, None]) / Z[:, None]
    pt = np.exp(o[ar, Y] - mx) / Z
    fac = pt / (pt + F32(orc.EPS_LOG)) if m.loss == 'cross-entropy' else np.ones(M, F32)
    Yt = np.array(Y)
    if swap:
        Yt[[0, 1]] = Yt[[1, 0]]
    tt = np.zeros_like(p)
    tt[ar, Yt] = 1
    return (fac[:, None] * (p - tt) * F32(1.0 / m.batch_size)).astype(F32)


def _device_like(m, X, Y, R, scores='3xtf32', drop_tile=None, swap=False, grad=None, after=None):
    """one full step of the float32 oracle m with the device's score and dL/do arithmetic; `grad(G)` edits the gradients before
    the update, `after(m)` the tables after it.  Returns (y, G)."""
    M = len(X)
    C = fso.forward_full(m, X, M, R=R, masks=m.make_masks(M), H=[h[:M] for h in m.H])[1]
    y = C['y_last']
    do = _device_do(m, _scores(y, m.Wy, m.By.reshape(-1), scores), np.asarray(Y), drop_tile, swap)
    G = dict(dSy=do.T @ y, dSBy=do.sum(axis=0).reshape(-1, 1))
    fso.gru_backward(m, C, do @ m.Wy, G)
    if grad:
        grad(G)
    m.apply_updates(C, G, M)
    if after:
        after(m)
    return y, G


def judge(m64, step, before, after, y, G32):
    """worst bound ratio of every check: the update of Wy / By and of each optimizer state tensor (row by row, one fp32 rounding
    per applied update), dvec per layer and dSx per lane"""
    X, Y, R = step
    C, G, E = fso.full_step_reference(m64, X, Y, R, y)
    out = {}

    def table(m, k):
        n, _, s = k.partition('.')
        return (m.Wy if n == 'Wy' else m.By) if not s else m.opt[(n, s)]
    for lo, hi, cnt, rows in fso.row_update_bounds(m64, C, G, E):
        for k, (_, ref1, allow) in rows.items():
            a0 = np.asarray(table(before, k)[lo:hi], np.float64)
            a1 = np.asarray(table(after, k)[lo:hi], np.float64)
            r0 = np.asarray(table(m64, k)[lo:hi])
            ulp = cnt.reshape(-1, 1) * 2.0 ** -23 * (np.abs(a0) + np.abs(a1))
            out[k + ' update'] = max(out.get(k + ' update', 0.0), fso.bound_ratio(a1 - a0, ref1 - r0, allow + ulp))
    for i, dv in enumerate(G32['dvec']):
        out['dvec%d' % i] = fso.bound_ratio(dv, G['dvec'][i], E['dvec'][i])
    if C['mode'] != 'none':
        out['dSx'] = fso.bound_ratio(G32['dSx'], G['dSx'], E['dSx'])
    return out


_CACHE = {}


def _base(name, spread):
    if (name, spread) not in _CACHE:
        m, step = _setup(name, spread)
        _CACHE[(name, spread)] = (m, _with_dtype(m, F32), step)
    return _CACHE[(name, spread)]


def _run(name, spread, how, **kw):
    m64, m32, step = _base(name, spread)
    m = copy.deepcopy(m32)
    if how == 'oracle':
        fso.train_step_full(m, *step)
        y, G = m.last_cache['y_last'], m.last_grads
    else:
        y, G = _device_like(m, *step, **kw)
    return judge(m64, step, m32, m, y, G)


def _fmt(r):
    return ', '.join('%s %.3g' % kv for kv in sorted(r.items(), key=lambda kv: -kv[1]))


PARAMS = [(n, s) for n in CASES for s in SPREADS]


@pytest.mark.parametrize('name,spread', PARAMS, ids=['%s-%s' % p for p in PARAMS])
def test_bound_is_met_by_float32(name, spread):
    """the float32 oracle and the float32 emulation of the device's 3xTF32 step meet the bound on every element; the oracle with
    a margin of 2 at least"""
    for how in ('oracle', 'device 3xTF32'):
        r = _run(name, spread, how)
        worst = max(r.values())
        print('%s %s, %s: worst bound ratio %.3g (%s)' % (name, spread, how, worst, _fmt(r)))
        assert worst <= (0.5 if how == 'oracle' else 1.0), '%s: %s' % (how, _fmt(r))


def _nontarget(n, Y):
    k = np.ones(n, bool)
    k[np.asarray(Y)] = False
    return k


def _scale_nontarget(f):
    def grad(G):
        nt = _nontarget(len(G['dSBy']), _STEP[0][1])
        G['dSy'][nt] *= F32(f)
        G['dSBy'][nt] *= F32(f)
    return dict(grad=grad)


def _keep_tile(lo, hi):
    def after(m):
        m0 = _STEP[1]
        m.Wy[lo:hi], m.By[lo:hi] = m0.Wy[lo:hi], m0.By[lo:hi]
        for k in m.opt:
            if k[0] in ('Wy', 'By'):
                m.opt[k][lo:hi] = m0.opt[k][lo:hi]
    return dict(after=after)


def _keep_nontarget_acc():
    def after(m):
        m0 = _STEP[1]
        nt = _nontarget(len(m.By), _STEP[0][1])
        for n in ('Wy', 'By'):
            m.opt[(n, 'acc')][nt] = m0.opt[(n, 'acc')][nt]
    return dict(after=after)


_STEP = [None, None]      # (step, float32 state before it) of the mutant being run
MUTANTS = {
    'non-target rows x (1 + 1e-4)': lambda: _scale_nontarget(1 + 1e-4),
    '1xTF32 scores': lambda: dict(scores='1xtf32'),
    'one 64-item tile not updated': lambda: _keep_tile(1024, 1088),
    'non-target acc not updated': _keep_nontarget_acc,
    "two lanes' targets swapped in dL/do": lambda: dict(swap=True),
    "merge drops one tile's sum-exp": lambda: dict(drop_tile=5),
}
MPARAMS = [(n, s, k) for n, s in PARAMS for k in MUTANTS]


@pytest.mark.parametrize('name,spread,mutant', MPARAMS, ids=['%s-%s-%s' % p for p in MPARAMS])
def test_bound_has_teeth(name, spread, mutant):
    """each planted error in the 3xTF32 emulation misses the bound; the report names the checks that caught it"""
    m64, m32, step = _base(name, spread)
    _STEP[:] = [step, m32]
    r = _run(name, spread, 'device', **MUTANTS[mutant]())
    caught = {k: v for k, v in r.items() if v > 1.0}
    print('%s %s, planted %r: caught by %s' % (name, spread, mutant, _fmt(caught) if caught else 'nothing'))
    assert caught, 'the planted error %r meets the bound: %s' % (mutant, _fmt(r))
