"""
TEST INFRASTRUCTURE ONLY -- CPU restatement (NumPy) of the GRU4Rec session-parallel training step.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import
this module, and only as the checker.  The product path (gru4rec_b200/) never imports it.

Pinning status: the reference (hidasib/GRU4Rec @ a4ed5fb) ships no tests and no golden vectors and
needs Theano, which is not installable here.  This restatement is pinned three ways (see
DESIGN.md "Oracle"): (1) against golden vectors produced by running the reference's own
gru4rec.py / evaluation.py graph-building code on top of oracle/theano_shim (a minimal
Theano-API emulator on torch autograd; generating script oracle/make_golden.py, fixtures in
tests/golden/); (2) hand-derived backward vs. torch.autograd of the forward; (3) float64 central
finite differences.  Theano's MRG31k3p streams, cuBLAS rounding and GPU scatter race winners remain
"parity unpinned" (no reference artefact exists for them).

Every function cites the reference file:line it follows (paths relative to /root/reference).
"""
import numpy as np

EPS_LOG = 1e-24


# --------------------------------------------------------------------------------------------
# activations (gru4rec.py:189-223)
# --------------------------------------------------------------------------------------------
def parse_act(name):
    """gru4rec.py:144-161 -> (kind, p1, p2)."""
    if name in ('linear', 'relu', 'tanh', 'softmax', 'softmax_logit'):
        return (name, 0.0, 0.0)
    if name.startswith('leaky-'):
        return ('leaky', float(name.split('-')[1]), 0.0)
    if name.startswith('elu-'):
        return ('elu', float(name.split('-')[1]), 0.0)
    if name.startswith('selu-'):
        p = [float(x) for x in name.split('-')[1:]]
        return ('selu', p[0], p[1])
    raise NotImplementedError


def act_fwd(act, X):
    kind, p1, p2 = act
    dt = X.dtype.type
    if kind == 'linear':
        return X
    if kind == 'relu':
        return np.maximum(X, dt(0))
    if kind == 'tanh':
        return np.tanh(X)
    if kind == 'leaky':
        return np.where(X >= 0, X, dt(p1) * X)
    if kind == 'elu':  # gru4rec.py:214-218
        return np.where(X >= 0, X, dt(p1) * (np.exp(np.minimum(X, 0)) - dt(1)))
    if kind == 'selu':  # gru4rec.py:208-213  (lmbd, alpha)
        return dt(p1) * np.where(X >= 0, X, dt(p2) * (np.exp(np.minimum(X, 0)) - dt(1)))
    if kind == 'softmax':  # gru4rec.py:193-195
        e = np.exp(X - X.max(axis=1, keepdims=True))
        return e / e.sum(axis=1, keepdims=True)
    if kind == 'softmax_logit':  # gru4rec.py:196-198
        Xm = X - X.max(axis=1, keepdims=True)
        return np.log(np.exp(Xm).sum(axis=1, keepdims=True)) - Xm
    raise NotImplementedError


def act_bwd(act, X, Yv, dY):
    """dL/dX given pre-activation X, output Yv=act(X) and dL/dY."""
    kind, p1, p2 = act
    dt = X.dtype.type
    if kind == 'linear':
        return dY
    if kind == 'relu':
        return dY * (X > 0)
    if kind == 'tanh':
        return dY * (dt(1) - Yv * Yv)
    if kind == 'leaky':
        return dY * np.where(X >= 0, dt(1), dt(p1))
    if kind == 'elu':
        return dY * np.where(X >= 0, dt(1), dt(p1) * np.exp(np.minimum(X, 0)))
    if kind == 'selu':
        return dY * dt(p1) * np.where(X >= 0, dt(1), dt(p2) * np.exp(np.minimum(X, 0)))
    if kind == 'softmax':
        return Yv * (dY - (dY * Yv).sum(axis=1, keepdims=True))
    if kind == 'softmax_logit':
        p = np.exp(-Yv)  # softmax(X)
        return -dY + p * dY.sum(axis=1, keepdims=True)
    raise NotImplementedError


def sigmoid(x):
    return (1.0 / (1.0 + np.exp(-x))).astype(x.dtype)


# --------------------------------------------------------------------------------------------
# losses (gru4rec.py:225-248); yhat is [M, N], the target of row i is column i (gpu_ops.py:15-27)
# each returns (loss_sum, dL/dyhat)
# --------------------------------------------------------------------------------------------
def softmax_neg(X):
    """gru4rec.py:199-203: diagonal zeroed before the max, masked again after exp."""
    dt = X.dtype.type
    hm = np.ones_like(X)
    m = X.shape[0]
    hm[np.arange(m), np.arange(m)] = 0
    Xh = X * hm
    e = np.exp(Xh - Xh.max(axis=1, keepdims=True)) * hm
    return e / e.sum(axis=1, keepdims=True), hm


def loss_and_grad(loss, yhat, M, n_sample, bpreg=1.0, smoothing=0.0):
    dt = yhat.dtype.type
    m, n = yhat.shape
    ar = np.arange(m)
    diag = yhat[ar, ar]
    g = np.zeros_like(yhat)
    if loss == 'cross-entropy':  # gru4rec.py:225-230
        if smoothing:
            n_out = M + n_sample
            c1 = dt(1.0 - (n_out / (n_out - 1)) * smoothing)
            c2 = dt(smoothing / (n_out - 1))
            L = np.sum(c1 * (-np.log(diag + dt(EPS_LOG))) + c2 * np.sum(-np.log(yhat + dt(EPS_LOG)), axis=1))
            g = -c2 / (yhat + dt(EPS_LOG))
            g[ar, ar] += -c1 / (diag + dt(EPS_LOG))
        else:
            L = np.sum(-np.log(diag + dt(EPS_LOG)))
            g[ar, ar] = -dt(1) / (diag + dt(EPS_LOG))
        return dt(L), g
    if loss == 'xe_logit':  # gru4rec.py:231-236
        if smoothing:
            n_out = M + n_sample
            c1 = dt(1.0 - (n_out / (n_out - 1)) * smoothing)
            c2 = dt(smoothing / (n_out - 1))
            L = np.sum(c1 * diag + c2 * np.sum(yhat, axis=1))
            g[:] = c2
            g[ar, ar] += c1
        else:
            L = np.sum(diag)
            g[ar, ar] = dt(1)
        return dt(L), g
    if loss == 'bpr':  # gru4rec.py:237-238
        d = diag[:, None] - yhat
        s = sigmoid(d)
        L = np.sum(-np.log(s))
        gd = -(dt(1) - s)          # dL/dd
        g = -gd
        g[ar, ar] += gd.sum(axis=1)
        return dt(L), g
    if loss == 'bpr-max':  # gru4rec.py:239-241
        s, hm = softmax_neg(yhat)
        d = diag[:, None] - yhat
        sg = sigmoid(d)
        A = np.sum(sg * s, axis=1)
        Q = np.sum(yhat * yhat * s, axis=1)
        L = np.sum(-np.log(A + dt(EPS_LOG)) + dt(bpreg) * Q)
        invA = dt(1) / (A + dt(EPS_LOG))
        dsg = sg * (dt(1) - sg)
        # dL/ds_ij (through both terms)
        dLds = -invA[:, None] * sg + dt(bpreg) * yhat * yhat
        # softmax backward on negatives (diagonal has s=0 so it drops out)
        ds_to_y = s * (dLds - np.sum(dLds * s, axis=1, keepdims=True))
        g = ds_to_y
        # direct terms: sigma(d_ij) with d = y_ii - y_ij, and y_ij^2
        g += -invA[:, None] * s * dsg * (-1)
        g += dt(bpreg) * 2 * yhat * s
        g[ar, ar] += np.sum(-invA[:, None] * s * dsg, axis=1)
        return dt(L), g
    if loss == 'top1':  # gru4rec.py:242-244
        # NB the reference subtracts a COLUMN (gpu_diag(..., keepdims=True), broadcastable (False, True), custom_theano_ops.py:39)
        # from the row-mean VECTOR, which broadcasts to an [M x M] matrix before T.sum: the loss -- and every gradient -- is
        # M times the per-row expression.  Pinned by tests/golden/top1_embed_selu.npz (the shim reproduces the broadcast).
        nn_ = dt(M + n_sample)
        a = sigmoid(yhat - diag[:, None])
        b = sigmoid(yhat * yhat)
        c = sigmoid(diag * diag)
        Mf = dt(m)
        L = Mf * np.sum(np.mean(a + b, axis=1) - c / nn_)
        da = a * (dt(1) - a) / dt(n)
        db = b * (dt(1) - b) * 2 * yhat / dt(n)
        g = da + db
        g[ar, ar] += -da.sum(axis=1) - c * (dt(1) - c) * 2 * diag / nn_
        return dt(L), Mf * g
    if loss == 'top1-max':  # gru4rec.py:245-248
        s, hm = softmax_neg(yhat)
        a = sigmoid(yhat - diag[:, None])
        b = sigmoid(yhat * yhat)
        T_ = a + b
        L = np.sum(s * T_)
        dLds = T_
        g = s * (dLds - np.sum(dLds * s, axis=1, keepdims=True))
        da = s * a * (dt(1) - a)
        g += da + s * b * (dt(1) - b) * 2 * yhat
        g[ar, ar] += -da.sum(axis=1)
        return dt(L), g
    raise NotImplementedError


# --------------------------------------------------------------------------------------------
# counter-hash RNG used for dropout masks (device and oracle share this definition; the reference
# uses Theano MRG streams here, gru4rec.py:295-299 -- parity unpinned, so masks are defined by us)
# --------------------------------------------------------------------------------------------
def _mix32(x):
    x = x.astype(np.uint32)
    x ^= x >> np.uint32(16)
    x = (x * np.uint32(0x7feb352d)).astype(np.uint32)
    x ^= x >> np.uint32(15)
    x = (x * np.uint32(0x846ca68b)).astype(np.uint32)
    x ^= x >> np.uint32(16)
    return x


def hash_uniform(seed, step, stream, n):
    """uniform [0,1) float32 with 24 random bits for element idx in [0,n)."""
    with np.errstate(over='ignore'):
        idx = np.arange(n, dtype=np.uint32)
        k = _mix32(np.array([np.uint32(seed) ^ (np.uint32(0x9E3779B9) * np.uint32(stream + 1))], dtype=np.uint32))
        k = _mix32(k + np.uint32(step))
        r = _mix32(k + idx)
    return (r >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def dropout_mask(seed, step, stream, shape, drop_p, dtype=np.float32):
    """mask/retain as in gru4rec.py:295-299 (binomial(p=retain) == uniform < retain)."""
    retain = np.float32(1.0 - drop_p)
    u = hash_uniform(seed, step, stream, int(np.prod(shape))).reshape(shape)
    return ((u < retain).astype(dtype) / dtype(retain)).astype(dtype)


STREAM_EMBED = 100


# --------------------------------------------------------------------------------------------
# K2: GpuBinarySearchSorted semantics (custom_theano_ops.py:318-349)
# --------------------------------------------------------------------------------------------
def searchsorted_k2(d, x):
    d = np.asarray(d)
    x = np.asarray(x)
    ld = d.shape[0]
    res = np.searchsorted(d, x, side='right').astype(np.int64)
    res = np.minimum(res, ld - 1)
    res[x > d[-1]] = ld
    res[x <= d[0]] = 0
    return res


def searchsorted_k2_loop(d, x):
    """literal transcription of the kernel's control flow (small inputs only)."""
    ld = len(d)
    out = np.zeros(len(x), dtype=np.int64)
    for i, val in enumerate(x):
        a, b = 0, ld - 1
        if val > d[b]:
            a = b = ld
        elif val <= d[0]:
            a = b = 0
        while b - a > 0:
            h = (a + b) // 2
            if val < d[h]:
                b = h
            else:
                a = h + 1
        out[i] = b
    return out


def sampling_cdf(supports, alpha):
    """gru4rec.py:543-545 (float64) then float32 cast at :556."""
    pop = np.asarray(supports, dtype=np.float64) ** alpha
    pop = pop.cumsum() / pop.sum()
    pop[-1] = 1
    return pop


# --------------------------------------------------------------------------------------------
# MRG31k3p as used by theano.sandbox.rng_mrg.MRG_RandomStreams (third-party, recalled; SURVEY
# Appendix B -- parity unpinned).  Used for the GPU sample store uniforms (gru4rec.py:559).
# --------------------------------------------------------------------------------------------
M1 = 2147483647
M2 = 2147462579
A1p72 = np.array([[1516919229, 758510237, 499121365], [1884998244, 1516919229, 335398200], [601897748, 1884998244, 358115744]], dtype=np.int64)
A2p72 = np.array([[1228857673, 1496414766, 954677935], [1133297478, 1407477216, 1496414766], [2002613992, 1639496704, 1407477216]], dtype=np.int64)
A1p134 = np.array([[1702500920, 1849582496, 1656874625], [828554832, 1702500920, 1512419905], [1143731069, 828554832, 102237247]], dtype=np.int64)
A2p134 = np.array([[796789021, 1464208080, 607337906], [1241679051, 1431130166, 1464208080], [1401213391, 1178684362, 1431130166]], dtype=np.int64)
MRG_NORM = np.float32(4.6566126e-10)


def _matvec_mod(A, v, m):
    # python ints to avoid int64 overflow (entries < 2^31, products < 2^62, sums of 3 < 2^64 -> use object)
    return np.array([sum(int(A[i, j]) * int(v[j]) for j in range(3)) % m for i in range(3)], dtype=np.int64)


def mrg_ff(state, A1, A2):
    s = np.asarray(state, dtype=np.int64)
    return np.concatenate([_matvec_mod(A1, s[:3], M1), _matvec_mod(A2, s[3:], M2)])


def mrg_next(s):
    """one MRG31k3p step on a [n,6] int64 state array; returns float32 uniforms (in place update)."""
    x11, x12, x13, x21, x22, x23 = [s[:, i].copy() for i in range(6)]
    y1 = ((x12 & 511) << 22) + (x12 >> 9) + ((x13 & 16777215) << 7) + (x13 >> 24)
    y1 = np.where(y1 >= M1, y1 - M1, y1)
    y1 = y1 + x13
    y1 = np.where(y1 >= M1, y1 - M1, y1)
    x13, x12, x11 = x12, x11, y1
    y1 = ((x21 & 65535) << 15) + 21069 * (x21 >> 16)
    y1 = np.where(y1 >= M2, y1 - M2, y1)
    y2 = ((x23 & 65535) << 15) + 21069 * (x23 >> 16)
    y2 = np.where(y2 >= M2, y2 - M2, y2)
    y2 = y2 + x23
    y2 = np.where(y2 >= M2, y2 - M2, y2)
    y2 = y2 + y1
    y2 = np.where(y2 >= M2, y2 - M2, y2)
    x23, x22, x21 = x22, x21, y2
    s[:, 0], s[:, 1], s[:, 2], s[:, 3], s[:, 4], s[:, 5] = x11, x12, x13, x21, x22, x23
    diff = np.where(x11 <= x21, x11 - x21 + M1, x11 - x21)
    return diff.astype(np.float32) * MRG_NORM


class MRGStreams:
    """MRG_RandomStreams(seed=12345) restatement: .uniform(n) takes a fresh block of substreams."""
    NSTREAMS = 60 * 256

    def __init__(self, seed=12345):
        self.rstate = np.array([seed] * 6, dtype=np.int64)

    def n_streams(self, n):
        r = n
        if r > 6:
            r = r // 6
        return min(r, self.NSTREAMS)

    def substreams(self, n_streams):
        st = np.zeros((n_streams, 6), dtype=np.int64)
        st[0] = self.rstate
        for i in range(1, n_streams):
            st[i] = mrg_ff(st[i - 1], A1p72, A2p72)
        self.rstate = mrg_ff(self.rstate, A1p134, A2p134)
        return st

    def uniform_from_state(self, st, n):
        ns = st.shape[0]
        out = np.empty(n, dtype=np.float32)
        pos = 0
        while pos < n:
            k = min(ns, n - pos)
            out[pos:pos + k] = mrg_next(st[:k])      # a stream only advances when it produces a sample
            pos += k
        return out


# --------------------------------------------------------------------------------------------
# session-parallel schedule (gru4rec.py:585-651)
# --------------------------------------------------------------------------------------------
def build_train_schedule(data_items, offset_sessions, session_idx_arr, batch_size, n_sample):
    """Literal restatement of the epoch loop.  Returns a list of steps; each step is a dict with
    X, Y (int64 [M]), R (bool [M]), M, slots (physical H row of each lane; the reference compacts H
    at gru4rec.py:647-651, which is equivalent to dropping entries from `slots`)."""
    steps = []
    n_sessions = len(offset_sessions) - 1
    iters = np.arange(batch_size)
    maxiter = iters.max()
    start = offset_sessions[session_idx_arr[iters]].astype(np.int64)   # IndexError if n_sessions < batch_size
    end = offset_sessions[session_idx_arr[iters] + 1].astype(np.int64)
    slots = np.arange(batch_size)
    finished = False
    while not finished:
        minlen = (end - start).min()
        out_idx = data_items[start]
        for i in range(minlen - 1):
            in_idx = out_idx
            out_idx = data_items[start + i + 1]
            reset = (start + i + 1 == end - 1)
            steps.append(dict(X=in_idx.copy(), Y=out_idx.copy(), R=reset.copy(), M=len(iters), slots=slots.copy()))
        start = start + minlen - 1
        finished_mask = (end - start <= 1)
        n_finished = finished_mask.sum()
        iters[finished_mask] = maxiter + np.arange(1, n_finished + 1)
        maxiter += n_finished
        valid_mask = (iters < n_sessions)
        n_valid = valid_mask.sum()
        if (n_valid == 0) or (n_valid < 2 and n_sample == 0):
            finished = True
            break
        mask = finished_mask & valid_mask
        sessions = session_idx_arr[iters[mask]]
        start[mask] = offset_sessions[sessions]
        end[mask] = offset_sessions[sessions + 1]
        iters = iters[valid_mask]
        start = start[valid_mask]
        end = end[valid_mask]
        slots = slots[valid_mask]
    return steps


def build_eval_schedule(test_items, offset_sessions, batch_size):
    """evaluation.py:90-139.  Z = lanes whose H is zeroed BEFORE the step (host-side zeroing at :136-139)."""
    steps = []
    n_sessions = len(offset_sessions) - 1
    iters = np.arange(batch_size)
    maxiter = iters.max()
    start = offset_sessions[iters].astype(np.int64)
    end = offset_sessions[iters + 1].astype(np.int64)
    slots = np.arange(batch_size)
    zero_next = np.zeros(batch_size, dtype=bool)
    finished = False
    while not finished:
        minlen = (end - start).min()
        out_idx = test_items[start]
        for i in range(minlen - 1):
            in_idx = out_idx
            out_idx = test_items[start + i + 1]
            steps.append(dict(X=in_idx.copy(), Y=out_idx.copy(), Z=zero_next.copy(), M=len(iters), slots=slots.copy()))
            zero_next[:] = False
        start = start + minlen - 1
        finished_mask = (end - start <= 1)
        n_finished = finished_mask.sum()
        iters[finished_mask] = maxiter + np.arange(1, n_finished + 1)
        maxiter += n_finished
        valid_mask = (iters < n_sessions)
        n_valid = valid_mask.sum()
        if n_valid == 0:
            finished = True
            break
        mask = finished_mask & valid_mask
        sessions = iters[mask]
        start[mask] = offset_sessions[sessions]
        end[mask] = offset_sessions[sessions + 1]
        zero_next = zero_next | mask
        iters = iters[valid_mask]
        start = start[valid_mask]
        end = end[valid_mask]
        slots = slots[valid_mask]
        zero_next = zero_next[valid_mask]
    return steps


# --------------------------------------------------------------------------------------------
# the model
# --------------------------------------------------------------------------------------------
class OracleGRU4Rec:
    """NumPy restatement of GRU4Rec (gru4rec.py:27-781) for the training / scoring hot path."""

    def __init__(self, loss='bpr-max', final_act='linear', hidden_act='tanh', layers=[100], n_epochs=10, batch_size=32,
                 dropout_p_hidden=0.0, dropout_p_embed=0.0, learning_rate=0.1, momentum=0.0, lmbd=0.0, embedding=0,
                 n_sample=2048, sample_alpha=0.75, smoothing=0.0, constrained_embedding=False, adapt='adagrad',
                 adapt_params=[], grad_cap=0.0, bpreg=1.0, logq=0.0, sigma=0.0, init_as_normal=False,
                 train_random_order=False, time_sort=True, dtype=np.float32, dropout_seed=0):
        self.loss = loss
        self.final_act = final_act
        self.hidden_act = hidden_act
        self.layers = list(layers)
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.dropout_p_hidden = dropout_p_hidden
        self.dropout_p_embed = dropout_p_embed
        self.learning_rate = learning_rate
        self.momentum = momentum
        self.lmbd = lmbd
        self.embedding = self.layers[0] if embedding == 'layersize' else embedding
        self.n_sample = n_sample
        self.sample_alpha = sample_alpha
        self.smoothing = smoothing
        self.constrained_embedding = constrained_embedding
        self.adapt = adapt
        self.adapt_params = adapt_params
        self.grad_cap = grad_cap
        self.bpreg = bpreg
        self.logq = logq
        self.sigma = sigma
        self.init_as_normal = init_as_normal
        self.train_random_order = train_random_order
        self.time_sort = time_sort
        self.dtype = dtype
        self.dropout_seed = dropout_seed
        self.fact = parse_act(final_act)
        self.hact = parse_act(hidden_act)
        self.step_count = 0
        self.P0 = None

    # ---- init (gru4rec.py:254-294) ----
    def init_matrix(self, shape):
        sigma = self.sigma if self.sigma != 0 else np.sqrt(6.0 / (shape[0] + shape[1]))
        if self.init_as_normal:
            return (np.random.randn(*shape) * sigma).astype(self.dtype)
        return (np.random.rand(*shape) * sigma * 2 - sigma).astype(self.dtype)

    def init(self, n_items):
        self.n_items = n_items
        np.random.seed(42)
        self.Wx, self.Wh, self.Wrz, self.Bh, self.H = [], [], [], [], []
        self.E = None
        if self.constrained_embedding:
            n_features = self.layers[-1]
        elif self.embedding:
            self.E = self.init_matrix((n_items, self.embedding))
            n_features = self.embedding
        else:
            n_features = n_items
        for i in range(len(self.layers)):
            nin = self.layers[i - 1] if i > 0 else n_features
            m = [self.init_matrix((nin, self.layers[i])) for _ in range(3)]
            self.Wx.append(np.hstack(m))
            self.Wh.append(self.init_matrix((self.layers[i], self.layers[i])))
            m2 = [self.init_matrix((self.layers[i], self.layers[i])) for _ in range(2)]
            self.Wrz.append(np.hstack(m2))
            self.Bh.append(np.zeros((self.layers[i] * 3,), dtype=self.dtype))
            self.H.append(np.zeros((self.batch_size, self.layers[i]), dtype=self.dtype))
        self.Wy = self.init_matrix((n_items, self.layers[-1]))
        self.By = np.zeros((n_items, 1), dtype=self.dtype)
        self.init_opt_state()

    def set_weights(self, **w):
        for k, v in w.items():
            if isinstance(v, list):
                setattr(self, k, [np.array(a, dtype=self.dtype) for a in v])
            elif v is not None:
                setattr(self, k, np.array(v, dtype=self.dtype))
        self.n_items = self.Wy.shape[0]
        self.init_opt_state()

    def init_opt_state(self):
        """Anonymous shared variables created inside adagrad()/RMSprop() (gru4rec.py:331,401,425)."""
        self.opt = {}
        self.step_count = 0

    def _state(self, name, like, slot):
        key = (name, slot)
        if key not in self.opt:
            self.opt[key] = np.zeros_like(like)
        return self.opt[key]

    # ---- dense adaptive scalers (gru4rec.py:300-381) ----
    def _adapt_dense(self, name, p, g):
        dt = self.dtype
        eps = dt(1e-6)
        if self.adapt == 'adagrad':
            acc = self._state(name, p, 'acc')
            acc += g * g
            return g / np.sqrt(acc + eps)
        if self.adapt == 'rmsprop':
            v1 = dt(self.adapt_params[0]); v2 = dt(1.0 - self.adapt_params[0])
            acc = self._state(name, p, 'acc')
            acc[...] = v1 * acc + v2 * g * g
            return g / np.sqrt(acc + eps)
        if self.adapt == 'adadelta':
            v1 = dt(self.adapt_params[0]); v2 = dt(1.0 - self.adapt_params[0])
            acc = self._state(name, p, 'acc'); upd = self._state(name, p, 'upd')
            acc[...] = v1 * acc + v2 * g * g
            gs = (upd + eps) / (acc + eps)
            upd[...] = v1 * upd + v2 * gs * g * g
            return g * np.sqrt(gs)
        if self.adapt == 'adam':
            v1 = dt(self.adapt_params[0]); v2 = dt(1.0 - self.adapt_params[0])
            v3 = dt(self.adapt_params[1]); v4 = dt(1.0 - self.adapt_params[1])
            acc = self._state(name, p, 'acc'); mg = self._state(name, p, 'meang'); ct = self._state(name, p, 'countt')
            acc[...] = v3 * acc + v4 * g * g
            mg[...] = v1 * mg + v2 * g
            ct += 1
            return (mg / (1 - v1 ** ct)) / (np.sqrt(acc / (1 - v1 ** ct)) + eps)
        return g

    # ---- sparse adaptive scalers with the duplicate-index rules (gru4rec.py:315-381) ----
    def _adapt_sparse(self, name, P, idx, g):
        dt = self.dtype
        eps = dt(1e-6)
        if self.adapt == 'adagrad':
            acc = self._state(name, P, 'acc')
            acc_new = acc[idx] + g * g
            acc[idx] = acc_new            # set_subtensor: last duplicate wins (NumPy/Theano-CPU order)
            return g / np.sqrt(acc_new + eps)
        if self.adapt == 'rmsprop':
            v1 = dt(self.adapt_params[0]); v2 = dt(1.0 - self.adapt_params[0])
            acc = self._state(name, P, 'acc')
            acc[idx] = acc[idx] * v1
            np.add.at(acc, idx, v2 * g * g)
            return g / np.sqrt(acc[idx] + eps)
        if self.adapt == 'adadelta':
            v1 = dt(self.adapt_params[0]); v2 = dt(1.0 - self.adapt_params[0])
            acc = self._state(name, P, 'acc'); upd = self._state(name, P, 'upd')
            acc[idx] = acc[idx] * v1
            np.add.at(acc, idx, v2 * g * g)
            upd_s = upd[idx]
            gs = (upd_s + eps) / (acc[idx] + eps)
            upd[idx] = upd_s * v1
            np.add.at(upd, idx, v2 * gs * g * g)
            return g * np.sqrt(gs)
        if self.adapt == 'adam':
            v1 = dt(self.adapt_params[0]); v2 = dt(1.0 - self.adapt_params[0])
            v3 = dt(self.adapt_params[1]); v4 = dt(1.0 - self.adapt_params[1])
            acc = self._state(name, P, 'acc'); mg = self._state(name, P, 'meang'); ct = self._state(name, P, 'countt')
            ct_s = ct[idx]
            acc[idx] = acc[idx] * v3
            np.add.at(acc, idx, v4 * g * g)
            mg[idx] = mg[idx] * v1
            np.add.at(mg, idx, v2 * g * g)       # sic: the reference uses grad**2 here (gru4rec.py:325)
            ct_new = ct_s + dt(1.0)
            ct[idx] = ct_new
            return (mg[idx] / (1 - v1 ** ct_new)) / (np.sqrt(acc[idx] / (1 - v1 ** ct_new)) + eps)
        return g

    # ---- forward (gru4rec.py:433-506) ----
    def _gru_layer(self, i, vec, H, R, predict, masks, cache):
        """gru4rec.py:460-466 / 473-479."""
        L = self.layers[i]
        rz = sigmoid(vec[:, L:] + H @ self.Wrz[i])
        r = rz[:, :L]
        z = rz[:, L:]
        a_h = (H * r) @ self.Wh[i] + vec[:, :L]
        ht = act_fwd(self.hact, a_h)
        h = (self.dtype(1.0) - z) * H + z * ht
        mk = masks.get(('h', i))
        hd = h * mk if mk is not None else h
        if (not predict) and R is not None:
            H_new = np.where(np.asarray(R, dtype=bool).reshape(-1, 1), self.dtype(0), hd)
        else:
            H_new = hd
        cache.update(H=H, r=r, z=z, a_h=a_h, ht=ht, mk=mk, H_new=H_new)
        return hd

    def forward(self, X, Y, M, R=None, samples=None, predict=False, masks=None, H=None):
        """model() (gru4rec.py:433-506).  X,Y int arrays [M]; samples int array [S] or None.
        Returns (yhat, cache)."""
        masks = masks or {}
        H = [h[:M] for h in self.H] if H is None else H
        C = dict(layers=[])
        if samples is not None and Y is not None and not predict and self.n_sample > 0:
            Y = np.concatenate([Y, samples])          # gru4rec.py:435-437
        Sy = None
        if self.constrained_embedding:                # gru4rec.py:438-448
            Xc = np.concatenate([X, Y]) if Y is not None else X
            S = self.Wy[Xc]
            Sx = S[:M]
            Sy = S[M:]
            mk = masks.get('e')
            y = Sx * mk if mk is not None else Sx
            C.update(mode='shared', Xc=Xc, S=S, mk_e=mk)
            start = 0
        elif self.embedding:                          # gru4rec.py:449-456
            Sx = self.E[X]
            mk = masks.get('e')
            y = Sx * mk if mk is not None else Sx
            C.update(mode='embed', mk_e=mk)
            start = 0
        else:                                         # gru4rec.py:457-470
            Sx = self.Wx[0][X]
            vec = Sx + self.Bh[0]
            lc = dict(inp=None)
            y = self._gru_layer(0, vec, H[0], R, predict, masks, lc)
            C['layers'].append(lc)
            C.update(mode='none')
            start = 1
        C['Sx'] = Sx
        for i in range(start, len(self.layers)):      # gru4rec.py:471-479
            vec = y @ self.Wx[i] + self.Bh[i]
            lc = dict(inp=y)
            y = self._gru_layer(i, vec, H[i], R, predict, masks, lc)
            C['layers'].append(lc)
        C['y_last'] = y
        C['X'] = X
        C['Y'] = Y
        C['H_new'] = [lc['H_new'] for lc in C['layers']]
        if Y is not None:                             # gru4rec.py:480-497
            if (not self.constrained_embedding) or predict:
                Sy = self.Wy[Y]
            SBy = self.By[Y]
            C['Sy'] = Sy
            o = y @ Sy.T + SBy.flatten()
            if predict and self.final_act == 'softmax_logit':
                yhat = act_fwd(('softmax', 0, 0), o)
            else:
                if not predict and self.logq:
                    corr = np.log(np.concatenate([self.P0[Y[:M]], self.P0[Y[M:]] ** self.dtype(self.sample_alpha)]))
                    o = o - self.dtype(self.logq) * corr.astype(self.dtype)
                yhat = act_fwd(self.fact, o)
        else:                                         # gru4rec.py:498-506
            o = y @ self.Wy.T + self.By.flatten()
            if predict and self.final_act == 'softmax_logit':
                yhat = act_fwd(('softmax', 0, 0), o)
            else:
                if not predict and self.logq:
                    o = o - self.dtype(self.logq) * np.log(self.P0)
                yhat = act_fwd(self.fact, o)
        C['o'] = o
        C['yhat'] = yhat
        return yhat, C

    def make_masks(self, M):
        """dropout masks for the current step (definition shared with the device path)."""
        masks = {}
        if self.dropout_p_embed > 0 and (self.constrained_embedding or self.embedding):
            width = self.layers[-1] if self.constrained_embedding else self.embedding
            masks['e'] = dropout_mask(self.dropout_seed, self.step_count, STREAM_EMBED, (M, width), self.dropout_p_embed, self.dtype)
        if self.dropout_p_hidden > 0:
            for i, L in enumerate(self.layers):
                masks[('h', i)] = dropout_mask(self.dropout_seed, self.step_count, i, (M, L), self.dropout_p_hidden, self.dtype)
        return masks

    # ---- backward (T.grad at gru4rec.py:383-384; formulas SURVEY Appendix A, re-derived) ----
    def backward(self, C, M):
        dt = self.dtype
        L, dyhat = loss_and_grad(self.loss, C['yhat'], M, self.n_sample, self.bpreg, self.smoothing)
        cost = dt(L / dt(self.batch_size))
        dyhat = dyhat / dt(self.batch_size)
        do = act_bwd(self.fact, C['o'], C['yhat'], dyhat)
        y_last = C['y_last']
        Sy = C['Sy']
        G = dict()
        G['dSy'] = do.T @ y_last
        G['dSBy'] = do.sum(axis=0).reshape(-1, 1)
        dy = do @ Sy
        nl = len(self.layers)
        G['dWx'] = [None] * nl
        G['dWh'] = [None] * nl
        G['dWrz'] = [None] * nl
        G['dBh'] = [None] * nl
        G['dvec'] = [None] * nl           # [da_h | da_r | da_z] per layer: lets tests compare the device's gate gradients directly
        first = nl - len(C['layers'])
        for li in range(len(C['layers']) - 1, -1, -1):
            lc = C['layers'][li]
            i = first + li
            Lw = self.layers[i]
            dh = dy * lc['mk'] if lc['mk'] is not None else dy
            H, r, z, ht = lc['H'], lc['r'], lc['z'], lc['ht']
            dz = dh * (ht - H)
            dht = dh * z
            da_h = act_bwd(self.hact, lc['a_h'], ht, dht)
            G['dWh'][i] = (H * r).T @ da_h
            dHr = da_h @ self.Wh[i].T
            dr = dHr * H
            da_r = dr * r * (dt(1) - r)
            da_z = dz * z * (dt(1) - z)
            da_rz = np.hstack([da_r, da_z])
            G['dWrz'][i] = H.T @ da_rz
            dvec = np.hstack([da_h, da_rz])
            G['dvec'][i] = dvec
            G['dBh'][i] = dvec.sum(axis=0)
            if lc['inp'] is not None:
                G['dWx'][i] = lc['inp'].T @ dvec
                dy = dvec @ self.Wx[i].T
            else:
                G['dSx'] = dvec
                dy = None
        if C['mode'] in ('shared', 'embed'):
            G['dSx'] = dy * C['mk_e'] if C['mk_e'] is not None else dy
        return cost, G

    # ---- updates (gru4rec.py:382-432) ----
    def apply_updates(self, C, G, M):
        dt = self.dtype
        lr = dt(self.learning_rate); mu = dt(self.momentum); lmbd = dt(self.lmbd)
        nl = len(self.layers)
        dense = []
        wx_start = 0 if (self.embedding or self.constrained_embedding) else 1
        for i in range(wx_start, nl):
            dense.append(('Wx%d' % i, self.Wx[i], G['dWx'][i]))
        for i in range(nl):
            dense.append(('Wh%d' % i, self.Wh[i], G['dWh'][i]))
        for i in range(nl):
            dense.append(('Wrz%d' % i, self.Wrz[i], G['dWrz'][i]))
        for i in range(nl):
            dense.append(('Bh%d' % i, self.Bh[i], G['dBh'][i]))
        sparse = []
        X, Y = C['X'], C['Y']
        if C['mode'] == 'shared':
            sparse.append(('Wy', self.Wy, C['Xc'], np.vstack([G['dSx'], G['dSy']]), C['S']))
        elif C['mode'] == 'embed':
            sparse.append(('E', self.E, X, G['dSx'], C['Sx']))
            sparse.append(('Wy', self.Wy, Y, G['dSy'], C['Sy']))
        else:
            sparse.append(('Wx0', self.Wx[0], X, G['dSx'], C['Sx']))
            sparse.append(('Wy', self.Wy, Y, G['dSy'], C['Sy']))
        sparse.append(('By', self.By, Y, G['dSBy'], self.By[Y]))
        self.last_gscale = dt(1.0)        # the factor grad_cap applied to every gradient of this step
        if self.grad_cap > 0:  # gru4rec.py:386-389
            norm = dt(np.sqrt(sum(np.sum(g * g) for _, _, g in dense) + sum(np.sum(g * g) for _, _, _, g, _ in sparse)))
            if norm >= self.grad_cap:
                sc = dt(self.grad_cap) / norm
                self.last_gscale = sc
                dense = [(n, p, g * sc) for n, p, g in dense]
                sparse = [(n, p, ix, g * sc, sp) for n, p, ix, g, sp in sparse]
        # all right-hand sides use the OLD parameter values (Theano evaluates updates simultaneously)
        new_vals = []
        for name, p, g in dense:
            gs = self._adapt_dense(name, p, g.astype(dt))
            if self.momentum > 0:
                vel = self._state(name, p, 'vel')
                v2 = mu * vel - lr * (gs + lmbd * p)
                vel[...] = v2
                new_vals.append((p, p + v2))
            else:
                new_vals.append((p, p * (dt(1.0) - lr * lmbd) - lr * gs))
        sp_ops = []
        for name, P, idx, g, sparam in sparse:
            gs = self._adapt_sparse(name, P, idx, g.astype(dt))
            delta = lr * (gs + lmbd * sparam) if self.lmbd > 0 else lr * gs
            if self.momentum > 0:
                vel = self._state(name, P, 'vel')
                v2 = mu * vel[idx] - delta
                vel[idx] = v2              # set_subtensor, last duplicate wins
                sp_ops.append((P, idx, v2))
            else:
                sp_ops.append((P, idx, -delta))
        for p, v in new_vals:
            p[...] = v
        for P, idx, inc in sp_ops:
            np.add.at(P, idx, inc.astype(dt))   # inc_subtensor accumulates duplicates

    def train_step(self, X, Y, R, samples=None, masks=None, slots=None):
        """One call of train_function (gru4rec.py:584,623).  If `slots` is given, self.H rows are physical
        lanes and lane b of the batch lives in row slots[b] (equivalent to the host-side compaction)."""
        M = len(X)
        X = np.asarray(X, dtype=np.int64); Y = np.asarray(Y, dtype=np.int64)
        if masks is None:
            masks = self.make_masks(M)
        if slots is None:
            Hs = [h[:M] for h in self.H]
        else:
            Hs = [h[slots] for h in self.H]
        yhat, C = self.forward(X, Y, M, R=R, samples=samples, masks=masks, H=Hs)
        cost, G = self.backward(C, M)
        self.apply_updates(C, G, M)
        for i in range(len(self.layers)):
            if slots is None:
                self.H[i][:M] = C['H_new'][i]
            else:
                self.H[i][slots] = C['H_new'][i]
        self.step_count += 1
        self.last_cache = C
        self.last_grads = G
        return cost

    # ---- scoring path (gru4rec.py:729-741 + evaluation.py:57-75) ----
    def predict_step(self, X, H, slots=None, zero=None, Y=None):
        """symbolic_predict: full-catalogue scores (Y=None) or the scores of the columns Y, with the final activation taken
        over exactly those columns as the reference does (gru4rec.py:735-736); H (physical lanes) updated, no reset.
        `zero`: lanes whose state is zeroed before the step (evaluation.py:136-139)."""
        M = len(X)
        slots = np.arange(M) if slots is None else np.asarray(slots)
        if zero is not None:
            zs = slots[np.asarray(zero, dtype=bool)]
            for h in H:
                h[zs] = 0
        yhat, C = self.forward(np.asarray(X, dtype=np.int64), None if Y is None else np.asarray(Y, dtype=np.int64), M, predict=True, H=[h[slots] for h in H])
        for i in range(len(self.layers)):
            H[i][slots] = C['H_new'][i]
        return yhat

    @staticmethod
    def ranks(yhat, Y, mode='standard', items=None):
        """evaluation.py:52-65.  items=None: yhat is [M x n_items] and the target competes with the whole catalogue (itself
        included).  items given: yhat is [M x (M + len(items))] over the columns concat(targets, items) (evaluation.py:94-97);
        `others` are the candidate columns only (evaluation.py:55-56) -- the target's own score takes part only if the
        target is in the subset, so 'conservative' can produce rank 0."""
        M = len(Y)
        if items is None:
            targets = yhat[np.arange(M), Y]
            others = yhat
        else:
            targets = yhat[np.arange(M), np.arange(M)]
            others = yhat[:, M:]
        if mode == 'standard' or mode == 'tiebreaking':
            return (others > targets[:, None]).sum(axis=1) + 1
        if mode == 'conservative':
            return (others >= targets[:, None]).sum(axis=1)
        if mode == 'median':
            return (others > targets[:, None]).sum(axis=1) + 0.5 * ((others == targets[:, None]).sum(axis=1) - 1) + 1
        raise NotImplementedError

    def evaluate(self, test_items, offset_sessions, batch_size=100, cut_off=(20,), mode='standard', items=None):
        """evaluate_gpu (evaluation.py:15-147).  `items`: item INDICES of the candidate subset or None.
        Returns (recall list, mrr list)."""
        H = [np.zeros((batch_size, L), dtype=self.dtype) for L in self.layers]
        steps = build_eval_schedule(test_items, offset_sessions, batch_size)
        rec = np.zeros(len(cut_off)); mrr = np.zeros(len(cut_off)); n = 0
        if items is not None:
            items = np.asarray(items, dtype=np.int64)
        for st in steps:
            ycols = None if items is None else np.concatenate([np.asarray(st['Y'], dtype=np.int64), items])
            yhat = self.predict_step(st['X'], H, slots=st['slots'], zero=st['Z'], Y=ycols)
            rk = self.ranks(yhat, st['Y'], mode, items)
            with np.errstate(divide='ignore', invalid='ignore'):
                for j, c in enumerate(cut_off):
                    rec[j] += (rk <= c).sum()
                    mrr[j] += ((rk <= c) / rk).sum()
            n += st['M']
        return list(rec / n), list(mrr / n)


# --------------------------------------------------------------------------------------------
# host-side preparation of fit() (gru4rec.py:534-545, 585; datatools.py:12-39)
# --------------------------------------------------------------------------------------------
def prepare_fit_data(data, session_key='SessionId', item_key='ItemId', time_key='Time', time_sort=True):
    """Returns dict(itemids, data_items, offset_sessions, base_order, supports) from a DataFrame, following
    the reference's order of operations: id map in input order BEFORE sorting, sort by (session,time),
    CSR offsets, session order by first event time, item supports in id-map order."""
    import pandas as pd
    data = data.copy()
    itemids = data[item_key].unique()                                      # gru4rec.py:534
    n_items = len(itemids)
    itemidmap = pd.Series(data=np.arange(n_items), index=itemids, name='ItemIdx')
    data['ItemIdx'] = itemidmap[data[item_key].values].values              # gru4rec.py:537
    data = data.sort_values([session_key, time_key], kind='stable')        # datatools.py:32 (only if unsorted)
    offset = np.zeros(data[session_key].nunique() + 1, dtype=np.int32)     # datatools.py:36-39
    offset[1:] = data.groupby(session_key).size().cumsum()
    supports = data.groupby(item_key).size()[itemidmap.index.values].values  # gru4rec.py:539,543
    if time_sort:
        base_order = np.argsort(data.groupby(session_key)[time_key].min().values)   # gru4rec.py:585
    else:
        base_order = np.arange(len(offset) - 1)
    return dict(itemids=itemids, itemidmap=itemidmap, data_items=data['ItemIdx'].values.astype(np.int64),
                offset_sessions=offset, base_order=base_order, supports=supports, n_items=n_items)


def prepare_eval_data(test, itemidmap, session_key='SessionId', item_key='ItemId', time_key='Time'):
    """evaluation.py:77-78,93-94: inner-merge on known items, sort by (session,time,item), offsets."""
    import pandas as pd
    test = pd.merge(test, pd.DataFrame({'ItemIdx': itemidmap.values, item_key: itemidmap.index}), on=item_key, how='inner')
    test = test.sort_values([session_key, time_key, item_key])
    offset = np.zeros(test[session_key].nunique() + 1, dtype=np.int32)
    offset[1:] = test.groupby(session_key).size().cumsum()
    return test['ItemIdx'].values.astype(np.int64), offset
