"""GRU4Rec with the reference's class surface (hidasib/GRU4Rec gru4rec.py:27-781) on the H100 engine.

`run.py -g gru4rec_b200.gru4rec` (or the root-level shim module `gru4rec`) selects this class through the
reference's own plugin seam (run.py:21,39).  Constructor arguments, set_params() coercions and prints,
fit() / predict_next_batch() / savemodel() / loadmodel() signatures and printed lines follow the reference;
the per-mini-batch work runs in libg4r.so (hand-written sm_90a CUDA) through ctypes.  PyTorch is used
only to allocate the device workspace.  There is no CPU fallback.

Interface restatement, stated plainly: `__init__` (argument list, defaults, attribute assignments), `set_params` (the
coercion table and its `SET ... TO ...` / error prints), `init_matrix`, `generate_neg_samples` and the popularity / CDF
preamble of `fit` are the reference's statements almost line for line (gru4rec.py:97-135, 162-187, 254-260, 507-514,
534-556).  That is deliberate and required by the drop-in boundary: keyword names, defaults, coercions, printed lines,
exception types and the NumPy random-stream consumption order are the interface, and
tests/golden/set_params_cases.json + the golden fixtures pin them against the reference class.  Everything below that
surface (schedule, step, optimizers, evaluation, persistence plumbing, multi-GPU) is this repository's own design.
"""
import hashlib
import json
import os
import pickle
import time
import weakref
from types import SimpleNamespace
from collections import OrderedDict  # noqa: F401  (param files use it)

import numpy as np
import pandas as pd

from . import datatools
from . import _lib


class _DeviceParam(object):
    """Stand-in for a Theano shared variable: get_value()/set_value() round-trip through the engine."""

    def __init__(self, owner, name):
        self._owner = weakref.ref(owner)     # no reference cycle: the model (and its device engine) is freed by reference counting
        self.name = name

    def get_value(self, borrow=False):
        return self._owner()._get_param(self.name)

    def set_value(self, value, borrow=False):
        self._owner()._set_param(self.name, value)


class GRU4Rec:
    '''
    GRU4Rec(loss='bpr-max', final_act='elu-1', hidden_act='tanh', layers=[100],
                 n_epochs=10, batch_size=32, dropout_p_hidden=0.0, dropout_p_embed=0.0, learning_rate=0.1, momentum=0.0, lmbd=0.0, embedding=0, n_sample=2048, sample_alpha=0.75, smoothing=0.0, constrained_embedding=False,
                 adapt='adagrad', adapt_params=[], grad_cap=0.0, bpreg=1.0, logq=0.0,
                 sigma=0.0, init_as_normal=False, train_random_order=False, time_sort=True,
                 session_key='SessionId', item_key='ItemId', time_key='Time')
    Same parameters as the reference class (gru4rec.py:28-96), all optimizers (adagrad / rmsprop / adadelta / adam / None),
    grad_cap and smoothing included.  Not on the device path (NotImplementedError when fit() builds the engine): loss /
    final_act pairs other than {cross-entropy+softmax, xe_logit+softmax_logit, pairwise losses + elementwise activations},
    and rmsprop / adadelta / adam together with constrained_embedding.
    '''

    def __init__(self, loss='bpr-max', final_act='linear', hidden_act='tanh', layers=[100],
                 n_epochs=10, batch_size=32, dropout_p_hidden=0.0, dropout_p_embed=0.0, learning_rate=0.1, momentum=0.0, lmbd=0.0, embedding=0, n_sample=2048, sample_alpha=0.75, smoothing=0.0, constrained_embedding=False,
                 adapt='adagrad', adapt_params=[], grad_cap=0.0, bpreg=1.0, logq=0.0,
                 sigma=0.0, init_as_normal=False, train_random_order=False, time_sort=True,
                 session_key='SessionId', item_key='ItemId', time_key='Time'):
        self.layers = layers
        self.n_epochs = n_epochs
        self.batch_size = batch_size
        self.dropout_p_hidden = dropout_p_hidden
        self.dropout_p_embed = dropout_p_embed
        self.learning_rate = learning_rate
        self.adapt_params = adapt_params
        self.momentum = momentum
        self.sigma = sigma
        self.init_as_normal = init_as_normal
        self.session_key = session_key
        self.item_key = item_key
        self.time_key = time_key
        self.grad_cap = grad_cap
        self.bpreg = bpreg
        self.logq = logq
        self.train_random_order = train_random_order
        self.lmbd = lmbd
        if embedding == 'layersize':
            self.embedding = self.layers[0]
        else:
            self.embedding = embedding
        self.constrained_embedding = constrained_embedding
        self.time_sort = time_sort
        self.adapt = adapt
        self.loss = loss
        self.set_loss_function(self.loss)
        self.final_act = final_act
        self.set_final_activation(self.final_act)
        self.hidden_act = hidden_act
        self.set_hidden_activation(self.hidden_act)
        self.n_sample = n_sample
        self.sample_alpha = sample_alpha
        self.smoothing = smoothing
        # engine-side options (not part of the reference surface)
        self.device = 0
        self.dropout_seed = 0
        self.eval_lanes = 512            # run.py evaluates with batch_size=512 (run.py:127)
        self.step_mode = 2               # role-specialised persistent kernel where the shape allows, else generic persistent
        self.session_capacity = 100000   # sessions kept by recommend_sessions / feed_sessions (least recently used evicted)
        self.bptt = 1                    # > 1: truncated backpropagation through time, one update per window of bptt mini-batches (DESIGN §3l)
        self.full_softmax = False        # True: every training step scores and updates the whole catalogue, no sampling (DESIGN §3n)
        self._engine = None
        self._host = None                # numpy copies of the parameters when no engine is alive


    # ---- names that pickles written by the reference class refer to (gru4rec.py:136-161, 189-248) ----------------------
    # The reference pickles `self` including bound methods (loss_function = self.bpr_max, final_activation =
    # self.Elu(a).execute, ...).  These stubs make such pickles load into this class; the Theano graph builders themselves
    # have no counterpart here (the device kernels are selected from the `loss` / `final_act` / `hidden_act` strings).
    def _make_stub(name):
        def stub(self, *a, **k):
            raise NotImplementedError('Theano graph builders are not part of the CUDA implementation')
        stub.__name__ = name            # bound methods are pickled by name: it must be the reference's method name
        stub.__qualname__ = 'GRU4Rec.' + name
        return stub
    cross_entropy = _make_stub('cross_entropy'); cross_entropy_logits = _make_stub('cross_entropy_logits')
    bpr = _make_stub('bpr'); bpr_max = _make_stub('bpr_max'); top1 = _make_stub('top1'); top1_max = _make_stub('top1_max')
    linear = _make_stub('linear'); tanh = _make_stub('tanh'); softmax = _make_stub('softmax'); softmax_logit = _make_stub('softmax_logit')
    softmax_neg = _make_stub('softmax_neg'); relu = _make_stub('relu'); sigmoid = _make_stub('sigmoid')
    del _make_stub

    class Selu:
        def __init__(self, lmbd=1.0, alpha=1.0):
            self.lmbd = lmbd; self.alpha = alpha
        def execute(self, X):
            raise NotImplementedError('Theano graph builders are not part of the CUDA implementation')

    class Elu:
        def __init__(self, alpha=1.0):
            self.alpha = alpha
        def execute(self, X):
            raise NotImplementedError('Theano graph builders are not part of the CUDA implementation')

    class LeakyReLU:
        def __init__(self, leak=0.0):
            self.leak = leak
        def execute(self, X):
            raise NotImplementedError('Theano graph builders are not part of the CUDA implementation')

    # ---- same validation behaviour as the reference setters (gru4rec.py:136-161) ----
    def set_loss_function(self, loss):
        if loss not in ('cross-entropy', 'bpr', 'bpr-max', 'top1', 'top1-max', 'xe_logit'):
            raise NotImplementedError

    def set_final_activation(self, final_act):
        _lib.parse_act(final_act)

    def set_hidden_activation(self, hidden_act):
        if hidden_act in ('softmax', 'softmax_logit'):
            raise NotImplementedError
        _lib.parse_act(hidden_act)

    def set_params(self, **kvargs):
        """gru4rec.py:162-187, including the printed lines."""
        maxk_len = np.max([len(str(x)) for x in kvargs.keys()])
        maxv_len = np.max([len(str(x)) for x in kvargs.values()])
        for k, v in kvargs.items():
            if not hasattr(self, k):
                print('Unkown attribute: {}'.format(k))
                raise NotImplementedError
            else:
                if type(v) == str and k == 'adapt_params': v = [float(l) for l in v.split('/')]
                elif type(v) == str and type(getattr(self, k)) == list: v = [int(l) for l in v.split('/')]
                if type(v) == str and type(getattr(self, k)) == bool:
                    if v == 'True' or v == '1': v = True
                    elif v == 'False' or v == '0': v = False
                    else:
                        print('Invalid value for boolean parameter: {}'.format(v))
                        raise NotImplementedError
                if k == 'embedding' and v == 'layersize':
                    self.embedding = 'layersize'
                setattr(self, k, type(getattr(self, k))(v))
                if k == 'loss': self.set_loss_function(self.loss)
                if k == 'final_act': self.set_final_activation(self.final_act)
                if k == 'hidden_act': self.set_hidden_activation(self.hidden_act)
                print('SET   {}{}TO   {}{}(type: {})'.format(k, ' ' * (maxk_len - len(k) + 3), getattr(self, k), ' ' * (maxv_len - len(str(getattr(self, k))) + 3), type(getattr(self, k))))
        if self.embedding == 'layersize':
            self.embedding = self.layers[0]
            print('SET   {}{}TO   {}{}(type: {})'.format('embedding', ' ' * (maxk_len - len('embedding') + 3), getattr(self, 'embedding'), ' ' * (maxv_len - len(str(getattr(self, 'embedding'))) + 3), type(getattr(self, 'embedding'))))

    # ---- weight initialisation, draw order as in the reference (gru4rec.py:254-294) ----
    def init_matrix(self, shape):
        if self.sigma != 0: sigma = self.sigma
        else: sigma = np.sqrt(6.0 / (shape[0] + shape[1]))
        if self.init_as_normal:
            return np.asarray(np.random.randn(*shape) * sigma, dtype=np.float32)
        else:
            return np.asarray(np.random.rand(*shape) * sigma * 2 - sigma, dtype=np.float32)

    def _init_host_weights(self):
        np.random.seed(42)
        w = {}
        if self.constrained_embedding:
            n_features = self.layers[-1]
        elif self.embedding:
            w['E'] = self.init_matrix((self.n_items, self.embedding))
            n_features = self.embedding
        else:
            n_features = self.n_items
        for i in range(len(self.layers)):
            nin = self.layers[i - 1] if i > 0 else n_features
            m = [self.init_matrix((nin, self.layers[i])) for _ in range(3)]
            w['Wx%d' % i] = np.hstack(m)
            w['Wh%d' % i] = self.init_matrix((self.layers[i], self.layers[i]))
            m2 = [self.init_matrix((self.layers[i], self.layers[i])) for _ in range(2)]
            w['Wrz%d' % i] = np.hstack(m2)
            w['Bh%d' % i] = np.zeros((self.layers[i] * 3,), dtype=np.float32)
        w['Wy'] = self.init_matrix((self.n_items, self.layers[-1]))
        w['By'] = np.zeros((self.n_items, 1), dtype=np.float32)
        return w

    def init(self, data):
        datatools.sort_if_needed(data, [self.session_key, self.time_key])
        offset_sessions = datatools.compute_offset(data, self.session_key)
        self._host = self._init_host_weights()
        return offset_sessions

    # ---- engine management ----
    def _param_names(self):
        names = []
        for i in range(len(self.layers)):
            names += ['Wx%d' % i, 'Wh%d' % i, 'Wrz%d' % i, 'Bh%d' % i]
        names += ['Wy', 'By']
        if self.embedding and not self.constrained_embedding:
            names.append('E')
        return names

    def _make_config(self, sample_store, eval_lanes, training=True, single=False):
        """`training=False`: an engine for the scoring path only (evaluate_gpu / predict_next_batch of a loaded model): the
        optimiser options are irrelevant there, so a model the reference trained with adam / rmsprop / adadelta, grad_cap or
        smoothing can still be scored; fit() with those options raises NotImplementedError (SURVEY section 8 a14)."""
        cfg = _lib.G4RConfig()
        if training and self.adapt not in _lib.ADAPT:
            raise NotImplementedError('adapt=%r is not an optimizer of the reference (gru4rec.py:392-399)' % (self.adapt,))
        cfg.n_items = self.n_items
        cfg.n_layers = len(self.layers)
        for i, l in enumerate(self.layers):
            cfg.layers[i] = l
        cfg.batch_size = self.batch_size
        cfg.constrained_embedding = 1 if self.constrained_embedding else 0
        cfg.embedding = 0 if self.constrained_embedding else int(self.embedding or 0)
        cfg.loss = _lib.LOSS[self.loss]
        cfg.final_act, cfg.final_act_p1, cfg.final_act_p2 = _lib.parse_act(self.final_act)
        cfg.hidden_act, cfg.hidden_act_p1, cfg.hidden_act_p2 = _lib.parse_act(self.hidden_act)
        cfg.dropout_p_hidden = self.dropout_p_hidden
        cfg.dropout_p_embed = self.dropout_p_embed
        cfg.learning_rate = self.learning_rate
        cfg.momentum = self.momentum
        cfg.lmbd = self.lmbd
        cfg.n_sample = self.n_sample
        cfg.sample_alpha = self.sample_alpha
        cfg.smoothing = self.smoothing if training else 0.0
        cfg.bpreg = self.bpreg
        cfg.logq = self.logq
        cfg.adapt = _lib.ADAPT[self.adapt] if training else _lib.ADAPT[None]
        cfg.sample_store = int(sample_store)
        cfg.dropout_seed = self.dropout_seed
        cfg.mrg_seed = 12345
        _lib.set_adapt_params(cfg, self.adapt if training else None, self.adapt_params if training else [], self.grad_cap if training else 0.0)
        cfg.max_resident_steps = 0
        cfg.world_size, cfg.rank = (1, 0) if single else self._world()
        cfg.eval_batch_size = eval_lanes
        cfg.step_mode = self.step_mode
        cfg.bptt = int(self.bptt) if training else 1
        cfg.full_softmax = 1 if (training and self.full_softmax) else 0
        if self.step_mode == 2 and len(self.layers) == 1 and 120 < self.layers[0] <= 128 and not self.constrained_embedding and not self.embedding and self.batch_size <= 32:
            cfg.step_mode = 3        # the 48-CTA GRU group of step_mode 2 covers 120 hidden units; the cluster variant takes up to 128
        return cfg

    @staticmethod
    def _world():
        """(world_size, rank) of the torch.distributed job this process belongs to, or (1, 0)."""
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                return dist.get_world_size(), dist.get_rank()
        except Exception:
            pass
        return 1, 0

    def _build_engine(self, sample_store=0, eval_lanes=None, training=True, single=False, keep_sessions=True):
        """`single`: a one-GPU engine even under torchrun (the scoring path of every rank works on a full replica).
        `keep_sessions`: the session store of the old engine (recommend_sessions) moves to the new one."""
        eval_lanes = self.eval_lanes if eval_lanes is None else eval_lanes
        host = self._host if self._host is not None else self._pull_host()
        sessions = None
        if self._engine is not None:
            if keep_sessions and getattr(self._engine, 'session_capacity', None) is not None:
                sessions = (self._engine.session_capacity, self._engine.sessions_export())
            self._engine.close()
            self._engine = None
        world, rank = (1, 0) if single else self._world()
        if self._world()[0] > 1:
            import torch
            self.device = torch.cuda.current_device()
        eng = _lib.Engine(self._make_config(sample_store, eval_lanes, training, single=single), device=self.device)
        for name in self._param_names():
            eng.set(name, host[name])
        if world > 1:
            import torch.distributed as dist
            eng.init_multi_gpu(dist)
        if sessions is not None:
            eng.sessions_open(sessions[0])
            eng.sessions_import(*sessions[1])
        self._engine = eng
        self._engine_eval_lanes = eval_lanes
        self._engine_training = bool(training)     # it holds optimizer state: fit_more() / save_checkpoint() keep it
        self._host = None
        self._bind_params()
        return eng

    def _bind_params(self):
        n = len(self.layers)
        self.Wx = [_DeviceParam(self, 'Wx%d' % i) for i in range(n)]
        self.Wh = [_DeviceParam(self, 'Wh%d' % i) for i in range(n)]
        self.Wrz = [_DeviceParam(self, 'Wrz%d' % i) for i in range(n)]
        self.Bh = [_DeviceParam(self, 'Bh%d' % i) for i in range(n)]
        self.H = [_DeviceParam(self, 'H%d' % i) for i in range(n)]
        self.Wy = _DeviceParam(self, 'Wy')
        self.By = _DeviceParam(self, 'By')
        if self.embedding and not self.constrained_embedding:
            self.E = _DeviceParam(self, 'E')

    def _get_param(self, name):
        if self._engine is not None:
            a = self._engine.get(name)
            return a.reshape(-1) if name.startswith('Bh') else a
        return self._host[name]

    def _set_param(self, name, value):
        if self._engine is not None:
            self._engine.set(name, value)
        else:
            self._host[name] = np.asarray(value, dtype=np.float32)

    def _pull_host(self):
        return {name: self._get_param(name) for name in self._param_names()}

    def _ensure_engine(self, eval_lanes):
        """Engine for the scoring path (evaluate_gpu / predict_next_batch).  After a multi-GPU fit() the training engine holds
        1/world of the item tables: the parameters are assembled on the host and every rank scores on its own full replica."""
        if self._engine is None or self._engine_eval_lanes < eval_lanes or int(self._engine.cfg.world_size) > 1:
            self._build_engine(sample_store=0, eval_lanes=max(eval_lanes, self.eval_lanes), training=False, single=True)
        return self._engine

    def generate_neg_samples(self, pop, length):
        """Legacy host-side sampler (store_type='cpu'; gru4rec.py:507-514)."""
        if self.sample_alpha:
            sample = np.searchsorted(pop, np.random.rand(self.n_sample * length))
        else:
            sample = np.random.choice(self.n_items, size=self.n_sample * length)
        if length > 1:
            sample = sample.reshape((length, self.n_sample))
        return sample

    # ---- training (gru4rec.py:515-664) ----
    def fit(self, data, sample_store=10000000, store_type='gpu'):
        '''
        Trains the network.  Same arguments, data-frame side effects ('ItemIdx' column, in-place sort) and
        printed lines as the reference (gru4rec.py:515-664).
        '''
        offset_sessions = self._index_items(data)
        plan = self._plan_training(data, offset_sessions, sample_store, store_type)
        for _ in self._epochs(plan):
            pass

    def _index_items(self, data):
        '''fit()'s preamble: the id map in order of first appearance, the item index column, fresh weights; returns the session offsets'''
        self.predict = None
        self.error_during_train = False
        self._host_state = None
        # id map in order of first appearance, item index column, supports -- one factorize + one bincount (same values as the
        # reference's unique() / Series lookup / groupby().size() chain, gru4rec.py:534-545)
        codes, itemids = pd.factorize(data[self.item_key].values)
        if (codes < 0).any():
            raise KeyError('missing item id in the training data')
        self.n_items = len(itemids)
        self.itemidmap = pd.Series(data=np.arange(self.n_items), index=itemids, name='ItemIdx')
        data['ItemIdx'] = codes.astype(np.int64)
        return self.init(data)

    def _plan_training(self, data, offset_sessions, sample_store, store_type, build=None, restore=None, absent_logq=None):
        '''Everything between the item index and the epoch loop (gru4rec.py:539-585): sampling CDF and logQ support from `data`,
        the sample-store decision and its printed lines, the training engine -- from build(store size in ids), by default a new
        engine with the host weights -- and its first sample store.  `restore`: a checkpoint whose tensors, sample store and
        training state the engine takes over instead of drawing a store.  `absent_logq`: logQ support given to items that do
        not occur in `data` (fit_more; in fit() every item occurs).'''
        pop = pd.Series(np.bincount(data['ItemIdx'].values, minlength=self.n_items), index=self.itemidmap.index.values)
        P0 = None
        if self.logq:
            P0 = pop[self.itemidmap.index.values].values.astype(np.float32)
            if absent_logq is not None:
                P0[P0 == 0] = absent_logq
        generate_length = 0
        use_store = False
        self._check_full_softmax()
        if self.full_softmax:
            P0 = None
            print('Full softmax: every item is a score column of every mini-batch; n_sample, sample_alpha and logq (the correction of a sampled softmax) are not used')
        elif self.n_sample:
            pop = pop[self.itemidmap.index.values].values ** self.sample_alpha
            pop = pop.cumsum() / pop.sum()
            pop[-1] = 1
            if sample_store:
                generate_length = sample_store // self.n_sample
                if generate_length <= 1:
                    sample_store = 0
                    print('No example store was used')
                elif store_type == 'cpu':
                    use_store = True
                    print('Created sample store with {} batches of samples (type=CPU)'.format(generate_length))
                elif store_type == 'gpu':
                    use_store = True
                else:
                    print('Invalid store type {}'.format(store_type))
                    raise NotImplementedError
            else:
                print('No example store was used')
        per_step_sampling = False
        self._check_bptt(store_type)
        if self.n_sample and not use_store and not self.full_softmax:
            if store_type == 'cpu':
                # gru4rec.py:612-613: without a store every mini-batch draws its own row on the host (generate_neg_samples(pop, 1))
                per_step_sampling = True
            else:
                # the reference's device path has no per-step sampler: its loop dereferences an undefined sample pointer here
                raise NotImplementedError('n_sample > 0 needs a sample store when store_type is \'gpu\' (sample_store >= 2 * n_sample)')
        if self.adapt == 'adadelta' and self.learning_rate != 1.0:        # gru4rec.py:362-364
            print('Warn: learning_rate is not 1.0 while using adadelta. Setting learning_rate to 1.0')
            self.learning_rate = 1.0
        world, rank = self._world()
        if world > 1 and self.constrained_embedding:
            # the merged update of a shared table interleaves the input rows Wy[X] with the score columns of every rank; the
            # library refuses it too (g4r_mg_init) -- say so before any engine is built, identically on every rank
            raise NotImplementedError('constrained_embedding=True does not train on several GPUs yet: run fit() in one process '
                                      '(evaluate_gpu / predict_next_batch of the trained model do run under torchrun)')
        if world > 1 and store_type == 'cpu':
            # the host-side sampler draws from one NumPy stream and refills at rank-local step counts: the lock-step ranks
            # would diverge (different numbers of collectives) -- only the device store is defined for multi-GPU training
            raise NotImplementedError("store_type='cpu' is not available for multi-GPU training; use the device sample store")
        # the training engine carries no scoring lanes: the step scratch keeps the leading dimension of the mini-batch
        # (the scoring engine with `eval_lanes` lanes is created on the first evaluate_gpu / predict_next_batch call)
        n_store = sample_store if use_store else (2 * self.n_sample if per_step_sampling else 0)
        eng = self._build_engine(sample_store=n_store, eval_lanes=0, keep_sessions=False) if build is None else build(n_store)
        if P0 is not None:
            eng.set_logq_support(P0)
        if use_store:
            eng.set_sampling_cdf(pop.astype(np.float32))
        if restore is not None:
            self._push_train_state(eng, restore)
        if use_store:
            if store_type == 'gpu':
                if restore is None:
                    eng.generate_samples()
                print('Created sample store with {} batches of samples (type=GPU)'.format(generate_length))
            elif restore is None:
                eng.set_sample_store(self.generate_neg_samples(pop, generate_length))
        # first event time of every session = the time at its offset (the frame is sorted by session, time) -- gru4rec.py:585
        base_order = np.argsort(data[self.time_key].values[offset_sessions[:-1]]) if self.time_sort else np.arange(len(offset_sessions) - 1)
        return SimpleNamespace(eng=eng, pop=pop, generate_length=generate_length, use_store=use_store, per_step_sampling=per_step_sampling,
                               store_type=store_type, offset_sessions=offset_sessions, base_order=base_order,
                               data_items=data.ItemIdx.values, world=world, rank=rank)

    def _check_bptt(self, store_type):
        '''the training options bptt > 1 does not cover, refused before any engine is built'''
        bptt = int(self.bptt)
        if bptt < 1 or bptt > 64:
            raise ValueError('bptt must be in [1, 64], got %r' % (self.bptt,))
        if bptt == 1:
            return
        if self._world()[0] > 1:
            raise NotImplementedError('bptt > 1 trains on one GPU; truncated BPTT over several GPUs is not implemented')
        if self.n_sample and store_type == 'cpu':
            raise NotImplementedError("bptt > 1 draws its negatives from the device sample store: store_type='cpu' is not implemented")

    def _check_full_softmax(self):
        '''the training options full_softmax does not cover, refused before any engine is built'''
        if not self.full_softmax:
            return
        if (self.loss, self.final_act) not in (('cross-entropy', 'softmax'), ('xe_logit', 'softmax_logit')):
            raise NotImplementedError("full_softmax trains loss='cross-entropy' with final_act='softmax' or loss='xe_logit' with "
                                      "final_act='softmax_logit'; got %r / %r" % (self.loss, self.final_act))
        if self.smoothing > 0:
            raise NotImplementedError('full_softmax with label smoothing is not implemented')
        if self.grad_cap > 0:
            raise NotImplementedError('full_softmax with grad_cap is not implemented')
        if int(self.bptt) > 1:
            raise NotImplementedError('full_softmax with bptt > 1 is not implemented')
        if self._world()[0] > 1:
            raise NotImplementedError('full_softmax trains on one GPU; the full catalogue over several GPUs is not implemented')

    def _epochs(self, plan, epochs=None, every=None, resume=None):
        '''The epoch loop of fit() (gru4rec.py:586-664) as a generator: it yields a progress record wherever a checkpoint may be
        taken -- after every `every` mini-batches of an epoch (never, if None) and after each epoch's printed line.  A run
        continued from such a record (`resume`, on an engine restored to that moment) goes on bit for bit.  A record holds the
        epoch, the next step of its schedule, the costs of its steps so far (the epoch loss is one sum over all of them, so a
        resumed run adds them up exactly as the uninterrupted one does) and its session order.'''
        eng, world, rank = plan.eng, plan.world, plan.rank
        offset_sessions = plan.offset_sessions
        # under torchrun: synchronous data parallelism, every rank trains a shard of the sessions
        sched = None
        n_sample_eff = self.n_sample
        for epoch in (range(self.n_epochs) if epochs is None else epochs):
            t0 = time.time()
            if resume is not None and resume['step'] > 0:        # inside an epoch: hidden state and session order are the checkpoint's
                session_idx_arr = resume['order'] if self.train_random_order else plan.base_order
                done, costs = int(resume['step']), [np.asarray(resume['costs'], dtype=np.float32)]
            else:
                eng.reset_hidden()
                session_idx_arr = np.random.permutation(len(offset_sessions) - 1) if self.train_random_order else plan.base_order
                done, costs = 0, []
            resume = None
            if sched is None or self.train_random_order:
                n_steps = None
                if world > 1:
                    import torch.distributed as dist
                    from .parallel import shard_sessions, common_steps
                    session_idx_arr = shard_sessions(session_idx_arr, rank, world)
                sched = _lib.Schedule(plan.data_items, offset_sessions, session_idx_arr, self.batch_size, n_sample_eff, mode=0)
                n_steps = sched.n_steps if world == 1 else common_steps(sched.n_steps, dist)
                cc = sched.batch_sizes()[:n_steps].astype(np.float64)
            try:
                while True:
                    n = n_steps - done if every is None else min(every, n_steps - done)
                    costs.append(self._train_range(plan, sched, done, n))
                    done += n
                    if done >= n_steps:
                        break
                    yield dict(epoch=epoch, step=done, costs=np.concatenate(costs), order=session_idx_arr)
            except _lib.NaNError:
                print(str(epoch) + ': NaN error!')
                self.error_during_train = True
                if world > 1:      # the peers find out at their next exchange (time-out -> RuntimeError); nothing collective here
                    self._engine.close(); self._engine = None; self._host = None
                return
            c = costs[0] if len(costs) == 1 else np.concatenate(costs)
            sum_c, sum_e, n_mb = np.sum(c * cc), np.sum(cc), len(c)
            if world > 1:
                # one epoch line for the whole job: event-weighted loss, mini-batches and events of all ranks
                from .parallel import allreduce_sum
                sum_c, sum_e, n_mb = allreduce_sum([sum_c, sum_e, n_mb], dist)
            avgc = sum_c / sum_e
            if np.isnan(avgc):
                print('Epoch {}: NaN error!'.format(str(epoch)))
                self.error_during_train = True
                break
            t1 = time.time()
            dt = t1 - t0
            print('Epoch{} --> loss: {:.6f} \t({:.2f}s) \t[{:.2f} mb/s | {:.0f} e/s]'.format(epoch + 1, avgc, dt, n_mb / dt, sum_e / dt))
            yield dict(epoch=epoch + 1, step=0, costs=np.zeros(0, np.float32), order=None)
        if world > 1:
            self._release_multi_gpu_engine()

    def _train_range(self, plan, sched, first, n):
        '''costs of mini-batches [first, first + n) of the epoch's schedule, with the plan's sampler'''
        if plan.per_step_sampling:
            return self._train_epoch_per_step_samples(plan.eng, sched, plan.pop, first, n)
        if plan.use_store and plan.store_type == 'cpu':
            return self._train_epoch_cpu_store(plan.eng, sched, plan.pop, plan.generate_length, first, n)
        return plan.eng.train_steps(sched, first, n)

    # ---- continuing a trained model (additions to the reference surface; DESIGN §3i) ----
    _CKPT_VERSION = 1

    def _ctor_params(self):
        keys = ('loss', 'final_act', 'hidden_act', 'layers', 'n_epochs', 'batch_size', 'dropout_p_hidden', 'dropout_p_embed', 'learning_rate',
                'momentum', 'lmbd', 'embedding', 'n_sample', 'sample_alpha', 'smoothing', 'constrained_embedding', 'adapt', 'adapt_params',
                'grad_cap', 'bpreg', 'logq', 'sigma', 'init_as_normal', 'train_random_order', 'time_sort', 'session_key', 'item_key', 'time_key')
        as_json = lambda v: v.item() if isinstance(v, np.generic) else ([as_json(x) for x in v] if isinstance(v, (list, tuple)) else v)
        return {k: as_json(getattr(self, k)) for k in keys}

    def _state_names(self):
        '''optimizer-state tensors and training hidden states, as the engine names them'''
        slots = {None: (), 'adagrad': ('acc',), 'rmsprop': ('acc',), 'adadelta': ('acc', 'upd'), 'adam': ('acc', 'meang', 'countt')}[self.adapt]
        slots = slots + (('vel',) if self.momentum > 0 else ())
        return ['%s.%s' % (n, s) for n in self._param_names() for s in slots] + ['H%d' % i for i in range(len(self.layers))]

    def _has_train_state(self):
        return (self._engine is not None and getattr(self, '_engine_training', False)) or getattr(self, '_host_state', None) is not None

    def _pull_train_state(self):
        '''the training state of the live training engine as host arrays, or the one load_checkpoint() left; None if there is none'''
        eng = self._engine
        if eng is None or not getattr(self, '_engine_training', False):
            return getattr(self, '_host_state', None)
        rows = eng.sample_store_rows()
        return dict(tensors={n: eng.get(n) for n in self._state_names()}, blob=eng.train_state_export(),
                    store=eng.get_sample_store().astype(np.int32) if rows > 0 else None,
                    sample_store=int(eng.cfg.sample_store))

    def _push_train_state(self, eng, st):
        for name in self._param_names():
            if name in st.get('params', {}):
                eng.set(name, st['params'][name])
        for name, a in st['tensors'].items():
            eng.set(name, a)
        if st['store'] is not None:
            eng.set_sample_store(st['store'])
        eng.train_state_import(st['blob'])

    def save_checkpoint(self, path, _progress=None, _fingerprint=None):
        '''
        Writes everything needed to continue training this model to one .npz file (arrays and one JSON string; no pickle): the
        constructor parameters, the item id map, all parameters and -- when the model holds a training engine (after fit(),
        fit_more(), inside fit_resumable()) or came from load_checkpoint() -- all optimizer state, the training hidden state, the
        sample store and the engine's training state.  The file is written under a temporary name and moved into place.
        savemodel() pickles are unaffected (weights only, reference-compatible).
        '''
        st = self._pull_train_state()
        ids = np.asarray(self.itemidmap.index.values)
        ids_are_objects = ids.dtype.kind not in 'iufUS'          # item ids read as str: stored as a fixed-width string array
        meta = dict(version=self._CKPT_VERSION, params=self._ctor_params(), n_items=int(self.n_items), ids_are_objects=bool(ids_are_objects),
                    engine=dict(dropout_seed=int(self.dropout_seed), step_mode=int(self.step_mode), bptt=int(self.bptt),
                                full_softmax=bool(self.full_softmax)),
                    has_state=st is not None, sample_store=None if st is None else st['sample_store'], has_store=st is not None and st['store'] is not None,
                    fingerprint=_fingerprint, progress=None)
        arrays = {'itemids': ids.astype(str) if ids_are_objects else ids}
        host = self._host if self._engine is None else self._pull_host()
        arrays.update({'param/' + n: host[n] for n in self._param_names()})
        if st is not None:
            arrays.update({'state/' + n: a for n, a in st['tensors'].items()})
            arrays['blob'] = st['blob']
            if st['store'] is not None:
                arrays['sample_store'] = st['store']
        if _progress is not None:
            meta['progress'] = dict(epoch=int(_progress['epoch']), step=int(_progress['step']), has_order=_progress['order'] is not None)
            arrays['epoch_costs'] = _progress['costs']
            if _progress['order'] is not None:
                arrays['epoch_order'] = np.asarray(_progress['order'], dtype=np.int64)
            rng = np.random.get_state()
            meta['rng'] = [rng[0], int(rng[2]), int(rng[3]), float(rng[4])]
            arrays['rng_keys'] = rng[1]
        arrays['meta'] = np.array(json.dumps(meta))
        tmp = '%s.tmp.%d' % (path, os.getpid())
        try:
            with open(tmp, 'wb') as f:
                np.savez(f, **arrays)
                f.flush()
                os.fsync(f.fileno())
            os.replace(tmp, path)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)

    @staticmethod
    def _read_checkpoint(path):
        with np.load(path, allow_pickle=False) as z:
            meta = json.loads(str(z['meta']))
            if meta.get('version') != GRU4Rec._CKPT_VERSION:
                raise ValueError('%s: checkpoint version %r, this build reads version %d' % (path, meta.get('version'), GRU4Rec._CKPT_VERSION))
            ck = dict(meta=meta, itemids=z['itemids'], params={k[6:]: z[k] for k in z.files if k.startswith('param/')},
                      tensors={k[6:]: z[k] for k in z.files if k.startswith('state/')},
                      blob=z['blob'] if 'blob' in z.files else None, store=z['sample_store'] if 'sample_store' in z.files else None,
                      sample_store=meta['sample_store'])
            if meta['progress'] is not None:
                ck['progress'] = dict(epoch=meta['progress']['epoch'], step=meta['progress']['step'], costs=z['epoch_costs'],
                                      order=z['epoch_order'] if meta['progress']['has_order'] else None)
                r = meta['rng']
                ck['rng'] = (r[0], z['rng_keys'], r[1], r[2], r[3])
        return ck

    @classmethod
    def load_checkpoint(cls, path):
        '''The model save_checkpoint() wrote: parameters for scoring at once, and -- if the file holds them -- optimizer state,
        hidden state, sample store and training state, which fit_more() continues from.'''
        ck = cls._read_checkpoint(path)
        meta = ck['meta']
        gru = cls(**meta['params'])
        gru.dropout_seed, gru.step_mode = meta['engine']['dropout_seed'], meta['engine']['step_mode']
        gru.bptt = int(meta['engine'].get('bptt', 1))             # written before bptt existed: one update per mini-batch
        gru.full_softmax = bool(meta['engine'].get('full_softmax', False))    # written before full_softmax existed: sampled columns
        ids = ck['itemids'].astype(object) if meta['ids_are_objects'] else ck['itemids']
        gru.predict = None
        gru.error_during_train = False
        gru._host_state = dict(tensors=ck['tensors'], blob=ck['blob'], store=ck['store'], sample_store=ck['sample_store']) if meta['has_state'] else None
        gru.n_items = int(meta['n_items'])
        gru.itemidmap = pd.Series(data=np.arange(gru.n_items), index=ids, name='ItemIdx')
        gru._host = {n: (a.reshape(-1) if n.startswith('Bh') else a) for n, a in ck['params'].items()}
        gru._bind_params()
        return gru

    def _data_fingerprint(self, data, sample_store, store_type, params):
        '''what a checkpoint of fit_resumable() must agree with to be continued: the data (events, items, a hash of the item index
        column of the sorted frame), the sample-store arguments and the constructor parameters the run started with'''
        return dict(n_events=int(len(data)), n_items=int(self.n_items), items_sha256=hashlib.sha256(np.ascontiguousarray(data['ItemIdx'].values, dtype=np.int64).tobytes()).hexdigest(),
                    sample_store=int(sample_store), store_type=store_type, params=params)

    def fit_resumable(self, data, path, every_steps, sample_store=10000000, store_type='gpu', on_checkpoint=None):
        '''
        fit() that survives an interruption: the same loop, with a checkpoint (save_checkpoint's format, plus the progress of the
        run and NumPy's random state) written to `path` after every `every_steps` mini-batches of an epoch and after every epoch.
        If `path` exists and was written for the same data, sample-store arguments and constructor parameters, training continues
        from it, and the finished run equals an uninterrupted fit() bit for bit -- weights, optimizer state and the epoch loss
        lines; otherwise a warning is printed and training starts anew.  `on_checkpoint(epoch, step)`, if given, is called after
        each checkpoint is in place.  Single GPU only.
        '''
        if self._world()[0] > 1:
            raise NotImplementedError('fit_resumable() runs on one GPU; checkpoints of a multi-GPU run are not implemented')
        every_steps = int(every_steps)
        if every_steps < 1:
            raise ValueError('every_steps must be at least 1, got %d' % every_steps)
        if every_steps % int(self.bptt) != 0:
            raise ValueError('every_steps (%d) must be a multiple of bptt (%d): a checkpoint falls between two windows' % (every_steps, int(self.bptt)))
        params = self._ctor_params()
        ck = self._read_checkpoint(path) if os.path.exists(path) else None
        offset_sessions = self._index_items(data)
        fingerprint = self._data_fingerprint(data, sample_store, store_type, params)
        if ck is not None and (ck['meta']['fingerprint'] != fingerprint or ck.get('progress') is None or not ck['meta']['has_state']):
            print('WARNING: checkpoint {} was written for other data or parameters; starting a new run'.format(path))
            ck = None
        plan = self._plan_training(data, offset_sessions, sample_store, store_type, restore=ck)
        resume = None
        if ck is not None:
            resume = ck['progress']
            np.random.set_state(ck['rng'])
            print('Resuming from checkpoint {} (epoch {}, mini-batch {})'.format(path, resume['epoch'] + 1, resume['step']))
        for prog in self._epochs(plan, epochs=range(resume['epoch'] if resume else 0, self.n_epochs), every=every_steps, resume=resume):
            self.save_checkpoint(path, _progress=prog, _fingerprint=fingerprint)
            if on_checkpoint is not None:
                on_checkpoint(prog['epoch'], prog['step'])

    def _init_rows(self, rs, shape):
        '''init_matrix's rule (sigma, init_as_normal) for a matrix of `shape`, drawn from the RandomState `rs`'''
        sigma = self.sigma if self.sigma != 0 else np.sqrt(6.0 / (shape[0] + shape[1]))
        if self.init_as_normal:
            return np.asarray(rs.randn(*shape) * sigma, dtype=np.float32)
        return np.asarray(rs.rand(*shape) * sigma * 2 - sigma, dtype=np.float32)

    def fit_more(self, data, n_epochs=None, sample_store=10000000, store_type='gpu'):
        '''
        Continues training the current model (after fit(), fit_resumable(), load_checkpoint() or loadmodel()) on `data` for
        n_epochs epochs (default: self.n_epochs), through fit()'s loop and with its printed lines.

        Items of `data` that the model does not know are appended to the item id map in order of first appearance; existing
        indices never move, so session histories, candidate lists and saved models stay valid.  Their rows of Wy and of E / Wx0
        are drawn by init_matrix's rule for a matrix of the new rows' shape from RandomState(42 + number of items before); their
        By and all their optimizer state are zero.  All other optimizer state is kept if the model has any (a live training
        engine, or load_checkpoint()) and starts from zero if not (loadmodel(), or a scoring engine has replaced the training
        engine); one printed line says which.  The sampling distribution is recomputed from `data` over the grown catalogue: an
        item absent from `data` is never a target or a sample (its logQ support is set to 1, so that its correction is zero).
        The sample store is drawn anew from the continuing random streams, the dropout step counter continues, and the session
        store of recommend_sessions survives.  Single GPU only.
        '''
        if self._world()[0] > 1:
            raise NotImplementedError('fit_more() runs on one GPU; growing a row-sharded model is not implemented')
        if getattr(self, 'itemidmap', None) is None or (self._engine is None and self._host is None):
            raise RuntimeError('fit_more() continues a trained model: call fit(), load_checkpoint() or loadmodel() first')
        self.predict = None
        self.error_during_train = False
        ids = data[self.item_key].values
        known = self.itemidmap.index.get_indexer(ids) >= 0
        new_ids = pd.unique(ids[~known])
        n_old, n_add = int(self.n_items), len(new_ids)
        # the model as a training engine of its present size: the live one, or one built from the host copy (+ checkpoint state)
        kept = self._has_train_state()
        if self._engine is None or not getattr(self, '_engine_training', False):
            st = getattr(self, '_host_state', None)
            eng = self._build_engine(sample_store=st['sample_store'] if st else 0, eval_lanes=0, single=True)
            if st is not None:
                self._push_train_state(eng, st)
            self._host_state = None
        print('Optimizer state kept' if kept else 'No optimizer state to keep: it starts from zero')
        rows = {}
        if n_add:
            rs = np.random.RandomState(42 + n_old)
            if self.embedding and not self.constrained_embedding:
                rows['new_in'] = self._init_rows(rs, (n_add, self.embedding))
            elif not self.constrained_embedding:
                rows['new_in'] = np.hstack([self._init_rows(rs, (n_add, self.layers[0])) for _ in range(3)])
            rows['new_Wy'] = self._init_rows(rs, (n_add, self.layers[-1]))
            self.itemidmap = pd.Series(data=np.arange(n_old + n_add), index=np.concatenate([self.itemidmap.index.values, new_ids]), name='ItemIdx')
            self.n_items = n_old + n_add
            print('Added {} new items to the catalogue ({} items)'.format(n_add, self.n_items))
        data['ItemIdx'] = self.itemidmap.index.get_indexer(ids).astype(np.int64)
        datatools.sort_if_needed(data, [self.session_key, self.time_key])
        offset_sessions = datatools.compute_offset(data, self.session_key)
        plan = self._plan_training(data, offset_sessions, sample_store, store_type, build=lambda n_store: self._grow_engine(n_store, rows),
                                   absent_logq=1.0)
        for _ in self._epochs(plan, epochs=range(self.n_epochs if n_epochs is None else int(n_epochs))):
            pass

    def _grow_engine(self, n_store, rows):
        '''the training engine for the catalogue as it is now, holding everything the present engine holds (fit_more)'''
        old = self._engine
        if int(old.cfg.n_items) == self.n_items and int(old.cfg.sample_store) == int(n_store) and int(old.cfg.bptt) == int(self.bptt) and \
                bool(old.cfg.full_softmax) == bool(self.full_softmax):
            return old
        sessions = (old.session_capacity, old.sessions_export()) if getattr(old, 'session_capacity', None) is not None else None
        eng = _lib.Engine(self._make_config(n_store, 0, True, single=True), device=self.device)
        eng.copy_item_tables(old, **rows)
        if int(old.cfg.sample_store) or int(old.cfg.full_softmax):   # (an engine built only to hold a loaded model has no streams to continue)
            try:
                eng.train_state_import(old.train_state_export())
            except NotImplementedError:
                print('The sample store changes size: the sample streams and the dropout step counter start anew')
        old.close()
        if sessions is not None:
            eng.sessions_open(sessions[0])
            eng.sessions_import(*sessions[1])
        self._engine, self._engine_eval_lanes, self._engine_training, self._host = eng, 0, True, None
        self._bind_params()
        return eng

    def _release_multi_gpu_engine(self):
        """End of a multi-GPU fit(): every rank assembles the full parameter set on the host (the item tables are row-sharded
        over the ranks' library-owned segments), then all ranks release their training engines together -- no rank frees its
        segment while a peer still reads it.  Scoring / saving afterwards needs no collective (evaluate_gpu, predict_next_batch
        rebuild a single-GPU engine from the host copy; savemodel pickles it)."""
        eng = self._engine
        if eng is None:
            return
        host = self._pull_host()
        eng._quiesce()
        eng.close()
        self._engine = None
        self._host = host

    def _train_epoch_cpu_store(self, eng, sched, pop, generate_length, first=0, n=None):
        """store_type='cpu' (legacy, gru4rec.py:605-614): samples are drawn by NumPy on the host, one store at a time."""
        costs = [np.zeros(0, np.float32)]
        done, end = first, sched.n_steps if n is None else first + n
        while done < end:
            if eng.get_sample_pointer() >= generate_length:
                eng.set_sample_store(self.generate_neg_samples(pop, generate_length))
            n = min(end - done, generate_length - eng.get_sample_pointer())
            costs.append(eng.train_steps(sched, done, n))
            done += n
        return np.concatenate(costs)

    def _train_epoch_per_step_samples(self, eng, sched, pop, first=0, n=None):
        """store_type='cpu' without a store (gru4rec.py:612-613): one host draw of n_sample items per mini-batch."""
        costs = [np.zeros(0, np.float32)]
        for k in range(first, sched.n_steps if n is None else first + n):
            row = np.asarray(self.generate_neg_samples(pop, 1)).reshape(1, self.n_sample)
            eng.set_sample_store(np.vstack([row, row]))
            eng.set_sample_pointer(0)
            costs.append(eng.train_steps(sched, k, 1))
        return np.concatenate(costs)

    # ---- serving (gru4rec.py:665-728) ----
    def predict_next_batch(self, session_ids, input_item_ids, predict_for_item_ids=None, batch=100):
        '''
        Gives prediction scores for a selected set of items; same contract as the reference
        (gru4rec.py:665-728): hidden state kept per batch coordinate while the session id stays the same.
        Returns a DataFrame, rows = items, columns = events of the batch.
        '''
        if self.error_during_train: raise Exception
        eng, reset, in_idxs = self._next_batch_inputs(session_ids, input_item_ids, batch)
        preds = eng.predict(in_idxs, reset.astype(np.uint8)).T          # items x batch
        if predict_for_item_ids is not None:
            iIdxs = self.itemidmap[predict_for_item_ids].values
            preds = preds[iIdxs]
            if self.final_act in ('softmax', 'softmax_logit'):
                preds = preds / preds.sum(axis=0, keepdims=True)          # softmax over the requested subset
            return pd.DataFrame(data=preds, index=predict_for_item_ids)
        return pd.DataFrame(data=preds, index=self.itemidmap.index)

    def recommend_next_batch(self, session_ids, input_item_ids, k=20, batch=100, items=None, exclude=None, exclude_seen=False):
        '''
        The k best next items of every event of the batch, ranked on the device (an addition to the reference's surface).
        Shares predict_next_batch's per-lane session state, so the two methods can be called alternately.
        Returns (item_ids [batch, k] of the original item IDs, scores [batch, k] float32), best first.  Order: the score
        (the pre-activation score for softmax / softmax_logit), then the earlier item of the catalogue; the scores are the
        values predict_next_batch returns for those items.

        Filters, applied on the device:
          items         original item IDs: only these compete (as predict_for_item_ids; unknown IDs raise KeyError, duplicates
                        are ignored; softmax scores are normalised over them); k must not exceed their number
          exclude       one iterable of original item IDs (or None) per lane, never recommended to that lane (unknown IDs
                        are ignored)
          exclude_seen  also exclude every item fed into the lane since its session began, this call's input included
        With a filter, a lane with fewer than k eligible items is padded with item None and score NaN (the ID array is then
        of object dtype).
        '''
        if self.error_during_train: raise Exception
        k = _lib.check_topk(k, self.n_items)
        cand = None
        if items is not None:
            cand = self.itemidmap[items].values
            n_cand = len(np.unique(cand))
            if k > n_cand:
                raise ValueError('k = %d exceeds the %d distinct candidate items' % (k, n_cand))
        if exclude is not None and len(exclude) != batch:
            raise ValueError('exclude must hold one entry per lane (%d), got %d' % (batch, len(exclude)))
        eng, reset, in_idxs = self._next_batch_inputs(session_ids, input_item_ids, batch)
        if cand is None and exclude is None and not exclude_seen:
            out, scores = eng.predict_topk(in_idxs, k, reset.astype(np.uint8))
            return self.itemidmap.index.to_numpy()[out], scores
        excl = [self._item_indices(e) for e in exclude] if exclude is not None else [np.zeros(0, np.int64)] * batch
        if exclude_seen:
            excl = [np.concatenate([e, self._seen[b, :self._seen_n[b]]]) for b, e in enumerate(excl)]
        out, scores = eng.predict_topk(in_idxs, k, reset.astype(np.uint8), items=cand, exclude=excl)
        ids = self.itemidmap.index.to_numpy()
        miss = out < 0
        if not miss.any():
            return ids[out], scores
        res = ids[np.where(miss, 0, out)].astype(object)
        res[miss] = None
        return res, scores

    def _item_indices(self, item_ids):
        '''item indices of the known IDs among item_ids (unknown IDs are dropped)'''
        if item_ids is None:
            return np.zeros(0, np.int64)
        pos = self.itemidmap.index.get_indexer(pd.Index(list(item_ids)))
        return self.itemidmap.values[pos[pos >= 0]].astype(np.int64)

    def _next_batch_inputs(self, session_ids, input_item_ids, batch):
        '''session bookkeeping of predict_next_batch / recommend_next_batch: the hidden state of a lane is
        kept while its session id stays the same and zeroed when it changes or the batch size changes.  The items fed
        into each lane since its session began are kept alongside (_seen [batch, cap] + _seen_n, for exclude_seen) and
        cleared at the same points.'''
        eng = self._ensure_engine(batch)
        if getattr(self, 'predict', None) is None or self.predict_batch != batch:
            self.predict_batch = batch
            eng.reset_eval_hidden()
            self.current_session = np.ones(batch) * -1
            self.predict = True
            self._seen = np.zeros((batch, 8), dtype=np.int64)
            self._seen_n = np.zeros(batch, dtype=np.int64)
        session_ids = np.asarray(session_ids)
        reset = (session_ids != self.current_session)
        if reset.any():
            self.current_session = session_ids.copy()
        in_idxs = self.itemidmap[input_item_ids].values
        self._seen_n[reset] = 0
        if self._seen_n.max() >= self._seen.shape[1]:          # grow by doubling
            self._seen = np.concatenate([self._seen, np.zeros_like(self._seen)], axis=1)
        self._seen[np.arange(batch), self._seen_n] = in_idxs
        self._seen_n += 1
        return eng, reset, in_idxs

    # ---- serving by session key (an addition to the reference surface; DESIGN §3e) ----
    # The hidden state of every session lives in a device-resident store of the scoring engine, addressed by session id: events
    # of any number of interleaved sessions can arrive in any order and any call size.  Session ids are integers (the store's
    # keys are int64); string ids must be factorized by the caller.  The store holds `session_capacity` sessions; when a new
    # session needs room, the least recently used session not named in the call is dropped (its next event starts afresh).
    # The store survives rebuilds of the scoring engine and set_value(); fit() and loadmodel() start without sessions, and it
    # is never pickled.
    def recommend_sessions(self, session_ids, input_item_ids, k=20, items=None, exclude=None, exclude_seen=False):
        '''
        Session session_ids[i] has just seen item input_item_ids[i]: advances its state and returns its k best next items.
        A session id may appear at most once per call (ValueError); a session not in the store starts from a zero state.
        Returns (item_ids [n, k] of the original item IDs, scores [n, k] float32), best first, ranked as recommend_next_batch ranks
        a lane.  Filters as in recommend_next_batch, per event: `items` (original item IDs competing), `exclude` (one iterable of
        original item IDs or None per event), `exclude_seen` (every item fed to the session since it entered the store, this
        input included).  With a filter, missing places are padded with item None and score NaN.
        '''
        if self.error_during_train: raise Exception
        keys = self._session_keys(session_ids)
        k = _lib.check_topk(k, self.n_items)
        in_idxs = self._session_inputs(keys, input_item_ids)
        if len(np.unique(keys)) != len(keys):
            raise ValueError('a session id appears more than once in the call (feed_sessions takes repeated ids)')
        cand = None
        if items is not None:
            cand = self.itemidmap[items].values
            n_cand = len(np.unique(cand))
            if k > n_cand:
                raise ValueError('k = %d exceeds the %d distinct candidate items' % (k, n_cand))
        if exclude is not None and len(exclude) != len(keys):
            raise ValueError('exclude must hold one entry per event (%d), got %d' % (len(keys), len(exclude)))
        excl = None if exclude is None else [self._item_indices(e) for e in exclude]
        eng = self._session_engine()
        out, scores = eng.sessions_topk(keys, in_idxs, k, items=cand, exclude=excl, exclude_seen=exclude_seen)
        ids = self.itemidmap.index.to_numpy()
        miss = out < 0
        if not miss.any():
            return ids[out], scores
        res = ids[np.where(miss, 0, out)].astype(object)
        res[miss] = None
        return res, scores

    def feed_sessions(self, session_ids, input_item_ids):
        '''Advances sessions by their events without scoring; session ids may repeat (a session's events apply in order).'''
        if self.error_during_train: raise Exception
        keys = self._session_keys(session_ids)
        in_idxs = self._session_inputs(keys, input_item_ids)
        self._session_engine().sessions_feed(keys, in_idxs)

    def end_sessions(self, session_ids=None):
        '''Drops the given sessions from the store (unknown ids are ignored), or every session.'''
        keys = None if session_ids is None else self._session_keys(session_ids)
        if self._engine is not None and self._engine.session_capacity is not None:
            self._engine.sessions_end(keys)

    def export_sessions(self):
        '''
        Every session in the store, least recently used first: (session_ids int64 [n], states float32 [n, sum(layers)] -- the
        layers' hidden states concatenated --, history: a list of n arrays of the original item IDs fed since the session entered).
        '''
        width = int(sum(self.layers))
        if self._engine is None or self._engine.session_capacity is None:
            return np.zeros(0, np.int64), np.zeros((0, width), np.float32), []
        keys, states, off, items = self._engine.sessions_export()
        ids = self.itemidmap.index.to_numpy()
        return keys, states, [ids[items[off[i]:off[i + 1]]] for i in range(len(keys))]

    def import_sessions(self, session_ids, states, history=None):
        '''
        Inserts sessions as the most recently used, in order (the layout of export_sessions); a session id already in the store is
        overwritten.  history: one iterable of original item IDs per session (unknown IDs raise KeyError), or None.
        '''
        keys = self._session_keys(session_ids)
        if len(np.unique(keys)) != len(keys):
            raise ValueError('a session id appears more than once')
        states = np.asarray(states, dtype=np.float32)
        width = int(sum(self.layers))
        if states.shape != (len(keys), width):
            raise ValueError('states must have shape (%d, %d), got %s' % (len(keys), width, states.shape))
        if len(keys) > int(self.session_capacity):
            raise ValueError('%d sessions exceed session_capacity = %d' % (len(keys), int(self.session_capacity)))
        off = items = None
        if history is not None:
            if len(history) != len(keys):
                raise ValueError('history must hold one entry per session (%d), got %d' % (len(keys), len(history)))
            parts = [self.itemidmap[list(h)].values.astype(np.int64) if len(h) else np.zeros(0, np.int64) for h in history]
            off = np.zeros(len(keys) + 1, np.int64)
            off[1:] = np.cumsum([len(p) for p in parts])
            items = np.concatenate(parts) if parts else np.zeros(0, np.int64)
        self._session_engine().sessions_import(keys, states, off, items)

    @staticmethod
    def _session_keys(session_ids):
        '''session ids as int64 keys; TypeError unless they are integers'''
        a = np.asarray(session_ids)
        if a.ndim != 1:
            a = a.reshape(-1)
        if a.size == 0:
            return np.zeros(0, np.int64)
        if a.dtype.kind not in 'iu' or (a.dtype.kind == 'u' and a.max() > np.iinfo(np.int64).max):
            raise TypeError('session ids must be integers that fit int64 (factorize other ids first), got dtype %s' % a.dtype)
        return a.astype(np.int64)

    def _session_inputs(self, keys, input_item_ids):
        '''item indices of the inputs (KeyError for an unknown item ID)'''
        if len(input_item_ids) != len(keys):
            raise ValueError('session_ids and input_item_ids differ in length (%d, %d)' % (len(keys), len(input_item_ids)))
        if len(keys) == 0:
            return np.zeros(0, np.int64)
        return self.itemidmap[input_item_ids].values

    def _session_engine(self):
        '''the scoring engine with its session store open at session_capacity (a changed capacity keeps the most recent
        sessions that fit)'''
        eng = self._ensure_engine(1)
        cap = int(self.session_capacity)
        if eng.session_capacity != cap:
            old = eng.sessions_export() if eng.session_capacity is not None else None
            eng.sessions_open(cap)
            if old is not None:
                keys, states, off, items = old
                first = max(0, len(keys) - cap)
                eng.sessions_import(keys[first:], states[first:], off[first:] - off[first], items[off[first]:])
        return eng

    # ---- persistence (gru4rec.py:742-781): pickle of the object with NumPy parameters ----
    def __getstate__(self):
        st = dict(self.__dict__)
        host = self._host if self._engine is None else self._pull_host()
        for k in ('_engine', 'Wx', 'Wh', 'Wrz', 'Bh', 'H', 'Wy', 'By', 'E', '_host'):
            st.pop(k, None)
        n = len(self.layers)
        st['Wx'] = [host['Wx%d' % i] for i in range(n)]
        st['Wh'] = [host['Wh%d' % i] for i in range(n)]
        st['Wrz'] = [host['Wrz%d' % i] for i in range(n)]
        st['Bh'] = [host['Bh%d' % i].reshape(-1) for i in range(n)]
        st['H'] = [np.zeros((self.batch_size, self.layers[i]), dtype=np.float32) for i in range(n)]
        st['Wy'] = host['Wy']
        st['By'] = host['By']
        if 'E' in host:
            st['E'] = host['E']
        # what the reference class needs after unpickling (its __init__ is not run): the bound graph builders, pickled by
        # name (gru4rec.py:136-161) -- with this class registered as gru4rec.GRU4Rec the reference resolves its own methods
        st['loss_function'] = getattr(self, {'cross-entropy': 'cross_entropy', 'bpr': 'bpr', 'bpr-max': 'bpr_max', 'top1': 'top1',
                                             'top1-max': 'top1_max', 'xe_logit': 'cross_entropy_logits'}[self.loss])
        st['final_activation'] = self._act_object(self.final_act)
        st['hidden_activation'] = self._act_object(self.hidden_act)
        for k in ('device', 'dropout_seed', 'eval_lanes', 'step_mode', 'session_capacity', '_engine_eval_lanes', 'predict', 'predict_batch',
                  'current_session', '_seen', '_seen_n', '_engine_training', '_host_state'):
            st.pop(k, None)
        st['predict'] = None
        return st

    def _act_object(self, name):
        if name.startswith('leaky-'): return self.LeakyReLU(float(name.split('-')[1])).execute
        if name.startswith('elu-'): return self.Elu(float(name.split('-')[1])).execute
        if name.startswith('selu-'): return self.Selu(*[float(x) for x in name.split('-')[1:]]).execute
        return getattr(self, name)

    def __setstate__(self, st):
        st = dict(st)
        for k in ('loss_function', 'final_activation', 'hidden_activation'):   # bound Theano graph builders in reference pickles
            st.pop(k, None)
        self.__dict__.update(st)
        n = len(self.layers)
        host = {}
        for i in range(n):
            host['Wx%d' % i] = np.asarray(self.Wx[i], dtype=np.float32)
            host['Wh%d' % i] = np.asarray(self.Wh[i], dtype=np.float32)
            host['Wrz%d' % i] = np.asarray(self.Wrz[i], dtype=np.float32)
            host['Bh%d' % i] = np.asarray(self.Bh[i], dtype=np.float32).reshape(-1)
        host['Wy'] = np.asarray(self.Wy, dtype=np.float32)
        host['By'] = np.asarray(self.By, dtype=np.float32).reshape(-1, 1)
        if getattr(self, 'embedding', 0) and not getattr(self, 'constrained_embedding', False) and 'E' in st:
            host['E'] = np.asarray(self.E, dtype=np.float32)
        self._host = host
        self._engine = None
        self.predict = None
        for k, v in (('device', 0), ('dropout_seed', 0), ('eval_lanes', 512), ('step_mode', 2), ('session_capacity', 100000), ('bptt', 1), ('full_softmax', False)):
            if not hasattr(self, k):
                setattr(self, k, v)

    def savemodel(self, fname):
        with open(fname, 'wb') as f:
            pickle.dump(self, f)

    @classmethod
    def loadmodel(cls, fname):
        return pd.read_pickle(fname)


# Pickles name the class by module path.  The reference's models are `gru4rec.GRU4Rec`; registering this class under the
# same path makes pickles interchangeable in both directions (reference-written pickles load here; pickles written here
# load into the reference class, whose own graph builders are resolved by name).
GRU4Rec.__module__ = 'gru4rec'
GRU4Rec.__qualname__ = 'GRU4Rec'
for _n in ('Selu', 'Elu', 'LeakyReLU'):
    getattr(GRU4Rec, _n).__module__ = 'gru4rec'
    getattr(GRU4Rec, _n).__qualname__ = 'GRU4Rec.' + _n
import sys as _sys
if 'gru4rec' not in _sys.modules:
    import types as _types
    _m = _types.ModuleType('gru4rec')
    _m.GRU4Rec = GRU4Rec
    _sys.modules['gru4rec'] = _m
