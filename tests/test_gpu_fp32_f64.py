"""-m gpu: the fp32 training kernels -- k_fast (step_mode 2), its cluster variant (step_mode 3), k_persistent (step_mode 1 and the
fallback of modes 2 / 3) and the per-phase sequence (step_mode 0) -- and the device optimizers, step by step against a float64
oracle (gpu_utils.f64_run_steps): every product the kernel keeps, every gradient (plain SGD, recovered from the update) or every
update of the weights and the optimizer state (any other optimizer, from random non-zero state)."""
import numpy as np
import pytest
from gpu_utils import f64_setup, f64_run_steps, f64_failures

pytestmark = pytest.mark.gpu


def _mk(L, B, loss, fact, S=2048, **kw):
    mk = dict(layers=list(L) if isinstance(L, (list, tuple)) else [L], batch_size=B, n_sample=S, loss=loss, final_act=fact, adapt=None,
              learning_rate=0.5, momentum=0.0, sample_alpha=0.5)
    mk.update(kw)
    return mk


ADAGRAD = dict(adapt='adagrad', learning_rate=0.05)
FAST = dict(per_item=8)      # the heavy duplicates of step 2 in groups of 8: a chunk stays within the role-specialised kernels' 32 columns
P = 'persistent'

# name -> (model keywords, n_items, {step_mode: kernel path, or one per step (gpu_utils.STEP_PATHS)}, f64_step_inputs keywords).
# No embedding unless stated; 2048 samples = 132 column chunks on an H100.  Every optimizer case also runs step_mode 2 once: the
# role-specialised kernels take SGD / Adagrad only, so that is the generic path.
CASES = {
    # ---- role-specialised kernels (k_fast / cluster variant) ----
    'fast_L100_B32_bprmax': (_mk(100, 32, 'bpr-max', 'elu-0.5', bpreg=1.95), 5000, {2: 'fast', 3: 'fast'}, FAST),
    # the widest layer of k_fast's 48-CTA GRU group
    'fast_L120_xe_logq_drop': (_mk(120, 32, 'cross-entropy', 'softmax', logq=1.0, dropout_p_hidden=0.3), 4000, {2: 'fast'}, FAST),
    # only the cluster variant takes L = 128: step_mode 2 falls back to k_persistent
    'fast_L128_top1max': (_mk(128, 32, 'top1-max', 'tanh'), 4000, {3: 'fast', 2: P}, FAST),
    # L % 4 != 0, odd batch; the Adagrad + momentum + L2 epilogue
    'fast_L50_B13_top1_adagrad': (_mk(50, 13, 'top1', 'tanh', momentum=0.3, lmbd=1e-3, **ADAGRAD), 6000, {2: 'fast', 3: 'fast'}, FAST),
    # the headline catalogue
    'fast_L64_B16_xelogit_full': (_mk(64, 16, 'xe_logit', 'softmax_logit'), 37483, {2: 'fast'}, FAST),
    # step 1 has a duplicate group of 40 columns, wider than a chunk of k_fast (FK_CT = 32): that window falls back
    'fast_L100_wide_group': (_mk(100, 32, 'bpr-max', 'elu-0.5'), 3000, {2: [P, 'fast']}, dict(FAST, wide_group=40)),
    # ---- generic kernels ----
    # the shipped rsc15 shape (constrained embedding); step_mode 2 falls back (k_fast takes no embedding)
    'shared_rsc15': (_mk(100, 32, 'cross-entropy', 'softmax', constrained_embedding=True, logq=1.0, dropout_p_hidden=0.4, momentum=0.2, **ADAGRAD),
                     8000, {0: 'phases', 1: P, 2: P}, dict(input_in_scores=True)),
    'shared_rsc15_sgd': (_mk(100, 32, 'cross-entropy', 'softmax', constrained_embedding=True, logq=1.0, dropout_p_hidden=0.4), 8000,
                         {0: 'phases', 1: P, 2: P}, dict(input_in_scores=True)),
    'embed64_L96_100_bprmax_drop': (_mk([96, 100], 32, 'bpr-max', 'elu-0.5', embedding=64, dropout_p_hidden=0.2, dropout_p_embed=0.3),
                                    5000, {0: 'phases', 1: P}, {}),
    'none_3x40_relu_top1max': (_mk([40, 40, 40], 24, 'top1-max', 'tanh', S=512, hidden_act='relu'), 3000, {0: 'phases', 1: P}, {}),
    # B = 64: past k_fast's 32 lanes
    'shared_L128_B64_bpr': (_mk(128, 64, 'bpr', 'linear', constrained_embedding=True), 6000, {0: 'phases', 1: P}, dict(input_in_scores=True)),
    # ---- device optimizers ----
    'adam_none_L64_xe': (_mk(64, 32, 'cross-entropy', 'softmax', adapt='adam', adapt_params=[0.9, 0.999], learning_rate=0.01), 4000,
                         {0: 'phases', 1: P, 2: P}, {}),
    'adam_embed32_2layer_mom_l2': (_mk([48, 64], 32, 'bpr-max', 'elu-0.5', embedding=32, adapt='adam', adapt_params=[0.9, 0.999],
                                       learning_rate=0.01, momentum=0.3, lmbd=1e-3), 4000, {0: 'phases', 1: P, 2: P}, {}),
    'rmsprop_none_mom_l2': (_mk(80, 32, 'top1-max', 'tanh', adapt='rmsprop', adapt_params=[0.9], learning_rate=0.01, momentum=0.3,
                                lmbd=1e-3), 4000, {0: 'phases', 1: P, 2: P}, {}),
    'adadelta_embed48': (_mk(64, 32, 'cross-entropy', 'softmax', embedding=48, adapt='adadelta', adapt_params=[0.95], learning_rate=0.5),
                         4000, {0: 'phases', 1: P, 2: P}, {}),
    # grad_cap below the gradient norm: every recovered gradient is g * cap / norm (checked: the scale is < 1)
    'gradcap_low_sgd': (_mk(64, 32, 'bpr-max', 'elu-0.5', grad_cap=1e-3), 4000, {0: 'phases', 1: 'phases', 2: 'phases'}, {}),
    # grad_cap above the norm: the scale is exactly 1
    'gradcap_high_adagrad': (_mk(64, 32, 'bpr-max', 'elu-0.5', grad_cap=1e3, **ADAGRAD), 4000, {0: 'phases', 2: 'phases'}, {}),
    'smooth_xe': (_mk(64, 32, 'cross-entropy', 'softmax', smoothing=0.1), 4000, {0: 'phases', 1: 'phases', 2: 'phases'}, {}),
    'smooth_xelogit': (_mk(64, 32, 'xe_logit', 'softmax_logit', smoothing=0.1), 4000, {0: 'phases', 1: 'phases', 2: 'phases'}, {}),
    'rmsprop_cap_smooth_embed': (_mk(64, 32, 'cross-entropy', 'softmax', embedding=48, adapt='rmsprop', adapt_params=[0.9], learning_rate=0.01,
                                     grad_cap=1e-2, smoothing=0.1), 4000, {0: 'phases', 2: 'phases'}, {}),
}
PARAMS = [(name, sm) for name in CASES for sm in CASES[name][2]]


@pytest.mark.parametrize('name,step_mode', PARAMS, ids=['%s-mode%d' % p for p in PARAMS])
def test_fp32_step_matches_float64(name, step_mode):
    """Two steps (M = B; then M < B, a reset lane, a duplicated input, a target among the samples and heavily duplicated samples)
    of each kernel against a float64 oracle re-seeded from the device before each step: the cost, y / H / dvec of every layer,
    dSx, the DSY rows the kernel writes, and -- plain SGD -- every gradient recovered from the update, or -- any other optimizer --
    the updates of every weight and optimizer state.  The handle's counters show which kernel ran.  Failures are listed as
    'max err / max |ref|  /  max relative err above 1 % of max' against the bar of gpu_utils.F64_REL / F64_RTOL (4e-5 / 1e-3).
    Worst tensor per family -- the device on an H100 80GB HBM3 (400 W power limit); a float32 run of the oracle on the same inputs:
    role-specialised 6.5e-7 / 1.2e-5, 2.9e-6 / 6.9e-5; generic kernels 1.3e-6 / 2.5e-5, 8.7e-6 / 2.8e-4; optimizers 1.0e-6 /
    1.7e-5, 1.1e-5 / 2.0e-4.  With deliberate defects: k_fast's dWrz x 1.02, the smoothing statistics merged over the first 32
    chunks only, the DBY term left out of the grad_cap norm, rmsprop / adadelta state decayed once per duplicate, adam's sparse
    bias correction with the old count, and the shared-mode input rows reading the live Wy.acc -- each fails cases here."""
    mk, n_items, modes, inputs = CASES[name]
    eng, store, steps, P0 = f64_setup(mk, n_items, step_mode, **inputs)
    checks, _, scales = f64_run_steps(eng, mk, n_items, store, steps, P0, modes[step_mode])
    failed = f64_failures(checks)
    assert not failed, '\n'.join(failed)
    if mk.get('grad_cap', 0) and mk['grad_cap'] < 1:
        assert max(scales) < 1, scales
    elif mk.get('grad_cap', 0):
        assert scales == [1.0, 1.0], scales
    eng.close()
