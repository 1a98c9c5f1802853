"""ctypes binding of libg4r.so (include/g4r.h).  There is no CPU path: loading fails loudly if the
library is missing, and creating a handle fails loudly if no CUDA device is visible."""
import ctypes as C
import math
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libg4r.so')
G4R_MAX_LAYERS = 8
G4R_TOPK_MAX = 1024
SCHED_POSITIONS = 2          # Schedule(mode=1 | SCHED_POSITIONS): an evaluation schedule that records input positions

G4R_OK, G4R_ERR_INVALID, G4R_ERR_INDEX, G4R_ERR_CUDA, G4R_ERR_NAN, G4R_ERR_STATE = 0, -1, -2, -3, -4, -5
LOSS = {'cross-entropy': 0, 'bpr-max': 1, 'top1-max': 2, 'bpr': 3, 'top1': 4, 'xe_logit': 5}
ACT = {'linear': 0, 'relu': 1, 'tanh': 2, 'leaky': 3, 'elu': 4, 'selu': 5, 'softmax': 6, 'softmax_logit': 7}
ADAPT = {None: 0, 'adagrad': 1, 'rmsprop': 2, 'adadelta': 3, 'adam': 4}


class G4RConfig(C.Structure):
    _fields_ = [
        ('n_items', C.c_int32), ('n_layers', C.c_int32), ('layers', C.c_int32 * G4R_MAX_LAYERS), ('batch_size', C.c_int32),
        ('embedding', C.c_int32), ('constrained_embedding', C.c_int32), ('loss', C.c_int32),
        ('final_act', C.c_int32), ('final_act_p1', C.c_float), ('final_act_p2', C.c_float),
        ('hidden_act', C.c_int32), ('hidden_act_p1', C.c_float), ('hidden_act_p2', C.c_float),
        ('dropout_p_hidden', C.c_float), ('dropout_p_embed', C.c_float),
        ('learning_rate', C.c_float), ('momentum', C.c_float), ('lmbd', C.c_float),
        ('n_sample', C.c_int32), ('sample_alpha', C.c_float),
        ('smoothing', C.c_float), ('bpreg', C.c_float), ('logq', C.c_float),
        ('adapt', C.c_int32), ('sample_store', C.c_int32), ('dropout_seed', C.c_uint32), ('mrg_seed', C.c_uint32),
        ('max_resident_steps', C.c_int32), ('device', C.c_int32), ('world_size', C.c_int32), ('rank', C.c_int32),
        ('eval_batch_size', C.c_int32), ('step_mode', C.c_int32), ('mg_replicated', C.c_int32), ('eval_tc', C.c_int32),
        ('adapt_p1', C.c_float), ('adapt_p1c', C.c_float), ('adapt_p2', C.c_float), ('adapt_p2c', C.c_float), ('grad_cap', C.c_float),
        ('bptt', C.c_int32), ('full_softmax', C.c_int32),
    ]


EXPORTS = [
    'g4r_version', 'g4r_workspace_bytes', 'g4r_create', 'g4r_destroy', 'g4r_last_error', 'g4r_stream',
    'g4r_tensor_shape', 'g4r_set_tensor', 'g4r_get_tensor', 'g4r_reset_hidden',
    'g4r_set_sampling_cdf', 'g4r_set_logq_support', 'g4r_generate_samples', 'g4r_generate_samples_from_uniform',
    'g4r_set_sample_store', 'g4r_get_sample_store', 'g4r_sample_store_rows', 'g4r_set_sample_pointer', 'g4r_get_sample_pointer',
    'g4r_mrg_uniform', 'g4r_searchsorted', 'g4r_gather_rows',
    'g4r_schedule_build', 'g4r_schedule_build_history', 'g4r_schedule_free', 'g4r_schedule_steps', 'g4r_schedule_events', 'g4r_schedule_export', 'g4r_schedule_positions',
    'g4r_train_step', 'g4r_train_steps', 'g4r_upload_steps', 'g4r_run_uploaded', 'g4r_kernel_launches',
    'g4r_profile_uploaded', 'g4r_phase_name', 'g4r_phase_count', 'g4r_persistent_stamps', 'g4r_fast_windows', 'g4r_bptt_windows', 'g4r_full_steps', 'g4r_uses_tensor_cores', 'g4r_mg_unique_id', 'g4r_mg_init',
    'g4r_mg_sharded', 'g4r_mg_ipc_handle', 'g4r_mg_ipc_open', 'g4r_mg_owner', 'g4r_mg_local_row', 'g4r_mg_shard_rows', 'g4r_mg_segment_bytes',
    'g4r_eval_schedule', 'g4r_eval_events', 'g4r_eval_rest', 'g4r_eval_rest_pairs', 'g4r_eval_counts', 'g4r_set_eval_items', 'g4r_set_eval_exclude_seen', 'g4r_predict', 'g4r_reset_eval_hidden',
    'g4r_predict_topk', 'g4r_predict_topk_filtered',
    'g4r_sessions_open', 'g4r_sessions_count', 'g4r_sessions_feed', 'g4r_sessions_topk', 'g4r_sessions_end',
    'g4r_sessions_export', 'g4r_sessions_import',
    'g4r_train_state_bytes', 'g4r_train_state_export', 'g4r_train_state_import', 'g4r_copy_item_tables',
    'g4r_bl_create', 'g4r_bl_destroy', 'g4r_bl_last_error', 'g4r_bl_knn_fit', 'g4r_bl_set_pop', 'g4r_bl_rows_export',
    'g4r_bl_rows_import', 'g4r_bl_evaluate', 'g4r_bl_bpr_begin', 'g4r_bl_bpr_iterate', 'g4r_bl_bpr_export', 'g4r_bl_bpr_import',
    'g4r_bl_sknn_fit', 'g4r_bl_stan_fit', 'g4r_bl_stan_set_w1', 'g4r_bl_rules_fit', 'g4r_bl_vstan_set',
    'g4r_bl_narm_begin', 'g4r_bl_narm_epoch', 'g4r_bl_narm_grads', 'g4r_bl_narm_export', 'g4r_bl_narm_import', 'g4r_bl_narm_encode',
    'g4r_bl_sasrec_begin', 'g4r_bl_sasrec_epoch', 'g4r_bl_sasrec_grads', 'g4r_bl_sasrec_export', 'g4r_bl_sasrec_import',
    'g4r_bl_sasrec_encode', 'g4r_bl_srgnn_begin', 'g4r_bl_srgnn_epoch', 'g4r_bl_srgnn_grads', 'g4r_bl_srgnn_export',
    'g4r_bl_srgnn_import', 'g4r_bl_srgnn_encode', 'g4r_bl_stamp_begin', 'g4r_bl_stamp_epoch', 'g4r_bl_stamp_grads', 'g4r_bl_stamp_export',
    'g4r_bl_stamp_import', 'g4r_bl_stamp_encode', 'g4r_bl_nextitnet_begin', 'g4r_bl_nextitnet_epoch', 'g4r_bl_nextitnet_grads',
    'g4r_bl_nextitnet_export', 'g4r_bl_nextitnet_import', 'g4r_bl_nextitnet_encode', 'g4r_bl_bert4rec_begin', 'g4r_bl_bert4rec_epoch',
    'g4r_bl_bert4rec_grads', 'g4r_bl_bert4rec_export', 'g4r_bl_bert4rec_import', 'g4r_bl_bert4rec_encode',
]

_lib = None


def load():
    """Load libg4r.so (built in-tree by gru4rec_b200/csrc/build.sh / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError('libg4r.so not found at %s: build it with gru4rec_b200/csrc/build.sh '
                           '(there is no CPU fallback)' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, f32p = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_float)
    lib.g4r_version.restype = C.c_int
    lib.g4r_workspace_bytes.argtypes = [C.POINTER(G4RConfig), C.POINTER(C.c_size_t)]
    lib.g4r_create.argtypes = [C.POINTER(G4RConfig), vp, C.c_size_t, C.POINTER(vp)]
    lib.g4r_destroy.argtypes = [vp]
    lib.g4r_last_error.argtypes = [vp]; lib.g4r_last_error.restype = C.c_char_p
    lib.g4r_stream.argtypes = [vp]; lib.g4r_stream.restype = vp
    lib.g4r_tensor_shape.argtypes = [vp, C.c_char_p, C.POINTER(i64), C.POINTER(i64)]
    lib.g4r_set_tensor.argtypes = [vp, C.c_char_p, vp, i64, i64]
    lib.g4r_get_tensor.argtypes = [vp, C.c_char_p, vp, i64, i64]
    lib.g4r_reset_hidden.argtypes = [vp]
    lib.g4r_set_sampling_cdf.argtypes = [vp, vp, i64]
    lib.g4r_set_logq_support.argtypes = [vp, vp, i64]
    lib.g4r_generate_samples.argtypes = [vp]
    lib.g4r_generate_samples_from_uniform.argtypes = [vp, vp, i64]
    lib.g4r_set_sample_store.argtypes = [vp, vp, i64]
    lib.g4r_get_sample_store.argtypes = [vp, vp, i64]
    lib.g4r_sample_store_rows.argtypes = [vp]
    lib.g4r_set_sample_pointer.argtypes = [vp, i64]
    lib.g4r_get_sample_pointer.argtypes = [vp]; lib.g4r_get_sample_pointer.restype = i64
    lib.g4r_mrg_uniform.argtypes = [vp, vp, i64]
    lib.g4r_searchsorted.argtypes = [vp, vp, i64, vp, i64, vp]
    lib.g4r_gather_rows.argtypes = [vp, vp, i64, i64, vp, i64, vp]
    lib.g4r_schedule_build.argtypes = [vp, i64, vp, i64, vp, i32, i32, i32, C.POINTER(vp)]
    lib.g4r_schedule_build_history.argtypes = [vp, i64, vp, i64, vp, vp, i32, i32, C.POINTER(vp)]
    lib.g4r_schedule_free.argtypes = [vp]
    lib.g4r_schedule_steps.argtypes = [vp]; lib.g4r_schedule_steps.restype = i64
    lib.g4r_schedule_events.argtypes = [vp]; lib.g4r_schedule_events.restype = i64
    lib.g4r_schedule_export.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.g4r_schedule_positions.argtypes = [vp, vp]
    lib.g4r_train_step.argtypes = [vp, vp, vp, i32, vp, C.POINTER(C.c_float)]
    lib.g4r_train_steps.argtypes = [vp, vp, i64, i64, vp, C.POINTER(i64)]
    lib.g4r_upload_steps.argtypes = [vp, vp, i64, i64]
    lib.g4r_run_uploaded.argtypes = [vp, vp, C.POINTER(C.c_float)]
    lib.g4r_kernel_launches.argtypes = [vp]; lib.g4r_kernel_launches.restype = i64
    lib.g4r_profile_uploaded.argtypes = [vp, vp, vp, i32]
    lib.g4r_phase_name.argtypes = [i32]; lib.g4r_phase_name.restype = C.c_char_p
    lib.g4r_phase_count.restype = C.c_int
    lib.g4r_persistent_stamps.argtypes = [vp, i32, vp, i64]
    lib.g4r_fast_windows.argtypes = [vp, C.POINTER(i64)]; lib.g4r_fast_windows.restype = i64
    lib.g4r_bptt_windows.argtypes = [vp]; lib.g4r_bptt_windows.restype = i64
    lib.g4r_full_steps.argtypes = [vp]; lib.g4r_full_steps.restype = i64
    lib.g4r_uses_tensor_cores.argtypes = [vp]
    lib.g4r_mg_unique_id.argtypes = [vp]
    lib.g4r_mg_init.argtypes = [vp, vp]
    lib.g4r_mg_sharded.argtypes = [vp]
    lib.g4r_mg_ipc_handle.argtypes = [vp, vp]
    lib.g4r_mg_ipc_open.argtypes = [vp, vp, i32]
    lib.g4r_mg_owner.argtypes = [i64, i32]
    lib.g4r_mg_local_row.argtypes = [i64, i32]; lib.g4r_mg_local_row.restype = i64
    lib.g4r_mg_shard_rows.argtypes = [i64, i32, i32]; lib.g4r_mg_shard_rows.restype = i64
    lib.g4r_mg_segment_bytes.argtypes = [C.POINTER(G4RConfig), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.g4r_eval_schedule.argtypes = [vp, vp, vp, i32, i32, vp, vp, C.POINTER(i64)]
    lib.g4r_eval_events.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, C.POINTER(i64), vp, vp, vp]
    lib.g4r_eval_rest.argtypes = [vp, vp, vp, i32, i32, vp, C.POINTER(i64), C.POINTER(i64), vp, vp]
    lib.g4r_eval_rest_pairs.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    lib.g4r_eval_counts.argtypes = [vp, vp, i64]
    lib.g4r_set_eval_items.argtypes = [vp, vp, i64]
    lib.g4r_set_eval_exclude_seen.argtypes = [vp, i32]
    lib.g4r_predict.argtypes = [vp, vp, i32, vp, vp]
    lib.g4r_reset_eval_hidden.argtypes = [vp]
    lib.g4r_predict_topk.argtypes = [vp, vp, i32, vp, i32, vp, vp]
    lib.g4r_predict_topk_filtered.argtypes = [vp, vp, i32, vp, i32, vp, i64, vp, vp, vp, vp]
    lib.g4r_sessions_open.argtypes = [vp, i64]
    lib.g4r_sessions_count.argtypes = [vp, C.POINTER(i64)]; lib.g4r_sessions_count.restype = i64
    lib.g4r_sessions_feed.argtypes = [vp, vp, vp, i64]
    lib.g4r_sessions_topk.argtypes = [vp, vp, vp, i64, i32, vp, i64, vp, vp, i32, vp, vp]
    lib.g4r_sessions_end.argtypes = [vp, vp, i64]
    lib.g4r_sessions_export.argtypes = [vp, vp, vp, vp, vp]
    lib.g4r_sessions_import.argtypes = [vp, vp, vp, vp, vp, i64]
    lib.g4r_train_state_bytes.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.g4r_train_state_export.argtypes = [vp, vp, C.c_size_t]
    lib.g4r_train_state_import.argtypes = [vp, vp, C.c_size_t]
    lib.g4r_copy_item_tables.argtypes = [vp, vp, vp, vp, vp]
    lib.g4r_bl_create.argtypes = [i32, i32, i32, i32, C.POINTER(vp)]
    lib.g4r_bl_destroy.argtypes = [vp]
    lib.g4r_bl_last_error.argtypes = [vp]; lib.g4r_bl_last_error.restype = C.c_char_p
    lib.g4r_bl_knn_fit.argtypes = [vp, vp, i64, vp, i64, vp, vp, C.POINTER(i64), C.POINTER(C.c_size_t), C.POINTER(C.c_float)]
    lib.g4r_bl_set_pop.argtypes = [vp, vp, i64]
    lib.g4r_bl_rows_export.argtypes = [vp, vp, vp, vp]
    lib.g4r_bl_rows_import.argtypes = [vp, vp, vp, vp]
    lib.g4r_bl_evaluate.argtypes = [vp, vp, i64, vp, i64, vp, i32, vp, i32, vp, i64, i32, i32, vp, vp, C.POINTER(i64), vp, vp, vp]
    lib.g4r_bl_bpr_begin.argtypes = [vp, vp, vp, i64, i64, vp, vp, vp]
    f64 = C.c_double
    lib.g4r_bl_bpr_iterate.argtypes = [vp, vp, vp, f64, f64, f64, i32, C.POINTER(f64), C.POINTER(i64), C.POINTER(C.c_float)]
    lib.g4r_bl_bpr_export.argtypes = [vp, vp, vp]
    lib.g4r_bl_bpr_import.argtypes = [vp, vp, vp]
    lib.g4r_bl_sknn_fit.argtypes = [vp, vp, i64, vp, i64, vp, i32, i32]
    lib.g4r_bl_stan_fit.argtypes = [vp, vp, i64, vp, i64, vp, vp, vp, vp, i64, i32]
    lib.g4r_bl_stan_set_w1.argtypes = [vp, vp, i64]
    lib.g4r_bl_vstan_set.argtypes = [vp, i32, vp, i64, vp, i64]
    lib.g4r_bl_rules_fit.argtypes = [vp, vp, i64, vp, i64, i32, i32, C.POINTER(i64), C.POINTER(C.c_size_t), C.POINTER(C.c_float)]
    u32, f32 = C.c_uint32, C.c_float
    lib.g4r_bl_narm_begin.argtypes = [vp, i32, i32, i32, vp, i64, vp, i64, vp, i64]
    lib.g4r_bl_narm_epoch.argtypes = [vp, vp, i64, u32, f32, f32, f32, vp, C.POINTER(C.c_float)]
    lib.g4r_bl_narm_grads.argtypes = [vp, vp, i32, u32, i64, f32, f32, C.POINTER(C.c_float), vp]
    lib.g4r_bl_narm_export.argtypes = [vp, vp, i64]
    lib.g4r_bl_narm_import.argtypes = [vp, i32, i32, vp, i64]
    lib.g4r_bl_narm_encode.argtypes = [vp, vp, i64, vp, i64, vp, vp, i64]
    lib.g4r_bl_sasrec_begin.argtypes = [vp, i32, i32, i32, i32, vp, i64, vp, i64, vp, i64]
    lib.g4r_bl_sasrec_epoch.argtypes = [vp, vp, i64, u32, f32, f32, vp, C.POINTER(C.c_float)]
    lib.g4r_bl_sasrec_grads.argtypes = [vp, vp, i32, u32, i64, f32, C.POINTER(C.c_float), vp]
    lib.g4r_bl_sasrec_export.argtypes = [vp, vp, i64]
    lib.g4r_bl_sasrec_import.argtypes = [vp, i32, i32, i32, vp, i64]
    lib.g4r_bl_sasrec_encode.argtypes = [vp, vp, i64, vp, i64, vp, vp, i64]
    lib.g4r_bl_srgnn_begin.argtypes = [vp, i32, i32, i32, vp, i64, vp, i64, vp, i64]
    lib.g4r_bl_srgnn_epoch.argtypes = [vp, vp, i64, f32, f32, vp, C.POINTER(C.c_float)]
    lib.g4r_bl_srgnn_grads.argtypes = [vp, vp, i32, C.POINTER(C.c_float), vp]
    lib.g4r_bl_srgnn_export.argtypes = [vp, vp, i64]
    lib.g4r_bl_srgnn_import.argtypes = [vp, i32, i32, vp, i64]
    lib.g4r_bl_srgnn_encode.argtypes = [vp, vp, i64, vp, i64, vp, vp, i64]
    lib.g4r_bl_stamp_begin.argtypes = [vp, i32, i32, vp, i64, vp, i64, vp, i64]
    lib.g4r_bl_stamp_epoch.argtypes = [vp, vp, i64, f32, vp, C.POINTER(C.c_float)]
    lib.g4r_bl_stamp_grads.argtypes = [vp, vp, i32, C.POINTER(C.c_float), vp]
    lib.g4r_bl_stamp_export.argtypes = [vp, vp, i64]
    lib.g4r_bl_stamp_import.argtypes = [vp, i32, vp, i64]
    lib.g4r_bl_stamp_encode.argtypes = [vp, vp, i64, vp, i64, vp, vp, i64]
    lib.g4r_bl_nextitnet_begin.argtypes = [vp, vp, i32, i32, i32, i32, vp, i64, vp, i64, vp, i64]
    lib.g4r_bl_nextitnet_epoch.argtypes = [vp, vp, i64, f32, vp, C.POINTER(C.c_float)]
    lib.g4r_bl_nextitnet_grads.argtypes = [vp, vp, i32, C.POINTER(C.c_float), vp]
    lib.g4r_bl_nextitnet_export.argtypes = [vp, vp, i64]
    lib.g4r_bl_nextitnet_import.argtypes = [vp, vp, i32, i32, i32, vp, i64]
    lib.g4r_bl_nextitnet_encode.argtypes = [vp, vp, i64, vp, i64, vp, vp, i64]
    lib.g4r_bl_bert4rec_begin.argtypes = [vp, i32, i32, i32, i32, vp, i64, vp, i64, vp, i64]
    lib.g4r_bl_bert4rec_epoch.argtypes = [vp, vp, i64, vp, i64, u32, f32, f32, vp, C.POINTER(C.c_float)]
    lib.g4r_bl_bert4rec_grads.argtypes = [vp, vp, i32, vp, i64, u32, i64, f32, C.POINTER(C.c_float), vp]
    lib.g4r_bl_bert4rec_export.argtypes = [vp, vp, i64]
    lib.g4r_bl_bert4rec_import.argtypes = [vp, i32, i32, i32, vp, i64]
    lib.g4r_bl_bert4rec_encode.argtypes = [vp, vp, i64, vp, i64, vp, vp, i64]
    _lib = lib
    return lib


class NaNError(ArithmeticError):
    def __init__(self, msg, step):
        ArithmeticError.__init__(self, msg)
        self.step = step


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def parse_act(name):
    """'elu-0.5' -> (ACT code, p1, p2)   (gru4rec.py:144-161)."""
    if name in ('linear', 'relu', 'tanh', 'softmax', 'softmax_logit'):
        return ACT[name], 0.0, 0.0
    if name.startswith('leaky-'):
        return ACT['leaky'], float(name.split('-')[1]), 0.0
    if name.startswith('elu-'):
        return ACT['elu'], float(name.split('-')[1]), 0.0
    if name.startswith('selu-'):
        p = [float(x) for x in name.split('-')[1:]]
        return ACT['selu'], p[0], p[1]
    raise NotImplementedError


SEEN_BUDGET = 256 << 20     # bytes of exclude_seen's device lists per evaluation call (g4r_set_eval_exclude_seen)


def seen_budget():
    """the library's budget for exclude_seen's lists: SEEN_BUDGET, lowered by G4R_SEEN_BUDGET in the environment (for tests)"""
    env = os.environ.get('G4R_SEEN_BUDGET')
    return SEEN_BUDGET if env is None else min(SEEN_BUDGET, max(0, int(env)))


def check_topk(k, n_items):
    """k of a top-k request: 1 <= k <= min(n_items, G4R_TOPK_MAX), else ValueError"""
    if not isinstance(k, (int, np.integer)) or isinstance(k, bool) or not 1 <= k <= min(n_items, G4R_TOPK_MAX):
        raise ValueError('k must be an integer in 1 .. min(n_items, %d) = %d, got %r' % (G4R_TOPK_MAX, min(n_items, G4R_TOPK_MAX), k))
    return int(k)


def set_adapt_params(cfg, adapt, adapt_params, grad_cap):
    """adapt_params as the reference uses them (gru4rec.py:301-304,342-343,368-369); the complements are taken in double like there"""
    ap = [float(x) for x in (adapt_params or [])]
    if adapt in ('rmsprop', 'adadelta') and len(ap) < 1 or adapt == 'adam' and len(ap) < 2:
        raise IndexError('list index out of range')          # what the reference raises when adapt_params is too short
    cfg.adapt_p1 = ap[0] if len(ap) > 0 else 0.0
    cfg.adapt_p1c = (1.0 - ap[0]) if len(ap) > 0 else 0.0
    cfg.adapt_p2 = ap[1] if len(ap) > 1 else 0.0
    cfg.adapt_p2c = (1.0 - ap[1]) if len(ap) > 1 else 0.0
    cfg.grad_cap = float(grad_cap or 0.0)


def make_config(n_items, mk, sample_store=0, eval_lanes=0, max_resident_steps=0, step_mode=0, world_size=1, rank=0, replicated=False, eval_tc=None, bptt=1, full_softmax=False):
    cfg = G4RConfig()
    layers = mk.get('layers', [100])
    cfg.n_items = n_items
    cfg.n_layers = len(layers)
    for i, l in enumerate(layers):
        cfg.layers[i] = l
    cfg.batch_size = mk.get('batch_size', 32)
    cfg.constrained_embedding = 1 if mk.get('constrained_embedding') else 0
    cfg.embedding = 0 if mk.get('constrained_embedding') else int(mk.get('embedding', 0) or 0)
    cfg.loss = LOSS[mk.get('loss', 'bpr-max')]
    cfg.final_act, cfg.final_act_p1, cfg.final_act_p2 = parse_act(mk.get('final_act', 'linear'))
    cfg.hidden_act, cfg.hidden_act_p1, cfg.hidden_act_p2 = parse_act(mk.get('hidden_act', 'tanh'))
    cfg.dropout_p_hidden = mk.get('dropout_p_hidden', 0.0)
    cfg.dropout_p_embed = mk.get('dropout_p_embed', 0.0)
    cfg.learning_rate = mk.get('learning_rate', 0.1)
    cfg.momentum = mk.get('momentum', 0.0)
    cfg.lmbd = mk.get('lmbd', 0.0)
    cfg.n_sample = mk.get('n_sample', 2048)
    cfg.sample_alpha = mk.get('sample_alpha', 0.75)
    cfg.smoothing = mk.get('smoothing', 0.0)
    cfg.bpreg = mk.get('bpreg', 1.0)
    cfg.logq = mk.get('logq', 0.0)
    cfg.adapt = ADAPT[mk.get('adapt', 'adagrad')]
    cfg.sample_store = sample_store
    cfg.dropout_seed = mk.get('dropout_seed', 0)
    cfg.mrg_seed = 12345
    cfg.max_resident_steps = max_resident_steps
    cfg.world_size, cfg.rank = world_size, rank
    cfg.eval_batch_size = eval_lanes
    cfg.step_mode = step_mode
    cfg.mg_replicated = 1 if replicated else 0     # multi-GPU: replicated tables + NCCL exchange instead of row sharding
    cfg.eval_tc = 0 if eval_tc is None else (2 if eval_tc else 1)   # scoring path: auto / force tensor-core tiles / force fp32 FFMA tiles
    set_adapt_params(cfg, mk.get('adapt', 'adagrad'), mk.get('adapt_params', []), mk.get('grad_cap', 0.0))
    cfg.bptt = bptt              # truncated backpropagation through time over windows of this many mini-batches (DESIGN §3l)
    cfg.full_softmax = 1 if full_softmax else 0      # train against the whole catalogue instead of sampled columns (DESIGN §3n)
    return cfg



class Schedule(object):
    """Host-side schedule of one epoch (gru4rec.py:594-651 / evaluation.py:90-139), built in C++.  n_history (evaluation
    schedules only): per session id, the number of its leading events that are history; only events whose target lies past
    them are counted (n_events, flag bit 4 of export()['F'], the outputs of eval_schedule / eval_events)."""

    def __init__(self, data_items, offset_sessions, session_order, batch_size, n_sample, mode=0, n_history=None):
        lib = load()
        self._lib = lib
        di = np.ascontiguousarray(data_items, dtype=np.int64)
        off = np.ascontiguousarray(offset_sessions, dtype=np.int32)
        order = None if session_order is None else np.ascontiguousarray(session_order, dtype=np.int64)
        h = C.c_void_p()
        # n_sessions = number of sessions this schedule walks: all of them, or the entries of a (possibly sharded) order
        n_sess = len(off) - 1 if order is None else len(order)
        if order is not None and len(order) and (order.min() < 0 or order.max() >= len(off) - 1):
            raise IndexError('session_order refers to a session that does not exist')
        if n_history is None:
            rc = lib.g4r_schedule_build(_ptr(di), len(di), _ptr(off), n_sess, _ptr(order), batch_size, n_sample, mode, C.byref(h))
        else:
            nh = np.ascontiguousarray(n_history, dtype=np.int32)
            if len(nh) != len(off) - 1 or n_sample != 0:
                raise ValueError('n_history needs one entry per session and an evaluation schedule')
            rc = lib.g4r_schedule_build_history(_ptr(di), len(di), _ptr(off), n_sess, _ptr(order), _ptr(nh), batch_size, mode, C.byref(h))
        if rc == G4R_ERR_INDEX:
            raise IndexError(lib.g4r_last_error(None).decode())
        if rc != 0:
            raise RuntimeError(lib.g4r_last_error(None).decode())
        self.h = h
        self.batch_size = batch_size
        self.history = n_history is not None
        self.n_steps = lib.g4r_schedule_steps(h)
        self.n_events = lib.g4r_schedule_events(h)

    def export(self):
        n, B = self.n_steps, self.batch_size
        X = np.empty((n, B), np.int32); Y = np.empty((n, B), np.int32); F = np.empty((n, B), np.uint8)
        M = np.empty(n, np.int32); S = np.empty((n, B), np.int32)
        self._lib.g4r_schedule_export(self.h, _ptr(X), _ptr(Y), _ptr(F), _ptr(M), _ptr(S))
        return dict(X=X, Y=Y, F=F, M=M, slots=S)

    def positions(self):
        """[n_steps, batch_size] int64 (schedules built with mode=1 | SCHED_POSITIONS): index in data_items of every lane's input,
        -1 on unused lanes; the lane's target is the next entry."""
        P = np.empty((self.n_steps, self.batch_size), np.int64)
        rc = self._lib.g4r_schedule_positions(self.h, _ptr(P))
        if rc != 0:
            raise RuntimeError(self._lib.g4r_last_error(None).decode())
        return P

    def counted(self):
        """[n_steps, batch_size] bool: the lanes whose event is counted (every used lane unless built with n_history), in the
        (step, lane) order eval_events numbers the events in."""
        e = self.export()
        used = np.arange(self.batch_size)[None, :] < e['M'][:, None]
        return used & ((e['F'] & 4) != 0) if self.history else used

    def batch_sizes(self):
        """M of every mini-batch (the weights of the epoch loss, gru4rec.py:654) without copying the index arrays."""
        M = np.empty(self.n_steps, np.int32)
        self._lib.g4r_schedule_export(self.h, None, None, None, _ptr(M), None)
        return M

    def __del__(self):
        try:
            if self.h:
                self._lib.g4r_schedule_free(self.h)
                self.h = None
        except Exception:
            pass


class Engine(object):
    """Owns one g4r_handle.  Device memory is allocated through torch (used only as an allocator)."""

    def __init__(self, cfg, device=0, use_torch_allocator=True):
        lib = load()
        self.lib = lib
        self.cfg = cfg
        cfg.device = device
        nbytes = C.c_size_t()
        rc = lib.g4r_workspace_bytes(C.byref(cfg), C.byref(nbytes))
        if rc != 0:
            raise NotImplementedError(lib.g4r_last_error(None).decode())
        self._ws = None
        ws_ptr = None
        if use_torch_allocator:
            import torch
            if not torch.cuda.is_available():
                raise RuntimeError('gru4rec_b200 needs a CUDA device (H100 / sm_90a); there is no CPU fallback')
            if cfg.full_softmax and torch.cuda.mem_get_info(device)[0] < nbytes.value:
                raise NotImplementedError('full_softmax: the training workspace needs %d bytes of device memory, %d are free on cuda:%d'
                                          % (nbytes.value, torch.cuda.mem_get_info(device)[0], device))
            self._ws = torch.empty(nbytes.value, dtype=torch.uint8, device='cuda:%d' % device)
            ws_ptr = C.c_void_p(self._ws.data_ptr())
        h = C.c_void_p()
        rc = lib.g4r_create(C.byref(cfg), ws_ptr, nbytes.value, C.byref(h))
        if rc != 0:
            msg = lib.g4r_last_error(None).decode()
            if rc == G4R_ERR_INVALID:
                raise NotImplementedError(msg)
            raise RuntimeError('g4r_create failed: ' + msg)
        self.h = h
        self.workspace_bytes = nbytes.value

    def close(self):
        if getattr(self, 'h', None):
            self.lib.g4r_destroy(self.h)
            self.h = None
            self._ws = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, nan_step=None):
        if rc == 0:
            return
        msg = self.lib.g4r_last_error(self.h).decode()
        if rc == G4R_ERR_INDEX:
            raise IndexError(msg)
        if rc == G4R_ERR_INVALID:
            raise NotImplementedError(msg)
        if rc == G4R_ERR_NAN:
            raise NaNError(msg, nan_step)
        raise RuntimeError('libg4r: %s (status %d)' % (msg, rc))

    # ---- tensors ----
    def shape(self, name):
        r, c = C.c_int64(), C.c_int64()
        self._check(self.lib.g4r_tensor_shape(self.h, name.encode(), C.byref(r), C.byref(c)))
        return r.value, c.value

    def set(self, name, arr):
        r, c = self.shape(name)
        a = np.ascontiguousarray(np.asarray(arr, dtype=np.float32).reshape(r, c))
        self._check(self.lib.g4r_set_tensor(self.h, name.encode(), _ptr(a), r, c))

    def get(self, name):
        r, c = self.shape(name)
        if name.split('.')[0] in ('Wy', 'By', 'Wx0'):
            self._quiesce()
        a = np.empty((r, c), dtype=np.float32)
        self._check(self.lib.g4r_get_tensor(self.h, name.encode(), _ptr(a), r, c))
        return a

    def reset_hidden(self):
        self._check(self.lib.g4r_reset_hidden(self.h))

    # ---- sampling ----
    def set_sampling_cdf(self, P):
        P = np.ascontiguousarray(P, dtype=np.float32)
        self._check(self.lib.g4r_set_sampling_cdf(self.h, _ptr(P), len(P)))

    def set_logq_support(self, P0):
        P0 = np.ascontiguousarray(P0, dtype=np.float32)
        self._check(self.lib.g4r_set_logq_support(self.h, _ptr(P0), len(P0)))

    def generate_samples(self):
        self._check(self.lib.g4r_generate_samples(self.h))

    def generate_samples_from_uniform(self, u):
        u = np.ascontiguousarray(u, dtype=np.float32)
        self._check(self.lib.g4r_generate_samples_from_uniform(self.h, _ptr(u), u.size))

    def sample_store_rows(self):
        return self.lib.g4r_sample_store_rows(self.h)

    def set_sample_store(self, st):
        st = np.ascontiguousarray(st, dtype=np.int64)
        self._check(self.lib.g4r_set_sample_store(self.h, _ptr(st), st.shape[0]))

    def get_sample_store(self):
        rows = self.sample_store_rows()
        st = np.empty((rows, self.cfg.n_sample), dtype=np.int64)
        self._check(self.lib.g4r_get_sample_store(self.h, _ptr(st), rows))
        return st

    def set_sample_pointer(self, p):
        self._check(self.lib.g4r_set_sample_pointer(self.h, p))

    def get_sample_pointer(self):
        return self.lib.g4r_get_sample_pointer(self.h)

    def mrg_uniform(self, n):
        out = np.empty(n, dtype=np.float32)
        self._check(self.lib.g4r_mrg_uniform(self.h, _ptr(out), n))
        return out

    # ---- stand-alone ops ----
    def searchsorted(self, d, x):
        d = np.ascontiguousarray(d, dtype=np.float32); x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty(x.shape, dtype=np.int64)
        self._check(self.lib.g4r_searchsorted(self.h, _ptr(d), d.size, _ptr(x), x.size, _ptr(y)))
        return y

    def gather_rows(self, table, idx):
        table = np.ascontiguousarray(table, dtype=np.float32); idx = np.ascontiguousarray(idx, dtype=np.int64)
        out = np.empty((idx.size, table.shape[1]), dtype=np.float32)
        self._check(self.lib.g4r_gather_rows(self.h, _ptr(table), table.shape[0], table.shape[1], _ptr(idx), idx.size, _ptr(out)))
        return out

    # ---- training ----
    def train_step(self, X, Y, R=None):
        X = np.ascontiguousarray(X, dtype=np.int32); Y = np.ascontiguousarray(Y, dtype=np.int32)
        Rp = None if R is None else np.ascontiguousarray(np.asarray(R).reshape(-1), dtype=np.int8)
        cost = C.c_float()
        self._check(self.lib.g4r_train_step(self.h, _ptr(X), _ptr(Y), len(X), _ptr(Rp), C.byref(cost)))
        return np.float32(cost.value)

    def train_steps(self, sched, first=0, n=None):
        n = sched.n_steps - first if n is None else n
        if self.cfg.world_size > 1:
            # ranks advance in lock step (one merged update per mini-batch): a different n would dead-lock the collectives
            import torch
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                dev = 'cuda' if dist.get_backend() == 'nccl' else 'cpu'
                t = torch.tensor([n, -n], dtype=torch.int64, device=dev)
                dist.all_reduce(t, op=dist.ReduceOp.MIN)
                if int(t[0]) != n or int(-t[1]) != n:
                    raise ValueError('train_steps: every rank must run the same number of steps (got %d, range %d..%d)' % (n, int(t[0]), int(-t[1])))
        costs = np.empty(n, dtype=np.float32)
        nan_step = C.c_int64(-1)
        rc = self.lib.g4r_train_steps(self.h, sched.h, first, n, _ptr(costs), C.byref(nan_step))
        self._check(rc, nan_step.value)
        return costs

    def upload_steps(self, sched, first, n):
        self._check(self.lib.g4r_upload_steps(self.h, sched.h, first, n))

    def run_uploaded(self, n, want_cost=True):
        costs = np.empty(n, dtype=np.float32) if want_cost else None
        ms = C.c_float()
        self._check(self.lib.g4r_run_uploaded(self.h, _ptr(costs), C.byref(ms)))
        return costs, ms.value

    def profile_uploaded(self):
        """{phase name: (total device ms, launches)} for one pass over the uploaded window."""
        n = self.lib.g4r_phase_count()
        ms = np.zeros(n, dtype=np.float32); cnt = np.zeros(n, dtype=np.int32)
        self._check(self.lib.g4r_profile_uploaded(self.h, _ptr(ms), _ptr(cnt), n))
        return {self.lib.g4r_phase_name(i).decode(): (float(ms[i]), int(cnt[i])) for i in range(n) if cnt[i] > 0}

    def persistent_stamps(self, enable=True, n_steps=0):
        out = np.zeros((n_steps, 16), dtype=np.uint64) if n_steps > 0 else None
        self._check(self.lib.g4r_persistent_stamps(self.h, 1 if enable else 0, _ptr(out), n_steps))
        return out

    def init_multi_gpu(self, dist):
        """Create the NCCL communicator of this handle: rank 0's unique id is broadcast through torch.distributed."""
        import torch
        buf = (C.c_char * 128)()
        if dist.get_rank() == 0:
            rc = self.lib.g4r_mg_unique_id(buf)
            if rc != 0:
                raise RuntimeError('ncclGetUniqueId failed')
        t = torch.tensor(list(bytes(buf)), dtype=torch.uint8, device='cuda' if dist.get_backend() == 'nccl' else 'cpu')
        dist.broadcast(t, 0)
        raw = bytes(t.cpu().tolist())
        idbuf = (C.c_char * 128).from_buffer_copy(raw)
        self._check(self.lib.g4r_mg_init(self.h, idbuf))
        self._dist = dist
        if self.sharded():
            # row-sharded tables: every rank maps the segments of all peers (cudaIpc); the 64-byte handles travel by all-gather
            mh = (C.c_char * 64)()
            self._check(self.lib.g4r_mg_ipc_handle(self.h, mh))
            dev = 'cuda' if dist.get_backend() == 'nccl' else 'cpu'
            mine = torch.tensor(list(bytes(mh)), dtype=torch.uint8, device=dev)
            allh = [torch.empty_like(mine) for _ in range(dist.get_world_size())]
            dist.all_gather(allh, mine)
            raw = b''.join(bytes(t.cpu().tolist()) for t in allh)
            buf2 = (C.c_char * len(raw)).from_buffer_copy(raw)
            self._check(self.lib.g4r_mg_ipc_open(self.h, buf2, dist.get_world_size()))
            dist.barrier()

    def sharded(self):
        return bool(self.lib.g4r_mg_sharded(self.h))

    def _quiesce(self):
        """sharded tensors are assembled from all ranks' memory: every rank must have finished its device work"""
        d = getattr(self, '_dist', None)
        if d is not None and self.sharded():
            import torch
            torch.cuda.synchronize()
            d.barrier()

    def uses_tensor_cores(self):
        return bool(self.lib.g4r_uses_tensor_cores(self.h))

    def fast_windows(self):
        fb = C.c_int64()
        n = self.lib.g4r_fast_windows(self.h, C.byref(fb))
        return n, fb.value

    def bptt_windows(self):
        """windows trained with truncated backpropagation through time (bptt > 1)"""
        return self.lib.g4r_bptt_windows(self.h)

    def full_steps(self):
        """training steps run against the whole catalogue (full_softmax)"""
        return self.lib.g4r_full_steps(self.h)

    def kernel_launches(self):
        return self.lib.g4r_kernel_launches(self.h)

    def stream(self):
        return self.lib.g4r_stream(self.h)

    # ---- training state (g4r_train_state_*, g4r_copy_item_tables; DESIGN §3i) ----
    def train_state_export(self):
        """uint8 array: the global step, sample pointer and MRG stream states of the handle -- with the named tensors and the
        sample store, everything a new handle needs to continue this one's run bit for bit"""
        n = C.c_size_t()
        self._check(self.lib.g4r_train_state_bytes(self.h, C.byref(n)))
        blob = np.zeros(n.value, dtype=np.uint8)
        self._check(self.lib.g4r_train_state_export(self.h, _ptr(blob), n.value))
        return blob

    def train_state_import(self, blob):
        """Takes over a train_state_export() blob (after set_sample_store, which rewinds the pointer).  A blob that is truncated,
        of another version, or exported with another n_sample / store size / seed raises NotImplementedError and changes nothing."""
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        self._check(self.lib.g4r_train_state_import(self.h, _ptr(blob), blob.size))

    def copy_item_tables(self, src, new_Wy=None, new_By=None, new_in=None):
        """Device-to-device copy of every parameter, optimizer-state tensor and training hidden state of Engine `src`, whose
        catalogue is a prefix of this one's: the item tables keep src's rows and take new_Wy / new_By / new_in (E, or Wx0 of a
        model without embedding) in the added rows, zero where None; added rows of the optimizer state are zero."""
        n_add = int(self.cfg.n_items) - int(src.cfg.n_items)

        def block(name, a):
            return None if a is None or n_add <= 0 else np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(n_add, self.shape(name)[1]))
        wy, by = block('Wy', new_Wy), block('By', new_By)
        nin = None if self.cfg.constrained_embedding else block('E' if self.cfg.embedding else 'Wx0', new_in)
        self._check(self.lib.g4r_copy_item_tables(self.h, src.h, _ptr(wy), _ptr(by), _ptr(nin)))

    # ---- scoring ----
    def eval_schedule(self, sched, cut_off, mode=0):
        cut = np.ascontiguousarray(cut_off, dtype=np.int32)
        rec = np.zeros(len(cut), dtype=np.float64); mrr = np.zeros(len(cut), dtype=np.float64)
        n = C.c_int64()
        self._check(self.lib.g4r_eval_schedule(self.h, sched.h, _ptr(cut), len(cut), mode, _ptr(rec), _ptr(mrr), C.byref(n)))
        return rec, mrr, n.value

    def eval_events(self, sched, cut_off, mode=0, k=0):
        """eval_schedule with per-event outputs, events in the order the schedule consumes them (Schedule.positions maps them to
        the data): (recall sums, mrr sums, n_events, counts int32 [n_events, 2], items int32 [n_events, k], scores float32
        [n_events, k]).  The sums equal eval_schedule's bit for bit; counts are (#greater, #equal) as eval_counts gives them; with
        k > 0 every event's top-k list as predict_topk ranks the lane after the input (with set_eval_items, among those items);
        k = 0: items / scores are None.  With set_eval_exclude_seen(True) an event whose target its session has already input
        counts (-1, -1), and the lists leave out the session's inputs (item -1, score NaN past the eligible items)."""
        cut = np.ascontiguousarray(cut_off, dtype=np.int32)
        rec = np.zeros(len(cut), dtype=np.float64); mrr = np.zeros(len(cut), dtype=np.float64)
        n = C.c_int64()
        counts = np.empty((sched.n_events, 2), dtype=np.int32)
        items = scores = None
        if k:
            items = np.empty((sched.n_events, k), dtype=np.int32); scores = np.empty((sched.n_events, k), dtype=np.float32)
        self._check(self.lib.g4r_eval_events(self.h, sched.h, _ptr(cut), len(cut), mode, int(k), _ptr(rec), _ptr(mrr), C.byref(n),
                                             _ptr(counts), _ptr(items), _ptr(scores)))
        return rec, mrr, n.value, counts, items, scores

    def eval_rest(self, sched, cut_off, mode=0):
        """Rest-of-session ranking of the schedule's counted events (schedules built with mode=1 | SCHED_POSITIONS): every
        distinct later item of an event's session ranked as if it were the target, under set_eval_items / set_eval_exclude_seen
        (a seen or unlisted item is a miss, counts (-1, -1)).  Returns (sums float64 [6, n_cut]: per cut-off the sums of
        HitRate, Precision, Recall, MRR, NDCG and MAP over the events; n_events; n_pairs; counts int32 [n_pairs, 2] in the event
        order of eval_events, each event's items in first-occurrence order; offsets int64 [n_events + 1] of each event's pairs).
        Over the relevant-list budget (lanes x longest session - 1 int32 within 256 MiB): NotImplementedError."""
        cut = np.ascontiguousarray(cut_off, dtype=np.int32)
        ne, npairs = C.c_int64(), C.c_int64()
        if self.lib.g4r_eval_rest_pairs(sched.h, C.byref(ne), C.byref(npairs)) != 0:
            raise RuntimeError('libg4r: %s' % self.lib.g4r_last_error(None).decode())
        counts = np.empty((npairs.value, 2), dtype=np.int32)
        offsets = np.empty(ne.value + 1, dtype=np.int64)
        sums = np.zeros(6 * len(cut), dtype=np.float64)
        n, n_pairs = C.c_int64(), C.c_int64()
        self._check(self.lib.g4r_eval_rest(self.h, sched.h, _ptr(cut), len(cut), mode, _ptr(sums), C.byref(n), C.byref(n_pairs),
                                           _ptr(counts), _ptr(offsets)))
        return sums.reshape(6, len(cut)), n.value, n_pairs.value, counts, offsets

    def eval_counts(self, n_lanes):
        """[n_lanes x 2] int32: (#items scoring above the target, #items tied with it incl. the target) of every lane of the last
        mini-batch ranked by eval_schedule (a diagnostic of the ranking kernels)."""
        out = np.zeros((n_lanes, 2), dtype=np.int32)
        self._check(self.lib.g4r_eval_counts(self.h, _ptr(out), n_lanes))
        return out

    def set_eval_items(self, items=None):
        """Candidate item indices for eval_schedule (evaluate_gpu(items=...)); None / empty restores the whole catalogue."""
        if items is None or len(items) == 0:
            self._check(self.lib.g4r_set_eval_items(self.h, None, 0))
            return
        it = np.ascontiguousarray(items, dtype=np.int64)
        self._check(self.lib.g4r_set_eval_items(self.h, _ptr(it), it.size))

    def set_eval_exclude_seen(self, on):
        """exclude_seen for later eval_schedule / eval_events calls: each event is ranked without the items its session has
        input so far (the current input included); a target among them is a miss.  A schedule whose seen lists (lanes x longest
        session - 1 int32) exceed 256 MiB is refused (NotImplementedError from G4R_ERR_INVALID) before any device work."""
        self._check(self.lib.g4r_set_eval_exclude_seen(self.h, 1 if on else 0))

    def predict(self, X, reset_mask=None):
        X = np.ascontiguousarray(X, dtype=np.int32)
        rm = None if reset_mask is None else np.ascontiguousarray(reset_mask, dtype=np.uint8)
        out = np.empty((len(X), self.cfg.n_items), dtype=np.float32)
        self._check(self.lib.g4r_predict(self.h, _ptr(X), len(X), _ptr(rm), _ptr(out)))
        return out

    def predict_topk(self, X, k, reset_mask=None, items=None, exclude=None):
        """predict() reduced on the device to the k best items of every lane: (items int32 [batch, k], scores float32 [batch, k]),
        best first.  Order: the activated score (the pre-activation score for softmax), then the smaller item index; the scores
        are predict()'s values.  Advances the hidden state exactly as predict() does.

        Filters (g4r_predict_topk_filtered): `items`, an array of item indices, restricts the ranking to its distinct items (the
        softmax normaliser then runs over them); `exclude`, one int array (or None) per lane, removes those items from that
        lane's list.  A lane with fewer than k eligible items gets them best first, then item -1 with score NaN."""
        X = np.ascontiguousarray(X, dtype=np.int32)
        rm = None if reset_mask is None else np.ascontiguousarray(reset_mask, dtype=np.uint8)
        if items is None and exclude is None:
            k = check_topk(k, self.cfg.n_items)
            out_i = np.empty((len(X), k), dtype=np.int32)
            out_s = np.empty((len(X), k), dtype=np.float32)
            self._check(self.lib.g4r_predict_topk(self.h, _ptr(X), len(X), _ptr(rm), k, _ptr(out_i), _ptr(out_s)))
            return out_i, out_s
        k, cand, off, ex = self._topk_filters(len(X), k, items, exclude)
        out_i = np.empty((len(X), k), dtype=np.int32)
        out_s = np.empty((len(X), k), dtype=np.float32)
        self._check(self.lib.g4r_predict_topk_filtered(self.h, _ptr(X), len(X), _ptr(rm), k, _ptr(cand), 0 if cand is None else cand.size,
                                                       _ptr(off), _ptr(ex), _ptr(out_i), _ptr(out_s)))
        return out_i, out_s

    def _topk_filters(self, n, k, items, exclude):
        """k checked against the candidates, and the filter arrays of g4r_predict_topk_filtered / g4r_sessions_topk: candidate
        item indices (or None), exclusion offsets [n + 1] and items (or None)"""
        cand = None
        n_distinct = self.cfg.n_items
        if items is not None:
            cand = np.asarray(items, dtype=np.int64).reshape(-1)
            if cand.size and (cand.min() < 0 or cand.max() >= self.cfg.n_items):
                raise IndexError('candidate item index out of range')
            cand = np.ascontiguousarray(cand, dtype=np.int32)
            n_distinct = int(np.count_nonzero(np.bincount(cand, minlength=self.cfg.n_items)))
        k = check_topk(k, n_distinct)
        off = ex = None
        if exclude is not None:
            if len(exclude) != n:
                raise ValueError('exclude must hold one entry per lane (%d), got %d' % (n, len(exclude)))
            parts = [np.asarray(e if e is not None else [], dtype=np.int64).reshape(-1) for e in exclude]
            off = np.zeros(n + 1, dtype=np.int64)
            off[1:] = np.cumsum([len(p) for p in parts])
            ex = np.concatenate(parts) if parts else np.zeros(0, np.int64)
            if ex.size and (ex.min() < 0 or ex.max() >= self.cfg.n_items):
                raise IndexError('excluded item index out of range')
            ex = np.ascontiguousarray(ex, dtype=np.int32)
        return k, cand, off, ex

    def reset_eval_hidden(self):
        self._check(self.lib.g4r_reset_eval_hidden(self.h))

    # ---- session store (g4r_sessions_*, DESIGN §3e) ----
    session_capacity = None       # capacity of the open store (None: not opened)

    def sessions_open(self, capacity):
        """(Re)creates an empty session store of `capacity` sessions."""
        self._check(self.lib.g4r_sessions_open(self.h, int(capacity)))
        self.session_capacity = int(capacity)

    def sessions_count(self):
        """(number of sessions, total length of their histories)"""
        nh = C.c_int64()
        n = self.lib.g4r_sessions_count(self.h, C.byref(nh))
        self._check(int(n) if n < 0 else 0)
        return int(n), nh.value

    def sessions_feed(self, keys, X):
        """Advances session keys[i] by item index X[i] without scoring (keys may repeat; a key's events apply in order)."""
        keys = np.ascontiguousarray(keys, dtype=np.int64); X = np.ascontiguousarray(X, dtype=np.int32)
        if keys.shape != X.shape:
            raise ValueError('keys and X differ in length')
        self._check(self.lib.g4r_sessions_feed(self.h, _ptr(keys), _ptr(X), keys.size))

    def sessions_topk(self, keys, X, k, items=None, exclude=None, exclude_seen=False):
        """predict_topk for sessions addressed by key (distinct within a call): advances session keys[i] by item index X[i] and
        returns its k best next items (items int32 [n, k], scores float32 [n, k]).  Filters as in predict_topk; exclude_seen
        also excludes the items fed to the session since it entered the store, this input included."""
        keys = np.ascontiguousarray(keys, dtype=np.int64); X = np.ascontiguousarray(X, dtype=np.int32)
        if keys.shape != X.shape:
            raise ValueError('keys and X differ in length')
        k, cand, off, ex = self._topk_filters(keys.size, k, items, exclude)
        out_i = np.empty((keys.size, k), dtype=np.int32)
        out_s = np.empty((keys.size, k), dtype=np.float32)
        self._check(self.lib.g4r_sessions_topk(self.h, _ptr(keys), _ptr(X), keys.size, k, _ptr(cand), 0 if cand is None else cand.size,
                                               _ptr(off), _ptr(ex), 1 if exclude_seen else 0, _ptr(out_i), _ptr(out_s)))
        return out_i, out_s

    def sessions_end(self, keys=None):
        """Drops the given sessions (unknown keys ignored), or every session."""
        if keys is None:
            self._check(self.lib.g4r_sessions_end(self.h, None, 0))
            return
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        self._check(self.lib.g4r_sessions_end(self.h, _ptr(keys), keys.size))

    def sessions_export(self):
        """Every session, least recently used first: keys int64 [n], states float32 [n, sum of layer widths], history offsets
        int64 [n + 1] and items int32."""
        n, nh = self.sessions_count()
        Lsum = int(sum(self.cfg.layers[i] for i in range(self.cfg.n_layers)))
        keys = np.empty(n, np.int64); states = np.empty((n, Lsum), np.float32)
        off = np.empty(n + 1, np.int64); items = np.empty(nh, np.int32)
        self._check(self.lib.g4r_sessions_export(self.h, _ptr(keys), _ptr(states), _ptr(off), _ptr(items)))
        return keys, states, off, items

    def sessions_import(self, keys, states, hist_off=None, hist_items=None):
        """Inserts sessions in order as the most recently used (layouts of sessions_export); existing keys are overwritten."""
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        Lsum = int(sum(self.cfg.layers[i] for i in range(self.cfg.n_layers)))
        states = np.ascontiguousarray(np.asarray(states, dtype=np.float32).reshape(keys.size, Lsum))
        off = None if hist_off is None else np.ascontiguousarray(hist_off, dtype=np.int64)
        it = None if hist_items is None else np.ascontiguousarray(hist_items, dtype=np.int32)
        if off is not None and off.size != keys.size + 1:
            raise ValueError('hist_off must have %d entries' % (keys.size + 1))
        self._check(self.lib.g4r_sessions_import(self.h, _ptr(keys), _ptr(states), _ptr(off), _ptr(it), keys.size))


BASELINE_KINDS = {'pop': 0, 'sessionpop': 1, 'itemknn': 2, 'bpr': 3, 'sknn': 5, 'stan': 6, 'sr': 8, 'ar': 9, 'vstan': 11, 'narm': 12, 'sasrec': 13, 'srgnn': 15, 'stamp': 17,
                  'nextitnet': 19, 'bert4rec': 21}
SKNN_SIMILARITY = {'cosine': 0, 'vector': 1}
RULES_WEIGHTING = {'div': 0, 'same': 1}
RULES_STEPS_MAX = 20
KEEP_MAX = 1024             # n_sims / k / pruning bound of the row-keeping baselines


def rules_scale(steps, weighting):
    """L of a rules fit: lcm(1 .. steps) for SR 'div' (every L / d is an integer), 1 for SR 'same' and for AR (steps None)"""
    L = 1
    if steps is not None and weighting == 'div':
        for d in range(2, steps + 1):
            L = L * d // math.gcd(L, d)
    return L


def rules_bound(session_offsets, items, n_items, steps, weighting):
    """the largest per-row bound of a rules fit's uint64 counts, as a Python int: SR occurrences * min(steps, longest session -
    1) * L, AR (steps None) the sum of n_s over the row item's occurrences"""
    off = np.asarray(session_offsets, dtype=np.int64)
    it = np.asarray(items, dtype=np.int64)
    lens = np.diff(off)
    if not it.size:
        return 0
    if steps is None:
        o = np.argsort(it, kind='stable')
        _, first = np.unique(it[o], return_index=True)
        return int(np.add.reduceat(np.repeat(lens, lens)[o], first).max())    # < 2^62 for fewer than 2^31 events
    occ = int(np.bincount(it, minlength=n_items).max())
    return occ * min(steps, max(int(lens.max()) - 1, 0)) * rules_scale(steps, weighting)


class Baselines(object):
    """Owns one g4r_baselines handle (DESIGN §3j): the fitted ItemKNN rows or Pop scores on the device, and the evaluation of
    a baseline, the BPR-MF fit and factors (DESIGN §3k), the SessionKNN, STAN and VSTAN indexes (DESIGN §3o, §3p, §3r), and the
    SR / AR fit into ItemKNN's rows (DESIGN §3q), and the NARM, SASRec, SR-GNN, STAMP, NextItNet and BERT4Rec fits and parameters
    (DESIGN §3s, §3t, §3u, §3v, §3w, §3x).  kind: 'pop', 'sessionpop', 'itemknn', 'bpr', 'sknn', 'stan', 'sr', 'ar', 'vstan', 'narm',
    'sasrec', 'srgnn', 'stamp', 'nextitnet' or 'bert4rec'; n_keep: top_n, n_sims, n_factors, k, pruning or embedding."""

    def __init__(self, kind, n_items, n_keep, device=0):
        lib = load()
        self.lib = lib
        self.kind, self.n_items, self.n_keep = kind, int(n_items), int(n_keep)
        h = C.c_void_p()
        rc = lib.g4r_bl_create(BASELINE_KINDS[kind], self.n_items, self.n_keep, device, C.byref(h))
        if rc != 0:
            msg = lib.g4r_bl_last_error(None).decode()
            raise (ValueError if rc == G4R_ERR_INVALID else RuntimeError)('g4r_bl_create: ' + msg)
        self.h = h

    def close(self):
        if getattr(self, 'h', None):
            self.lib.g4r_bl_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc == 0:
            return
        msg = self.lib.g4r_bl_last_error(self.h).decode()
        if rc == G4R_ERR_INDEX:
            raise IndexError(msg)
        if rc == G4R_ERR_INVALID:
            raise ValueError(msg)
        raise RuntimeError('libg4r: %s (status %d)' % (msg, rc))

    def knn_fit(self, session_offsets, items, a, b):
        """ItemKNN rows from the training events (session CSR of item indices) and the norm factors; returns
        (pair work, scratch bytes, fit kernel ms)"""
        off = np.ascontiguousarray(session_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        a = np.ascontiguousarray(a, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
        if a.size != self.n_items or b.size != self.n_items:
            raise ValueError('a and b need n_items entries')
        pw, sb, ms = C.c_int64(), C.c_size_t(), C.c_float()
        self._check(self.lib.g4r_bl_knn_fit(self.h, _ptr(off), off.size - 1, _ptr(it), it.size, _ptr(a), _ptr(b), C.byref(pw), C.byref(sb), C.byref(ms)))
        return pw.value, sb.value, ms.value

    def set_pop(self, scores):
        sc = np.ascontiguousarray(scores, dtype=np.float64)
        self._check(self.lib.g4r_bl_set_pop(self.h, _ptr(sc), sc.size))

    def rows_export(self):
        """(idx int32 [n_items, n_keep], sim float64 [n_items, n_keep], len int32 [n_items])"""
        idx = np.empty((self.n_items, self.n_keep), np.int32); sim = np.empty((self.n_items, self.n_keep), np.float64)
        ln = np.empty(self.n_items, np.int32)
        self._check(self.lib.g4r_bl_rows_export(self.h, _ptr(idx), _ptr(sim), _ptr(ln)))
        return idx, sim, ln

    def rows_import(self, idx, sim, ln):
        idx = np.ascontiguousarray(np.asarray(idx, dtype=np.int32).reshape(self.n_items, self.n_keep))
        sim = np.ascontiguousarray(np.asarray(sim, dtype=np.float64).reshape(self.n_items, self.n_keep))
        ln = np.ascontiguousarray(ln, dtype=np.int32)
        if ln.size != self.n_items:
            raise ValueError('len needs n_items entries')
        self._check(self.lib.g4r_bl_rows_import(self.h, _ptr(idx), _ptr(sim), _ptr(ln)))

    def evaluate(self, items, session_offsets, n_history, cut_off, mode, cand=None, exclude_seen=False, k=0, counts=True):
        """(recall sums, mrr sums, n_counted, counts int32 [n, 2] or None, items int32 [n, k] or None, scores float64 [n, k] or
        None), events in data order (g4r_bl_evaluate)"""
        it = np.ascontiguousarray(items, dtype=np.int32); off = np.ascontiguousarray(session_offsets, dtype=np.int64)
        nh = None if n_history is None else np.ascontiguousarray(n_history, dtype=np.int32)
        cut = np.ascontiguousarray(cut_off, dtype=np.int32)
        cd = None if cand is None else np.ascontiguousarray(cand, dtype=np.int32)
        lens = np.diff(off)
        n = int(np.maximum(0, lens - np.maximum(nh if nh is not None else 0, 1)).sum()) if lens.size else 0
        rec = np.zeros(len(cut)); mrr = np.zeros(len(cut)); nc = C.c_int64()
        cnt = np.empty((n, 2), np.int32) if counts else None
        ti = np.empty((n, k), np.int32) if k else None
        ts = np.empty((n, k), np.float64) if k else None
        self._check(self.lib.g4r_bl_evaluate(self.h, _ptr(it), it.size, _ptr(off), off.size - 1, _ptr(nh), int(mode), _ptr(cut), cut.size,
                                             _ptr(cd), 0 if cd is None else cd.size, 1 if exclude_seen else 0, int(k),
                                             _ptr(rec), _ptr(mrr), C.byref(nc), _ptr(cnt), _ptr(ti), _ptr(ts)))
        return rec, mrr, nc.value, cnt, ti, ts

    def bpr_begin(self, row_session, row_item, n_sessions, U, I, bI):
        """starts a BPR fit: the merged training rows' session and item indices and the initial U [n_sessions, F], I, bI"""
        rs = np.ascontiguousarray(row_session, dtype=np.int32); ri = np.ascontiguousarray(row_item, dtype=np.int32)
        U = np.ascontiguousarray(U, dtype=np.float64); I = np.ascontiguousarray(I, dtype=np.float64)
        bI = np.ascontiguousarray(bI, dtype=np.float64)
        if rs.size != ri.size or U.shape != (int(n_sessions), self.n_keep) or I.shape != (self.n_items, self.n_keep) or bI.size != self.n_items:
            raise ValueError('bpr_begin: need rows of equal length, U [n_sessions, n_factors], I [n_items, n_factors], bI [n_items]')
        if rs.size < self.n_items:
            raise ValueError('bpr_begin: need n_rows >= n_items (the negative draws index rows below n_items)')
        self._check(self.lib.g4r_bl_bpr_begin(self.h, _ptr(rs), _ptr(ri), rs.size, int(n_sessions), _ptr(U), _ptr(I), _ptr(bI)))
        self.bpr_rows, self.bpr_sessions = rs.size, int(n_sessions)

    def bpr_iterate(self, perm, negrow, learning_rate, lambda_session, lambda_item, max_warps=1 << 30):
        """one SGD pass in perm order with negative rows negrow; returns (mean log sigm, largest level, device ms)"""
        pm = np.asarray(perm)
        ng = np.asarray(negrow)
        if pm.shape != (self.bpr_rows,) or ng.shape != (self.bpr_rows,):
            raise ValueError('bpr_iterate: perm and negrow need one entry per training row')
        if pm.size and (pm.min() < 0 or pm.max() >= self.bpr_rows or ng.min() < 0 or ng.max() >= min(self.n_items, self.bpr_rows)):
            raise IndexError('bpr_iterate: perm must index the rows and negrow must be below min(n_items, n_rows)')
        pm = np.ascontiguousarray(pm, dtype=np.int32); ng = np.ascontiguousarray(ng, dtype=np.int32)
        mean, lv, ms = C.c_double(), C.c_int64(), C.c_float()
        self._check(self.lib.g4r_bl_bpr_iterate(self.h, _ptr(pm), _ptr(ng), float(learning_rate), float(lambda_session), float(lambda_item),
                                                int(min(max_warps, 1 << 30)), C.byref(mean), C.byref(lv), C.byref(ms)))
        return mean.value, lv.value, ms.value

    def bpr_export(self):
        """(U [n_sessions, F], I [n_items, F]) of the fit"""
        U = np.empty((self.bpr_sessions, self.n_keep)); I = np.empty((self.n_items, self.n_keep))
        self._check(self.lib.g4r_bl_bpr_export(self.h, _ptr(U), _ptr(I)))
        return U, I

    def bpr_import(self, I, bI):
        """the item factors and biases a BPR is evaluated with (a model loaded from a pickle)"""
        I = np.ascontiguousarray(I, dtype=np.float64); bI = np.ascontiguousarray(bI, dtype=np.float64)
        if I.shape != (self.n_items, self.n_keep) or bI.size != self.n_items:
            raise ValueError('bpr_import: need I [n_items, n_factors] and bI [n_items]')
        self._check(self.lib.g4r_bl_bpr_import(self.h, _ptr(I), _ptr(bI)))

    def sknn_fit(self, session_offsets, items, recency, sample_size, similarity):
        """the SessionKNN index: the training sessions' distinct items ascending as CSR, each session's recency rank (0: most
        recent), sample_size and 'cosine' / 'vector'"""
        off = np.ascontiguousarray(session_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        rc = np.ascontiguousarray(recency, dtype=np.int32)
        if rc.size != off.size - 1:
            raise ValueError('sknn_fit: need one recency rank per session')
        if similarity not in SKNN_SIMILARITY:
            raise ValueError('sknn_fit: similarity must be one of %s' % sorted(SKNN_SIMILARITY))
        self._check(self.lib.g4r_bl_sknn_fit(self.h, _ptr(off), off.size - 1, _ptr(it), it.size, _ptr(rc), int(sample_size),
                                             SKNN_SIMILARITY[similarity]))

    def stan_fit(self, session_offsets, items, positions, recency, w2, w3, sample_size):
        """the STAN (or VSTAN) index: sknn_fit's CSR and ranks, each entry's last position in its session, W2 per session (in the order of
        session_offsets) and the W3 table"""
        off = np.ascontiguousarray(session_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        pos = np.ascontiguousarray(positions, dtype=np.int32); rc = np.ascontiguousarray(recency, dtype=np.int32)
        w2 = np.ascontiguousarray(w2, dtype=np.float64); w3 = np.ascontiguousarray(w3, dtype=np.float64)
        if off.ndim != 1 or off.size < 2 or it.ndim != 1 or pos.shape != it.shape:
            raise ValueError('stan_fit: need session offsets and one position per item entry')
        if rc.shape != (off.size - 1,) or w2.shape != (off.size - 1,):
            raise ValueError('stan_fit: need one recency rank and one w2 weight per session')
        if w3.ndim != 1 or w3.size < 1:
            raise ValueError('stan_fit: w3 must be a non-empty 1-D table')
        self._check(self.lib.g4r_bl_stan_fit(self.h, _ptr(off), off.size - 1, _ptr(it), it.size, _ptr(pos), _ptr(rc), _ptr(w2), _ptr(w3),
                                             w3.size, int(sample_size)))

    def rules_fit(self, session_offsets, items, steps=None, weighting=None):
        """SR (steps 1 .. 20, weighting 'div' / 'same') or AR (steps and weighting None) rows from the training events as session
        CSR of item indices in time order; returns (pair work, scratch bytes, fit kernel ms).  Refuses a fit whose per-row bound
        (rules_bound) reaches 2^63 before the library is called."""
        if not 1 <= self.n_keep <= KEEP_MAX:
            raise ValueError('rules_fit: pruning must be in 1 .. %d, not %r' % (KEEP_MAX, self.n_keep))
        if self.kind == 'ar':
            if steps is not None or weighting is not None:
                raise ValueError('rules_fit: AR takes no steps or weighting')
        else:
            if isinstance(steps, bool) or not isinstance(steps, (int, np.integer)) or not 1 <= steps <= RULES_STEPS_MAX:
                raise ValueError('rules_fit: steps must be an integer in 1 .. %d, not %r' % (RULES_STEPS_MAX, steps))
            if weighting not in RULES_WEIGHTING:
                raise ValueError('rules_fit: weighting must be one of %s, not %r' % (sorted(RULES_WEIGHTING), weighting))
        off = np.ascontiguousarray(session_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        if off.ndim != 1 or off.size < 1 or it.ndim != 1:
            raise ValueError('rules_fit: need session offsets and a 1-D item array')
        if it.size and (it.min() < 0 or it.max() >= self.n_items):
            raise IndexError('rules_fit: item index out of range')
        if off[0] != 0 or off[-1] != it.size or (np.diff(off) < 0).any():
            raise ValueError('rules_fit: session offsets must rise from 0 to the number of events')
        if off.size - 1 > 2 ** 31 - 1 or it.size > 2 ** 31 - 1:
            raise ValueError('rules_fit: more than 2^31 - 1 sessions or events')
        if rules_bound(off, it, self.n_items, steps, weighting) >= 1 << 63:
            raise ValueError('rules_fit: a row\'s weight bound reaches 2^63 (uint64 counts could overflow)')
        pw, sb, ms = C.c_int64(), C.c_size_t(), C.c_float()
        self._check(self.lib.g4r_bl_rules_fit(self.h, _ptr(off), off.size - 1, _ptr(it), it.size, 0 if steps is None else int(steps),
                                              0 if weighting is None else RULES_WEIGHTING[weighting], C.byref(pw), C.byref(sb), C.byref(ms)))
        return pw.value, sb.value, ms.value

    def stan_set_w1(self, w1):
        """the STAN (or VSTAN) prefix-distance table W1[0 .. n): it must cover every counted event's prefix length"""
        w1 = np.ascontiguousarray(w1, dtype=np.float64)
        if w1.ndim != 1 or w1.size < 1:
            raise ValueError('stan_set_w1: w1 must be a non-empty 1-D table')
        self._check(self.lib.g4r_bl_stan_set_w1(self.h, _ptr(w1), w1.size))
        self.n_w1 = w1.size

    def vstan_set(self, similarity, f, w4):
        """the VSTAN settings after a stan_fit: the similarity ('cosine' or 'vector'), F per item (finite, >= 0) and the
        neighbour table W4[0 .. n) by prefix distance, entries in [0, 1]; W4 must cover every counted event's prefix length"""
        f = np.ascontiguousarray(f, dtype=np.float64); w4 = np.ascontiguousarray(w4, dtype=np.float64)
        if similarity not in SKNN_SIMILARITY:
            raise ValueError('vstan_set: similarity must be one of %s' % sorted(SKNN_SIMILARITY))
        if f.shape != (self.n_items,) or not (np.isfinite(f) & (f >= 0.0)).all():
            raise ValueError('vstan_set: f must hold one finite factor >= 0 per item')
        if w4.ndim != 1 or not 1 <= w4.size <= 1 << 30 or not ((w4 >= 0.0) & (w4 <= 1.0)).all():
            raise ValueError('vstan_set: w4 must be a non-empty 1-D table with entries in [0, 1]')
        self._check(self.lib.g4r_bl_vstan_set(self.h, SKNN_SIMILARITY[similarity], _ptr(f), f.size, _ptr(w4), w4.size))
        self.n_w4 = w4.size

    # ---- NARM (DESIGN §3s) ----
    def narm_n_params(self, hidden):
        d, H = self.n_keep, int(hidden)
        return self.n_items * d + 5 * d * H + 5 * H * H + 4 * H

    def _narm_params(self, hidden, params):
        th = np.ascontiguousarray(params, dtype=np.float32).ravel()
        if th.size != self.narm_n_params(hidden):
            raise ValueError('narm: need %d parameters (n_items d + 5 d H + 5 H^2 + 4 H), not %d' % (self.narm_n_params(hidden), th.size))
        return th

    def narm_begin(self, hidden, max_len, batch_size, piece_offsets, items, params):
        """starts a NARM fit: the training pieces (CSR of item indices, 2 .. max_len events each) and the initial flat parameters"""
        off = np.ascontiguousarray(piece_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        th = self._narm_params(hidden, params)
        self._check(self.lib.g4r_bl_narm_begin(self.h, int(hidden), int(max_len), int(batch_size), _ptr(off), off.size - 1, _ptr(it), it.size,
                                               _ptr(th), th.size))
        self.narm_hidden, self.narm_batch = int(hidden), int(batch_size)

    def narm_epoch(self, order, seed, learning_rate, dropout_emb, dropout_ct):
        """one epoch over the pieces in `order`; returns (per-step losses float32, device ms)"""
        od = np.ascontiguousarray(order, dtype=np.int32)
        losses = np.zeros(-(-od.size // self.narm_batch), np.float32); ms = C.c_float()
        self._check(self.lib.g4r_bl_narm_epoch(self.h, _ptr(od), od.size, int(seed) & 0xffffffff, float(learning_rate), float(dropout_emb),
                                               float(dropout_ct), _ptr(losses), C.byref(ms)))
        return losses, ms.value

    def narm_grads(self, pieces, seed, step, dropout_emb, dropout_ct):
        """(loss, flat gradient float32) of one mini-batch of pieces at the current parameters, without an update"""
        pc = np.ascontiguousarray(pieces, dtype=np.int32)
        g = np.empty(self.narm_n_params(self.narm_hidden), np.float32); loss = C.c_float()
        self._check(self.lib.g4r_bl_narm_grads(self.h, _ptr(pc), pc.size, int(seed) & 0xffffffff, int(step), float(dropout_emb), float(dropout_ct),
                                               C.byref(loss), _ptr(g)))
        return loss.value, g

    def narm_export(self):
        th = np.empty(self.narm_n_params(self.narm_hidden), np.float32)
        self._check(self.lib.g4r_bl_narm_export(self.h, _ptr(th), th.size))
        return th

    def narm_import(self, hidden, max_len, params):
        th = self._narm_params(hidden, params)
        self._check(self.lib.g4r_bl_narm_import(self.h, int(hidden), int(max_len), _ptr(th), th.size))
        self.narm_hidden = int(hidden)

    def narm_encode(self, items, session_offsets, n_history=None):
        """every counted event's q [n, d_e] float32, in evaluate's order"""
        it = np.ascontiguousarray(items, dtype=np.int32); off = np.ascontiguousarray(session_offsets, dtype=np.int64)
        nh = None if n_history is None else np.ascontiguousarray(n_history, dtype=np.int32)
        lens = np.diff(off)
        n = int(np.maximum(0, lens - np.maximum(nh if nh is not None else 0, 1)).sum()) if lens.size else 0
        q = np.empty((n, self.n_keep), np.float32)
        self._check(self.lib.g4r_bl_narm_encode(self.h, _ptr(it), it.size, _ptr(off), off.size - 1, _ptr(nh), _ptr(q), n))
        return q

    # ---- SASRec (DESIGN §3t) ----
    def sasrec_n_params(self, n_blocks, max_len):
        d = self.n_keep
        return self.n_items * d + int(max_len) * d + int(n_blocks) * (6 * d * d + 10 * d) + 2 * d

    def _sasrec_params(self, n_blocks, max_len, params):
        th = np.ascontiguousarray(params, dtype=np.float32).ravel()
        n = self.sasrec_n_params(n_blocks, max_len)
        if th.size != n:
            raise ValueError('sasrec: need %d parameters (n_items d + max_len d + n_blocks (6 d^2 + 10 d) + 2 d), not %d' % (n, th.size))
        return th

    def sasrec_begin(self, n_blocks, n_heads, max_len, batch_size, piece_offsets, items, params):
        """starts a SASRec fit: the training pieces (CSR of item indices, 2 .. max_len + 1 events each) and the initial flat
        parameters"""
        off = np.ascontiguousarray(piece_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        th = self._sasrec_params(n_blocks, max_len, params)
        self._check(self.lib.g4r_bl_sasrec_begin(self.h, int(n_blocks), int(n_heads), int(max_len), int(batch_size), _ptr(off), off.size - 1,
                                                 _ptr(it), it.size, _ptr(th), th.size))
        self.sasrec_shape, self.sasrec_batch = (int(n_blocks), int(max_len)), int(batch_size)

    def sasrec_epoch(self, order, seed, learning_rate, dropout):
        """one epoch over the pieces in `order`; returns (per-step losses float32, device ms)"""
        od = np.ascontiguousarray(order, dtype=np.int32)
        losses = np.zeros(-(-od.size // self.sasrec_batch), np.float32); ms = C.c_float()
        self._check(self.lib.g4r_bl_sasrec_epoch(self.h, _ptr(od), od.size, int(seed) & 0xffffffff, float(learning_rate), float(dropout),
                                                 _ptr(losses), C.byref(ms)))
        return losses, ms.value

    def sasrec_grads(self, pieces, seed, step, dropout):
        """(loss, flat gradient float32) of one mini-batch of pieces at the current parameters, without an update"""
        pc = np.ascontiguousarray(pieces, dtype=np.int32)
        g = np.empty(self.sasrec_n_params(*self.sasrec_shape), np.float32); loss = C.c_float()
        self._check(self.lib.g4r_bl_sasrec_grads(self.h, _ptr(pc), pc.size, int(seed) & 0xffffffff, int(step), float(dropout), C.byref(loss),
                                                 _ptr(g)))
        return loss.value, g

    def sasrec_export(self):
        th = np.empty(self.sasrec_n_params(*self.sasrec_shape), np.float32)
        self._check(self.lib.g4r_bl_sasrec_export(self.h, _ptr(th), th.size))
        return th

    def sasrec_import(self, n_blocks, n_heads, max_len, params):
        th = self._sasrec_params(n_blocks, max_len, params)
        self._check(self.lib.g4r_bl_sasrec_import(self.h, int(n_blocks), int(n_heads), int(max_len), _ptr(th), th.size))
        self.sasrec_shape = (int(n_blocks), int(max_len))

    def sasrec_encode(self, items, session_offsets, n_history=None):
        """every counted event's q [n, d] float32, in evaluate's order"""
        it = np.ascontiguousarray(items, dtype=np.int32); off = np.ascontiguousarray(session_offsets, dtype=np.int64)
        nh = None if n_history is None else np.ascontiguousarray(n_history, dtype=np.int32)
        lens = np.diff(off)
        n = int(np.maximum(0, lens - np.maximum(nh if nh is not None else 0, 1)).sum()) if lens.size else 0
        q = np.empty((n, self.n_keep), np.float32)
        self._check(self.lib.g4r_bl_sasrec_encode(self.h, _ptr(it), it.size, _ptr(off), off.size - 1, _ptr(nh), _ptr(q), n))
        return q

    # ---- SR-GNN (DESIGN §3u) ----
    def srgnn_n_params(self):
        d = self.n_keep
        return self.n_items * d + 15 * d * d + 14 * d

    def _srgnn_params(self, params):
        th = np.ascontiguousarray(params, dtype=np.float32).ravel()
        n = self.srgnn_n_params()
        if th.size != n:
            raise ValueError('srgnn: need %d parameters (n_items d + 15 d^2 + 14 d), not %d' % (n, th.size))
        return th

    def srgnn_begin(self, step, max_len, batch_size, session_offsets, items, params):
        """starts an SR-GNN fit: the training sessions (CSR of item indices, events in time order) and the initial flat parameters.
        The samples are every (prefix, next item) pair in session order"""
        off = np.ascontiguousarray(session_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        th = self._srgnn_params(params)
        self._check(self.lib.g4r_bl_srgnn_begin(self.h, int(step), int(max_len), int(batch_size), _ptr(off), off.size - 1, _ptr(it), it.size,
                                                _ptr(th), th.size))
        self.srgnn_batch = int(batch_size)

    def srgnn_epoch(self, order, learning_rate, l2):
        """one epoch over the samples in `order`; returns (per-step losses float32, device ms)"""
        od = np.ascontiguousarray(order, dtype=np.int32)
        losses = np.zeros(-(-od.size // self.srgnn_batch), np.float32); ms = C.c_float()
        self._check(self.lib.g4r_bl_srgnn_epoch(self.h, _ptr(od), od.size, float(learning_rate), float(l2), _ptr(losses), C.byref(ms)))
        return losses, ms.value

    def srgnn_grads(self, samples):
        """(loss, flat gradient of the loss float32) of one mini-batch of samples at the current parameters, without an update"""
        sm = np.ascontiguousarray(samples, dtype=np.int32)
        g = np.empty(self.srgnn_n_params(), np.float32); loss = C.c_float()
        self._check(self.lib.g4r_bl_srgnn_grads(self.h, _ptr(sm), sm.size, C.byref(loss), _ptr(g)))
        return loss.value, g

    def srgnn_export(self):
        th = np.empty(self.srgnn_n_params(), np.float32)
        self._check(self.lib.g4r_bl_srgnn_export(self.h, _ptr(th), th.size))
        return th

    def srgnn_import(self, step, max_len, params):
        th = self._srgnn_params(params)
        self._check(self.lib.g4r_bl_srgnn_import(self.h, int(step), int(max_len), _ptr(th), th.size))

    def srgnn_encode(self, items, session_offsets, n_history=None):
        """every counted event's s_h [n, d] float32, in evaluate's order"""
        it = np.ascontiguousarray(items, dtype=np.int32); off = np.ascontiguousarray(session_offsets, dtype=np.int64)
        nh = None if n_history is None else np.ascontiguousarray(n_history, dtype=np.int32)
        lens = np.diff(off)
        n = int(np.maximum(0, lens - np.maximum(nh if nh is not None else 0, 1)).sum()) if lens.size else 0
        q = np.empty((n, self.n_keep), np.float32)
        self._check(self.lib.g4r_bl_srgnn_encode(self.h, _ptr(it), it.size, _ptr(off), off.size - 1, _ptr(nh), _ptr(q), n))
        return q

    # ---- STAMP (DESIGN §3v) ----
    def stamp_n_params(self):
        d = self.n_keep
        return self.n_items * d + 5 * d * d + 4 * d

    def _stamp_params(self, params):
        th = np.ascontiguousarray(params, dtype=np.float32).ravel()
        n = self.stamp_n_params()
        if th.size != n:
            raise ValueError('stamp: need %d parameters (n_items d + 5 d^2 + 4 d), not %d' % (n, th.size))
        return th

    def stamp_begin(self, max_len, batch_size, session_offsets, items, params):
        """starts a STAMP fit: the training sessions (CSR of item indices, events in time order) and the initial flat parameters.
        The samples are every (prefix, next item) pair in session order"""
        off = np.ascontiguousarray(session_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        th = self._stamp_params(params)
        self._check(self.lib.g4r_bl_stamp_begin(self.h, int(max_len), int(batch_size), _ptr(off), off.size - 1, _ptr(it), it.size, _ptr(th), th.size))
        self.stamp_batch = int(batch_size)

    def stamp_epoch(self, order, learning_rate):
        """one epoch over the samples in `order`; returns (per-step losses float32, device ms)"""
        od = np.ascontiguousarray(order, dtype=np.int32)
        losses = np.zeros(-(-od.size // self.stamp_batch), np.float32); ms = C.c_float()
        self._check(self.lib.g4r_bl_stamp_epoch(self.h, _ptr(od), od.size, float(learning_rate), _ptr(losses), C.byref(ms)))
        return losses, ms.value

    def stamp_grads(self, samples):
        """(loss, flat gradient of the loss float32) of one mini-batch of samples at the current parameters, without an update"""
        sm = np.ascontiguousarray(samples, dtype=np.int32)
        g = np.empty(self.stamp_n_params(), np.float32); loss = C.c_float()
        self._check(self.lib.g4r_bl_stamp_grads(self.h, _ptr(sm), sm.size, C.byref(loss), _ptr(g)))
        return loss.value, g

    def stamp_export(self):
        th = np.empty(self.stamp_n_params(), np.float32)
        self._check(self.lib.g4r_bl_stamp_export(self.h, _ptr(th), th.size))
        return th

    def stamp_import(self, max_len, params):
        th = self._stamp_params(params)
        self._check(self.lib.g4r_bl_stamp_import(self.h, int(max_len), _ptr(th), th.size))

    def stamp_encode(self, items, session_offsets, n_history=None):
        """every counted event's q [n, d] float32, in evaluate's order"""
        it = np.ascontiguousarray(items, dtype=np.int32); off = np.ascontiguousarray(session_offsets, dtype=np.int64)
        nh = None if n_history is None else np.ascontiguousarray(n_history, dtype=np.int32)
        lens = np.diff(off)
        n = int(np.maximum(0, lens - np.maximum(nh if nh is not None else 0, 1)).sum()) if lens.size else 0
        q = np.empty((n, self.n_keep), np.float32)
        self._check(self.lib.g4r_bl_stamp_encode(self.h, _ptr(it), it.size, _ptr(off), off.size - 1, _ptr(nh), _ptr(q), n))
        return q

    # ---- NextItNet (DESIGN §3w) ----
    def nextitnet_n_params(self, n_dilations, kernel_size):
        d = self.n_keep
        return 2 * self.n_items * d + self.n_items + int(n_dilations) * (2 * int(kernel_size) * d * d + 6 * d)

    def _nextitnet_params(self, dilations, kernel_size, params):
        th = np.ascontiguousarray(params, dtype=np.float32).ravel()
        n = self.nextitnet_n_params(len(dilations), kernel_size)
        if th.size != n:
            raise ValueError('nextitnet: need %d parameters (2 n_items d + n_items + n_dilations (2 kernel_size d^2 + 6 d)), not %d' % (n, th.size))
        return th

    def nextitnet_begin(self, dilations, kernel_size, max_len, batch_size, piece_offsets, items, params):
        """starts a NextItNet fit: the training pieces (CSR of item indices, 2 .. max_len + 1 events each) and the initial flat
        parameters"""
        dl = np.ascontiguousarray(dilations, dtype=np.int32)
        off = np.ascontiguousarray(piece_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        th = self._nextitnet_params(dl, kernel_size, params)
        self._check(self.lib.g4r_bl_nextitnet_begin(self.h, _ptr(dl), dl.size, int(kernel_size), int(max_len), int(batch_size), _ptr(off),
                                                    off.size - 1, _ptr(it), it.size, _ptr(th), th.size))
        self.nextitnet_shape, self.nextitnet_batch = (dl.size, int(kernel_size)), int(batch_size)

    def nextitnet_epoch(self, order, learning_rate):
        """one epoch over the pieces in `order`; returns (per-step losses float32, device ms)"""
        od = np.ascontiguousarray(order, dtype=np.int32)
        losses = np.zeros(-(-od.size // self.nextitnet_batch), np.float32); ms = C.c_float()
        self._check(self.lib.g4r_bl_nextitnet_epoch(self.h, _ptr(od), od.size, float(learning_rate), _ptr(losses), C.byref(ms)))
        return losses, ms.value

    def nextitnet_grads(self, pieces):
        """(loss, flat gradient float32) of one mini-batch of pieces at the current parameters, without an update"""
        pc = np.ascontiguousarray(pieces, dtype=np.int32)
        g = np.empty(self.nextitnet_n_params(*self.nextitnet_shape), np.float32); loss = C.c_float()
        self._check(self.lib.g4r_bl_nextitnet_grads(self.h, _ptr(pc), pc.size, C.byref(loss), _ptr(g)))
        return loss.value, g

    def nextitnet_export(self):
        th = np.empty(self.nextitnet_n_params(*self.nextitnet_shape), np.float32)
        self._check(self.lib.g4r_bl_nextitnet_export(self.h, _ptr(th), th.size))
        return th

    def nextitnet_import(self, dilations, kernel_size, max_len, params):
        dl = np.ascontiguousarray(dilations, dtype=np.int32)
        th = self._nextitnet_params(dl, kernel_size, params)
        self._check(self.lib.g4r_bl_nextitnet_import(self.h, _ptr(dl), dl.size, int(kernel_size), int(max_len), _ptr(th), th.size))
        self.nextitnet_shape = (dl.size, int(kernel_size))

    def nextitnet_encode(self, items, session_offsets, n_history=None):
        """every counted event's q [n, d] float32, in evaluate's order"""
        it = np.ascontiguousarray(items, dtype=np.int32); off = np.ascontiguousarray(session_offsets, dtype=np.int64)
        nh = None if n_history is None else np.ascontiguousarray(n_history, dtype=np.int32)
        lens = np.diff(off)
        n = int(np.maximum(0, lens - np.maximum(nh if nh is not None else 0, 1)).sum()) if lens.size else 0
        q = np.empty((n, self.n_keep), np.float32)
        self._check(self.lib.g4r_bl_nextitnet_encode(self.h, _ptr(it), it.size, _ptr(off), off.size - 1, _ptr(nh), _ptr(q), n))
        return q

    # ---- BERT4Rec (DESIGN §3x) ----
    def bert4rec_n_params(self, n_blocks, max_len):
        d = self.n_keep
        return (self.n_items + 1) * d + int(max_len) * d + 2 * d + int(n_blocks) * (12 * d * d + 13 * d) + d * d + 3 * d + self.n_items

    def _bert4rec_params(self, n_blocks, max_len, params):
        th = np.ascontiguousarray(params, dtype=np.float32).ravel()
        n = self.bert4rec_n_params(n_blocks, max_len)
        if th.size != n:
            raise ValueError('bert4rec: need %d parameters ((n_items + 1) d + max_len d + 2 d + n_blocks (12 d^2 + 13 d) + d^2 + 3 d + n_items), '
                             'not %d' % (n, th.size))
        return th

    def bert4rec_begin(self, n_blocks, n_heads, max_len, batch_size, piece_offsets, items, params):
        """starts a BERT4Rec fit: the training pieces (CSR of item indices, 2 .. max_len events each, all inputs) and the initial
        flat parameters"""
        off = np.ascontiguousarray(piece_offsets, dtype=np.int64); it = np.ascontiguousarray(items, dtype=np.int32)
        th = self._bert4rec_params(n_blocks, max_len, params)
        self._check(self.lib.g4r_bl_bert4rec_begin(self.h, int(n_blocks), int(n_heads), int(max_len), int(batch_size), _ptr(off), off.size - 1,
                                                   _ptr(it), it.size, _ptr(th), th.size))
        self.bert4rec_shape, self.bert4rec_batch = (int(n_blocks), int(max_len)), int(batch_size)

    def bert4rec_epoch(self, order, masks, seed, learning_rate, dropout):
        """one epoch over the pieces in `order`, masks one byte (0 / 1) per stored entry; returns (per-step losses float32, device
        ms)"""
        od = np.ascontiguousarray(order, dtype=np.int32); mk = np.ascontiguousarray(masks, dtype=np.uint8)
        losses = np.zeros(-(-od.size // self.bert4rec_batch), np.float32); ms = C.c_float()
        self._check(self.lib.g4r_bl_bert4rec_epoch(self.h, _ptr(od), od.size, _ptr(mk), mk.size, int(seed) & 0xffffffff, float(learning_rate),
                                                   float(dropout), _ptr(losses), C.byref(ms)))
        return losses, ms.value

    def bert4rec_grads(self, pieces, masks, seed, step, dropout):
        """(loss, flat gradient float32) of one mini-batch of pieces at the current parameters, without an update"""
        pc = np.ascontiguousarray(pieces, dtype=np.int32); mk = np.ascontiguousarray(masks, dtype=np.uint8)
        g = np.empty(self.bert4rec_n_params(*self.bert4rec_shape), np.float32); loss = C.c_float()
        self._check(self.lib.g4r_bl_bert4rec_grads(self.h, _ptr(pc), pc.size, _ptr(mk), mk.size, int(seed) & 0xffffffff, int(step),
                                                   float(dropout), C.byref(loss), _ptr(g)))
        return loss.value, g

    def bert4rec_export(self):
        th = np.empty(self.bert4rec_n_params(*self.bert4rec_shape), np.float32)
        self._check(self.lib.g4r_bl_bert4rec_export(self.h, _ptr(th), th.size))
        return th

    def bert4rec_import(self, n_blocks, n_heads, max_len, params):
        th = self._bert4rec_params(n_blocks, max_len, params)
        self._check(self.lib.g4r_bl_bert4rec_import(self.h, int(n_blocks), int(n_heads), int(max_len), _ptr(th), th.size))
        self.bert4rec_shape = (int(n_blocks), int(max_len))

    def bert4rec_encode(self, items, session_offsets, n_history=None):
        """every counted event's q [n, d] float32, in evaluate's order"""
        it = np.ascontiguousarray(items, dtype=np.int32); off = np.ascontiguousarray(session_offsets, dtype=np.int64)
        nh = None if n_history is None else np.ascontiguousarray(n_history, dtype=np.int32)
        lens = np.diff(off)
        n = int(np.maximum(0, lens - np.maximum(nh if nh is not None else 0, 1)).sum()) if lens.size else 0
        q = np.empty((n, self.n_keep), np.float32)
        self._check(self.lib.g4r_bl_bert4rec_encode(self.h, _ptr(it), it.size, _ptr(off), off.size - 1, _ptr(nh), _ptr(q), n))
        return q
