/*
 * g4r.h -- C ABI of libg4r.so: the H100 (sm_90a) GRU4Rec session-parallel training step.
 *
 * This is the drop-in boundary for the hot path of hidasib/GRU4Rec.  In the reference the boundary is
 * the set of compiled Theano functions that gru4rec.py / evaluation.py call once per mini-batch; each
 * entry point below names the reference interface (file:line under /root/reference) it replaces.
 * Plain pointers and sizes only; no torch / Python types.  All functions return 0 on success or a
 * negative g4r_status; g4r_last_error() gives the message.  A handle is not thread-safe; one handle per
 * process per device (reference: single Python thread, single CUDA context, .theanorc_gru4rec:3).
 *
 * Unless a parameter is documented as a device pointer, buffers are HOST memory; the library does the
 * host<->device copies on its own stream (these copies are what bench.py's "e2e" number includes).
 */
#ifndef G4R_H
#define G4R_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define G4R_MAX_LAYERS 8

typedef enum {
  G4R_OK = 0,
  G4R_ERR_INVALID = -1,        /* bad argument / unsupported configuration (reference: NotImplementedError) */
  G4R_ERR_INDEX = -2,          /* index out of bounds (reference: IndexError, custom_theano_ops.py:586-591) */
  G4R_ERR_CUDA = -3,           /* CUDA runtime failure (reference: RuntimeError "gpuarray error") */
  G4R_ERR_NAN = -4,            /* NaN cost detected (reference: gru4rec.py:626-629) */
  G4R_ERR_STATE = -5
} g4r_status;

typedef enum { G4R_LOSS_XE = 0, G4R_LOSS_BPR_MAX = 1, G4R_LOSS_TOP1_MAX = 2, G4R_LOSS_BPR = 3, G4R_LOSS_TOP1 = 4,
               G4R_LOSS_XE_LOGIT = 5 } g4r_loss;                       /* gru4rec.py:136-143 */
typedef enum { G4R_ACT_LINEAR = 0, G4R_ACT_RELU = 1, G4R_ACT_TANH = 2, G4R_ACT_LEAKY = 3, G4R_ACT_ELU = 4,
               G4R_ACT_SELU = 5, G4R_ACT_SOFTMAX = 6, G4R_ACT_SOFTMAX_LOGIT = 7 } g4r_act;   /* gru4rec.py:144-161 */
typedef enum { G4R_ADAPT_NONE = 0, G4R_ADAPT_ADAGRAD = 1, G4R_ADAPT_RMSPROP = 2, G4R_ADAPT_ADADELTA = 3, G4R_ADAPT_ADAM = 4 } g4r_adapt;  /* gru4rec.py:300-381,392-399 */

/* Mirrors the GRU4Rec constructor arguments that shape the compiled step (gru4rec.py:97-135). */
typedef struct g4r_config {
  int32_t n_items;
  int32_t n_layers;
  int32_t layers[G4R_MAX_LAYERS];
  int32_t batch_size;
  int32_t embedding;              /* 0: none; >0: separate item embedding E of this width (gru4rec.py:449-456) */
  int32_t constrained_embedding;  /* 1: Wy doubles as the input embedding (gru4rec.py:438-448) */
  int32_t loss;                   /* g4r_loss */
  int32_t final_act;              /* g4r_act */
  float final_act_p1, final_act_p2;
  int32_t hidden_act;             /* g4r_act (elementwise ones) */
  float hidden_act_p1, hidden_act_p2;
  float dropout_p_hidden, dropout_p_embed;
  float learning_rate, momentum, lmbd;
  int32_t n_sample;
  float sample_alpha;
  float smoothing, bpreg, logq;
  int32_t adapt;                  /* g4r_adapt */
  int32_t sample_store;           /* capacity of the negative-sample store in ids (gru4rec.py:515,547); 0 = none */
  uint32_t dropout_seed;
  uint32_t mrg_seed;              /* MRG_RandomStreams seed (Theano default 12345) */
  int32_t max_resident_steps;     /* capacity (in mini-batches) of the device-resident schedule window; 0 = default */
  int32_t device;                 /* CUDA device ordinal */
  int32_t world_size, rank;       /* data-parallel geometry (1,0 for single GPU) */
  int32_t eval_batch_size;        /* lanes reserved for the scoring path (evaluation.py batch_size); 0 = batch_size */
  int32_t step_mode;              /* 0: one kernel per phase (CUDA-graph replay); 1: persistent cooperative kernel;
                                     2: role-specialised persistent kernel where the shape allows, else 1;
                                     3: as 2, launched as thread-block clusters: the GRU phases run on one cluster with the
                                        dense weights and optimizer state resident in shared memory (else 1);
                                     4: tensor-core step (wgmma GEMMs) whenever the model allows it -- modes 1-3 pick it
                                        automatically for constrained-embedding models with a layer of >= 160 units */
  int32_t mg_replicated;          /* 1: multi-GPU with replicated tables + NCCL exchange instead of row sharding */
  int32_t eval_tc;                /* scoring path: 0 auto, 1 fp32 FFMA tiles only, 2 wgmma (3xTF32) tiles whenever the ranking is full-catalogue;
                                     also the score tiles of full_softmax training (auto: wgmma from 64 lanes and 2048 items) */
  float adapt_p1, adapt_p1c;      /* adapt_params[0] and 1 - adapt_params[0] (rmsprop / adadelta decay; adam beta1), gru4rec.py:301-304,342-343,368-369 */
  float adapt_p2, adapt_p2c;      /* adapt_params[1] and 1 - adapt_params[1] (adam beta2) */
  float grad_cap;                 /* > 0: gradients are scaled to this global L2 norm when they exceed it (gru4rec.py:386-389) */
  int32_t bptt;                   /* 0 / 1: one update per mini-batch.  2..64: truncated backpropagation through time, one update per
                                     window of bptt consecutive mini-batches of the schedule (DESIGN §3l).  Single GPU; step_mode
                                     has no effect.  g4r_train_steps / g4r_upload_steps then take ranges that start at a multiple
                                     of bptt and hold whole windows unless they run to the schedule's end (else G4R_ERR_INVALID);
                                     g4r_train_step and g4r_profile_uploaded return G4R_ERR_STATE */
  int32_t full_softmax;           /* 0: sampled output layer (Y | samples).  1: every training step scores the whole catalogue 0..n_items-1,
                                     each item once, and updates every Wy / By row (DESIGN §3n).  loss XE / softmax or xe_logit /
                                     softmax_logit only; logq, n_sample, sample_alpha and sample_store are ignored (no sample store
                                     is allocated).  Refused (G4R_ERR_INVALID): smoothing > 0, grad_cap > 0, bptt > 1, world_size > 1.
                                     step_mode has no effect */
} g4r_config;

typedef struct g4r_handle g4r_handle;
typedef struct g4r_schedule g4r_schedule;

/* ---- lifecycle ------------------------------------------------------------------------------------ */
int g4r_version(void);
/* Bytes of device memory the handle needs; the caller may allocate them (e.g. a torch uint8 tensor used
 * purely as an allocator) and pass the DEVICE pointer to g4r_create, or pass NULL to let the library
 * cudaMalloc.  Replaces: theano.shared(...) allocations in GRU4Rec.init (gru4rec.py:267-294,331,401,425,556-558). */
int g4r_workspace_bytes(const g4r_config* cfg, size_t* bytes);
int g4r_create(const g4r_config* cfg, void* device_workspace, size_t workspace_bytes, g4r_handle** out);
int g4r_destroy(g4r_handle* h);
const char* g4r_last_error(const g4r_handle* h);   /* h may be NULL: last creation error */
/* cudaStream_t the step kernels are launched on (for CUDA-event timing by the caller). */
void* g4r_stream(g4r_handle* h);

/* ---- parameters: shared-variable get_value/set_value (gru4rec.py:745-767, 590, 649-651) ----------- */
/* names: "Wx0".."Wx7","Wh*","Wrz*","Bh*","H*","Wy","By","E", and optimizer state "<name>.acc" (adagrad / rmsprop / adadelta /
 * adam), "<name>.upd" (adadelta), "<name>.meang" and "<name>.countt" (adam), "<name>.vel" (momentum > 0). */
int g4r_tensor_shape(g4r_handle* h, const char* name, int64_t* rows, int64_t* cols);
int g4r_set_tensor(g4r_handle* h, const char* name, const float* host, int64_t rows, int64_t cols);
int g4r_get_tensor(g4r_handle* h, const char* name, float* host, int64_t rows, int64_t cols);
int g4r_reset_hidden(g4r_handle* h);               /* gru4rec.py:589-590 */

/* ---- negative sampling (gru4rec.py:539-566) ------------------------------------------------------- */
int g4r_set_sampling_cdf(g4r_handle* h, const float* P, int64_t n);     /* P (gru4rec.py:556) */
int g4r_set_logq_support(g4r_handle* h, const float* P0, int64_t n);    /* P0 (gru4rec.py:541) */
/* generate_samples(): MRG31k3p uniforms + binary search into P; resets the sample pointer (gru4rec.py:559-564). */
int g4r_generate_samples(g4r_handle* h);
/* Same search on caller-supplied uniforms (parity at the K2 boundary; custom_theano_ops.py:318-349). */
int g4r_generate_samples_from_uniform(g4r_handle* h, const float* u, int64_t n);
int g4r_set_sample_store(g4r_handle* h, const int64_t* st, int64_t rows);   /* rows x n_sample */
int g4r_get_sample_store(g4r_handle* h, int64_t* st, int64_t rows);
int g4r_sample_store_rows(g4r_handle* h);                                    /* generate_length (gru4rec.py:547) */
int g4r_set_sample_pointer(g4r_handle* h, int64_t p);                        /* STI (gru4rec.py:558,583) */
int64_t g4r_get_sample_pointer(g4r_handle* h);
/* Raw MRG uniforms (theano.sandbox.rng_mrg restatement) for tests. */
int g4r_mrg_uniform(g4r_handle* h, float* out, int64_t n);

/* ---- stand-alone custom ops (custom_theano_ops.py) ------------------------------------------------ */
/* GpuBinarySearchSorted (custom_theano_ops.py:275-407): y[i] = index of x[i] in sorted d. */
int g4r_searchsorted(g4r_handle* h, const float* d, int64_t n_d, const float* x, int64_t n_x, int64_t* y);
/* GpuAdvancedSubtensor1_fast (custom_theano_ops.py:409-595): out[i,:] = table[idx[i],:], negative wrap,
 * out-of-range -> G4R_ERR_INDEX. */
int g4r_gather_rows(g4r_handle* h, const float* table, int64_t rows, int64_t cols, const int64_t* idx, int64_t n_idx, float* out);

/* ---- session-parallel schedule (gru4rec.py:585-651; evaluation.py:90-139) -------------------------- */
/* Builds every mini-batch of one epoch on the host: X/Y item indices, reset flags, batch sizes, lane slots.
 * mode 0 = training order semantics (reset-after flags), 1 = evaluation (zero-before flags), 1 | G4R_SCHED_POSITIONS = evaluation
 * that also records every lane's input position (g4r_schedule_positions).
 * session_order: n_sessions session ids (gru4rec.py:585/593; a rank's shard in the multi-GPU path) or NULL for identity;
 * offset_sessions must cover every id that occurs in it. */
int g4r_schedule_build(const int64_t* data_items, int64_t n_events, const int32_t* offset_sessions, int64_t n_sessions,
                       const int64_t* session_order, int32_t batch_size, int32_t n_sample, int32_t mode, g4r_schedule** out);
int g4r_schedule_free(g4r_schedule* s);
int64_t g4r_schedule_steps(const g4r_schedule* s);
int64_t g4r_schedule_events(const g4r_schedule* s);       /* sum of batch sizes (history schedules: counted events) */
/* Copies out step arrays (each step padded to batch_size entries; unused lanes = -1 / 0). Any pointer may be NULL. */
int g4r_schedule_export(const g4r_schedule* s, int32_t* X, int32_t* Y, uint8_t* flags, int32_t* M, int32_t* slots);
/* Evaluation schedules built with mode 1 | G4R_SCHED_POSITIONS: pos[step * batch_size + b] = index in data_items of the input X
 * of lane b (its target is at pos + 1), -1 on unused lanes.  This maps the events of g4r_eval_events back to the test data.
 * G4R_ERR_STATE for a schedule built without the flag (other schedules do not spend the memory). */
#define G4R_SCHED_POSITIONS 2
int g4r_schedule_positions(const g4r_schedule* s, int64_t* pos);
/* Evaluation from each session's history (DESIGN §3h): the evaluation schedule (mode 1 or 1 | G4R_SCHED_POSITIONS) of the
 * sessions as g4r_schedule_build walks them, where session id j's first n_history[j] events are history (0 <= n_history[j] <=
 * its length).  A lane's event is counted only if its target is past the history: flag bit 2 (value 4) in g4r_schedule_export,
 * and g4r_schedule_events returns the number of counted events.  g4r_eval_schedule / g4r_eval_events on such a schedule run the
 * forward over every event but rank only the counted ones: their sums, counts and lists are those of the same call on the plain
 * schedule of the same data restricted to the counted events, which g4r_eval_events numbers in (step, lane) order -- mini-batch
 * by mini-batch, the counted lanes of each in lane order.  G4R_ERR_INVALID on a bad mode or n_history entry. */
int g4r_schedule_build_history(const int64_t* data_items, int64_t n_events, const int32_t* offset_sessions, int64_t n_sessions,
                               const int64_t* session_order, const int32_t* n_history, int32_t batch_size, int32_t mode, g4r_schedule** out);

/* ---- the compiled step: train_function(X, Y, M, R) -> cost (gru4rec.py:584,623) ------------------- */
/* One mini-batch from host arrays; returns the cost (D2H) like the reference call. */
int g4r_train_step(g4r_handle* h, const int32_t* X, const int32_t* Y, int32_t M, const int8_t* R, float* cost);
/* Steps [first, first+n) of a schedule: uploads the window, runs every step on the device without host
 * round trips, regenerates the sample store when the pointer wraps (gru4rec.py:618-621), copies the n
 * costs back.  NaN cost -> G4R_ERR_NAN with *nan_step set (gru4rec.py:626-629). */
int g4r_train_steps(g4r_handle* h, const g4r_schedule* s, int64_t first, int64_t n, float* cost_out, int64_t* nan_step);
/* Two-phase variant used for device-resident timing: upload (H2D + per-step column plans) then run. */
int g4r_upload_steps(g4r_handle* h, const g4r_schedule* s, int64_t first, int64_t n);
int g4r_run_uploaded(g4r_handle* h, float* cost_out /* may be NULL */, float* device_ms /* may be NULL */);
/* Re-runs the uploaded window with CUDA events around every kernel launch; sums device time and launch counts
 * per phase (index i is named by g4r_phase_name(i); n_phases must be >= g4r_phase_count()).  For bench.py's
 * roofline: achieved bytes/s of the dominant kernel = its algorithmic bytes / its mean duration. */
int g4r_profile_uploaded(g4r_handle* h, float* phase_ms, int32_t* phase_launches, int32_t n_phases);
const char* g4r_phase_name(int32_t i);
/* step_mode 2: number of windows run by the role-specialised kernel, and (out) windows that fell back to the
 * generic persistent kernel because a chunk of score columns was wider than 16. */
int64_t g4r_fast_windows(const g4r_handle* h, int64_t* fallback_windows);
/* bptt > 1: number of windows trained (each one backward through time and one update) */
int64_t g4r_bptt_windows(const g4r_handle* h);
/* full_softmax = 1: number of training steps run against the whole catalogue */
int64_t g4r_full_steps(const g4r_handle* h);
/* 1 if the handle trains with the tensor-core step (wgmma 3xTF32 GEMMs with fused epilogues, csrc/g4r_tcstep.cuh): constrained
 * embedding, one layer, batch <= 256, SGD / Adagrad (+momentum); automatic for layers >= 160 units, forced with step_mode 4. */
int g4r_uses_tensor_cores(const g4r_handle* h);
/* Persistent mode (step_mode 1): enable %globaltimer stamps at the phase boundaries of every step and/or read
 * the stamps of the last window (16 uint64 slots per step; slots 0..5 used: start, after GRU forward, after scores,
 * after statistics, after loss-gradient/update, end). */
int g4r_persistent_stamps(g4r_handle* h, int32_t enable, unsigned long long* out, int64_t n_steps);
int g4r_phase_count(void);
/* Counters for bench.py: kernels launched by this handle so far. */
int64_t g4r_kernel_launches(const g4r_handle* h);

/* ---- training state: checkpoint / resume and catalogue growth (DESIGN §3i; no reference counterpart) -----------------------
 * A training handle consists of its named tensors (parameters, optimizer state "<name>.acc" / ".upd" / ".meang" / ".countt" /
 * ".vel", the hidden state "H<l>": g4r_get_tensor / g4r_set_tensor), the sample store (g4r_get_sample_store /
 * g4r_set_sample_store) and the state these three functions move as one versioned blob: the global step that keys the dropout
 * masks, the sample pointer, and the MRG31k3p base and stream states.  A handle that receives all of them continues the run of
 * the handle they came from bit for bit.  The blob names the n_sample, sample-store rows, seeds and world / rank it is valid
 * for.  g4r_train_state_import checks magic, version, size and those fields before it changes anything: G4R_ERR_INVALID leaves
 * the handle as it was.  Call it after g4r_set_sample_store (which rewinds the sample pointer).  G4R_ERR_STATE on a multi-GPU
 * handle. */
int g4r_train_state_bytes(g4r_handle* h, size_t* bytes);
int g4r_train_state_export(g4r_handle* h, void* host, size_t bytes);
int g4r_train_state_import(g4r_handle* h, const void* host, size_t bytes);
/* Catalogue growth: a handle keeps its n_items, so a model takes in new items by moving to a new handle.  Copies, device to
 * device, every parameter, optimizer-state tensor and training hidden state of `src` into `dst`, whose n_items is >= src's.
 * Item tables (Wy, By, E, and Wx0 of a model without embedding) and each of their state tensors keep rows 0 .. n_old-1 as
 * they are; rows n_old .. n_new-1 of the weights come from new_Wy [n_new - n_old x L_last], new_By [n_new - n_old] and new_in
 * (the new rows of E, or of Wx0 without embedding: [n_new - n_old x embedding | 3 L_0]; ignored with constrained_embedding),
 * row-major host blocks, NULL = zero; the new rows of every state tensor are zero.  The handles must be single-GPU, on one
 * device, and agree in layers, batch size, embedding mode, optimizer and whether momentum is on (everything that shapes a
 * copied tensor), else G4R_ERR_INVALID before anything is written.  Nothing else moves: sampling tables, sample store and the
 * training-state blob are the caller's to set. */
int g4r_copy_item_tables(g4r_handle* dst, g4r_handle* src, const float* new_Wy, const float* new_By, const float* new_in);

/* ---- multi-GPU (one process per GPU; SURVEY section 8e) -------------------------------------------------------
 * Handles created with world_size > 1 compute gradients only; g4r_train_steps then exchanges them over NCCL
 * (all-gather of row gradients, all-reduce of dense gradients) and applies the merged update on every rank.
 * Rank 0 obtains a 128-byte NCCL unique id, the caller broadcasts it (e.g. torch.distributed), every rank calls
 * g4r_mg_init.  All ranks must call g4r_train_steps with the same number of steps. */
int g4r_mg_unique_id(char* out128);
int g4r_mg_init(g4r_handle* h, const char* id128);
/* Row-sharded layout (the default for world_size > 1 when the role-specialised kernel covers the shape: no-embedding mode, one
 * layer of <= 120 units, batch <= 32; cfg.mg_replicated = 1 forces the replicated NCCL path above).  Row i of Wy / By / Wx0 and
 * of their optimizer state lives only on rank i % world_size (local row i / world_size) in a library-owned segment that the
 * peers map with cudaIpc; parameter rows are fetched from their owners and gradient rows are stored into the owners' inboxes
 * over NVLink INSIDE the persistent kernel, the owners apply the merged update to their 1/world_size of the rows, and the
 * dense GRU gradients are pushed to all peers and summed in rank order.  NCCL only carries the per-window all-gather of the
 * sorted column lists.  Call order: g4r_create -> g4r_mg_init -> g4r_mg_ipc_handle (all-gather the 64-byte handles in rank
 * order) -> g4r_mg_ipc_open.  g4r_set_tensor / g4r_get_tensor keep the single-GPU shapes ("Wy" is n_items x L): set scatters
 * the caller's full matrix to this rank's rows, get assembles the full matrix from all shards (all ranks idle).
 * There is no reference counterpart (the reference is single-device, .theanorc_gru4rec:3); SURVEY section 8e is the spec. */
int g4r_mg_sharded(const g4r_handle* h);                               /* 1 if the handle uses the row-sharded layout */
int g4r_mg_ipc_handle(g4r_handle* h, char* out64);                    /* cudaIpcMemHandle_t of this rank's segment */
int g4r_mg_ipc_open(g4r_handle* h, const char* handles, int32_t world);   /* world x 64 bytes, rank order */
/* Ownership arithmetic and buffer sizing of the sharded layout (pure host functions, usable without a device). */
int g4r_mg_owner(int64_t item, int32_t world);
int64_t g4r_mg_local_row(int64_t item, int32_t world);
int64_t g4r_mg_shard_rows(int64_t n_items, int32_t world, int32_t rank);
int g4r_mg_segment_bytes(const g4r_config* cfg, size_t* total, size_t* inbox_bytes, size_t* inbox_in_bytes, size_t* dense_bytes);

/* ---- scoring path: evaluate(X, Y, M) (evaluation.py:76,108) and predict (gru4rec.py:706-710) ------- */
/* Runs a whole evaluation schedule: full-catalogue scores, rank of the target, per-cutoff hit counts and
 * reciprocal-rank sums.  mode: 0 standard, 1 conservative, 2 median, 3 tiebreaking (evaluation.py:55,60-65; the tie-breaking noise U(0,1) * 1e-10 is a
 * counter hash here, Theano's MRG stream in the reference).
 * recall_sum/mrr_sum: n_cut doubles each (sums, not yet divided by the number of events). */
int g4r_eval_schedule(g4r_handle* h, const g4r_schedule* s, const int32_t* cut_off, int32_t n_cut, int32_t mode,
                      double* recall_sum, double* mrr_sum, int64_t* n_events);
/* Diagnostic: the per-lane counts of the last mini-batch ranked by g4r_eval_schedule.  out[2 b] = number of items whose score
 * beats the target score of lane b, out[2 b + 1] = number of items whose score equals it (the target itself included).
 * n_lanes <= the scoring batch size; lanes past that mini-batch's size hold stale values. */
int g4r_eval_counts(g4r_handle* h, int32_t* out, int64_t n_lanes);
/* evaluate_gpu(items=...) (evaluation.py:15,52-56,84-100): rank the targets against the `n` candidate item indices instead of
 * the whole catalogue for subsequent g4r_eval_schedule calls (the target's own score competes only if the target is listed,
 * as in the reference); n = 0 restores the full-catalogue ranking.  G4R_ERR_INDEX on an out-of-range index. */
int g4r_set_eval_items(g4r_handle* h, const int64_t* items, int64_t n);
/* evaluate_gpu(exclude_seen=True) (DESIGN §3g): on != 0 makes subsequent g4r_eval_schedule / g4r_eval_events calls rank each
 * event without the items its session has input so far, the current input included (recommend_next_batch's exclude_seen rule);
 * with g4r_set_eval_items every occurrence of such an item in the candidate list goes.  An event whose target is among them is a
 * miss: rank +inf, nothing added to the sums, (-1, -1) in g4r_eval_events' out_counts; its lists hold only eligible items, the
 * slots past them item -1 and score NaN.  The seen lists take eval batch size x (longest session of the schedule - 1) int32 on
 * the device; a schedule for which that exceeds 256 MiB is refused with G4R_ERR_INVALID before any device work.  on = 0
 * restores the plain ranking. */
int g4r_set_eval_exclude_seen(g4r_handle* h, int32_t on);
/* g4r_eval_schedule with per-event outputs (DESIGN §3f).  Events are numbered in the order the schedule consumes them: mini-batch
 * by mini-batch, lanes 0 .. M-1 of each (g4r_schedule_positions maps them to the test data).  recall_sum / mrr_sum / n_events
 * are bit for bit those of g4r_eval_schedule with the same arguments.  out_counts [n_events x 2]: (#items scoring above the
 * target, #items tied with it, the target included), as g4r_eval_counts, under the same mode and candidate items.  k > 0: the
 * k best items of every event, as g4r_predict_topk_filtered ranks the lane after the event's input (ranking key, ties, scores;
 * with g4r_set_eval_items only the distinct candidates compete, softmax normaliser over them), into out_items / out_scores
 * [n_events x k]; k = 0: no lists (out_items / out_scores may be NULL).  The lists and the counts follow different tie rules.
 * Runs in windows of mini-batches with no host round trip inside a window; the window is shortened to bound its device buffers
 * (G4R_EVENTS_WINDOW in the environment, read when a handle first runs this, caps it further).  G4R_ERR_INVALID unless
 * 0 <= k <= min(distinct candidates, G4R_TOPK_MAX). */
int g4r_eval_events(g4r_handle* h, const g4r_schedule* s, const int32_t* cut_off, int32_t n_cut, int32_t mode, int32_t k,
                    double* recall_sum, double* mrr_sum, int64_t* n_events, int32_t* out_counts, int32_t* out_items, float* out_scores);
/* Rest-of-session evaluation (DESIGN §3m) on a schedule built with mode 1 | G4R_SCHED_POSITIONS (plain or history): every event
 * g4r_eval_schedule counts is ranked against each distinct item of the rest of its session (first occurrence first, the next
 * item first), each as if it were the event's target, with the same competitors, mode, g4r_set_eval_items and
 * g4r_set_eval_exclude_seen.  A relevant item the session has already input, or (with candidate items) one that is not listed,
 * is a miss.  sums_out [6 x n_cut]: per cut-off the sums over the events of HitRate, Precision, Recall, MRR, NDCG and MAP, in
 * double, accumulated in a fixed order.  out_counts [n_pairs x 2] (NULL: not written): (#greater, #equal) of every pair, (-1, -1)
 * for a miss, events in the order of g4r_eval_events, each event's items in first-occurrence order; out_offsets [n_events + 1]
 * (NULL: not written): every event's first pair.  The relevant lists take lanes x (longest session - 1) int32 under the 256 MiB
 * budget of the seen lists (G4R_SEEN_BUDGET lowers it): over it G4R_ERR_INVALID before any device work.  G4R_ERR_STATE for a
 * schedule built without positions.  The pairs take the tile kind of the next-item ranking (fp32, or wgmma under
 * cfg.eval_tc / wgmma_tiles). */
int g4r_eval_rest(g4r_handle* h, const g4r_schedule* s, const int32_t* cut_off, int32_t n_cut, int32_t mode, double* sums_out,
                  int64_t* n_events, int64_t* n_pairs, int32_t* out_counts, int64_t* out_offsets);
/* host only: the counted events and (event, relevant item) pairs g4r_eval_rest will report for schedule s (positions needed) */
int g4r_eval_rest_pairs(const g4r_schedule* s, int64_t* n_events, int64_t* n_pairs);

/* predict_next_batch's device call: scores of all items for `batch` lanes; reset_mask zeroes lanes first
 * (gru4rec.py:712-717).  out: [batch x n_items] row-major. */
int g4r_predict(g4r_handle* h, const int32_t* X, int32_t batch, const uint8_t* reset_mask, float* out);
#define G4R_TOPK_MAX 1024
/* predict_next_batch's device call, reduced on the device to the k best items of every lane (ranking key and ties: DESIGN §3d).
 * Advances the scoring-path hidden state like g4r_predict.  out_items / out_scores: [batch x k] row-major, best first.
 * G4R_ERR_INVALID unless 1 <= k <= min(n_items, G4R_TOPK_MAX); G4R_ERR_INDEX on an out-of-range item. */
int g4r_predict_topk(g4r_handle* h, const int32_t* X, int32_t batch, const uint8_t* reset_mask, int32_t k,
                     int32_t* out_items, float* out_scores);
/* g4r_predict_topk with filters (DESIGN §3d).  Only the distinct items of cand[0 .. n_cand) compete (cand == NULL: the whole
 * catalogue; duplicates ignored); lane b never receives items excl_items[excl_off[b] .. excl_off[b+1]) (excl_off == NULL: no
 * exclusions; lists need not be sorted, duplicates allowed).  Ranking key, tie rule and scores as g4r_predict_topk, except that
 * the softmax / softmax_logit normaliser runs over the distinct candidates; exclusions never change a score.  Slots past a
 * lane's eligible items: item -1, score NaN.  G4R_ERR_INVALID unless 1 <= k <= min(distinct candidates, G4R_TOPK_MAX) and
 * excl_off is non-decreasing from 0; G4R_ERR_INDEX on an out-of-range item.  Any error leaves the hidden state untouched.
 * The candidate set is kept on the device between calls and re-uploaded only when its content changes. */
int g4r_predict_topk_filtered(g4r_handle* h, const int32_t* X, int32_t batch, const uint8_t* reset_mask, int32_t k,
                              const int32_t* cand, int64_t n_cand, const int64_t* excl_off, const int32_t* excl_items,
                              int32_t* out_items, float* out_scores);
/* Zero the scoring-path hidden state (gru4rec.py:696-697). */
int g4r_reset_eval_hidden(g4r_handle* h);

/* ---- session store: scoring-path state addressed by session key (DESIGN §3e; no reference counterpart) ----------------------
 * An int64 session key maps to a row of a device table of `capacity` hidden states per layer, separate from the lanes of
 * g4r_predict / g4r_predict_topk and from the training state.  Every event that names a session makes it the most recently used,
 * in call order.  A key not in the store takes a free row, else the row of the least recently used session that the call does
 * not name; that session's state and history are dropped, and the new session starts from a zero state.  The store also keeps
 * each session's input items since it entered (exclude_seen).  Every argument is checked before the store changes: after an
 * error, keys, recency order, states and histories are as they were.  G4R_ERR_INVALID when a call names more distinct keys than
 * the capacity; G4R_ERR_INDEX on an out-of-range item; G4R_ERR_STATE on a row-sharded multi-GPU handle or before
 * g4r_sessions_open.  The results do not depend on how the events of a session are spread over calls. */
/* (Re)creates an empty store of `capacity` sessions (1 .. 2^31 - 1); an existing store is dropped. */
int g4r_sessions_open(g4r_handle* h, int64_t capacity);
/* Number of sessions in the store (0 if none is open); *n_history_items (may be NULL): total length of their histories. */
int64_t g4r_sessions_count(const g4r_handle* h, int64_t* n_history_items);
/* Advances sessions without scoring: event i feeds item X[i] to session keys[i].  Keys may repeat; the events of one key apply
 * in call order.  The whole call runs on the device without host round trips. */
int g4r_sessions_feed(g4r_handle* h, const int64_t* keys, const int32_t* X, int64_t n);
/* Advances session keys[i] by item X[i] and ranks its next items as g4r_predict_topk_filtered ranks a lane (same ranking key,
 * ties, scores, filters and empty slots): out_items / out_scores [n x k].  Each key at most once per call (G4R_ERR_INVALID
 * otherwise); any n (the call runs in chunks of the scoring lanes).  excl_off / excl_items: per-event exclusions as in
 * g4r_predict_topk_filtered (excl_off has n + 1 entries).  exclude_seen != 0: the session's history, this input included, is
 * excluded too. */
int g4r_sessions_topk(g4r_handle* h, const int64_t* keys, const int32_t* X, int64_t n, int32_t k,
                      const int32_t* cand, int64_t n_cand, const int64_t* excl_off, const int32_t* excl_items,
                      int32_t exclude_seen, int32_t* out_items, float* out_scores);
/* Drops the sessions keys[0 .. n) (unknown keys ignored); keys == NULL: every session. */
int g4r_sessions_end(g4r_handle* h, const int64_t* keys, int64_t n);
/* Every session, least recently used first (sizes from g4r_sessions_count): keys [n], states [n x sum of layer widths] (the
 * layers' states concatenated), histories as CSR: hist_off [n + 1], hist_items [n_history_items].  Any pointer may be NULL. */
int g4r_sessions_export(g4r_handle* h, int64_t* keys, float* states, int64_t* hist_off, int32_t* hist_items);
/* Inserts n sessions in order as the most recently used (layouts of g4r_sessions_export; hist_off == NULL: empty histories).
 * A key already in the store is overwritten; keys must be distinct, and at most the capacity.  Other sessions may be evicted. */
int g4r_sessions_import(g4r_handle* h, const int64_t* keys, const float* states, const int64_t* hist_off,
                        const int32_t* hist_items, int64_t n);

/* ---- session baselines: ItemKNN, Pop and SessionPop of the reference's baselines.py (baselines.py:52-301; DESIGN §3j) -------
 * (BPR-MF and SessionKNN below share the handle and g4r_bl_evaluate.)
 * A separate handle: a baseline has no training config.  Item indices are 0 .. n_items - 1.  Every argument is checked before any
 * device work; G4R_ERR_STATE for a call the handle's kind does not have or before the model is fitted. */
typedef struct g4r_baselines g4r_baselines;
#define G4R_BL_POP 0
#define G4R_BL_SESSIONPOP 1
#define G4R_BL_ITEMKNN 2
/* n_keep: n_sims of ItemKNN (1 .. 1024), top_n of Pop / SessionPop.  Device memory is allocated by the library. */
int g4r_bl_create(int32_t kind, int32_t n_items, int32_t n_keep, int32_t device, g4r_baselines** out);
int g4r_bl_destroy(g4r_baselines* b);
const char* g4r_bl_last_error(const g4r_baselines* b);   /* b may be NULL: last creation error */
/* ItemKNN fit (baselines.py:235-276) from the training events as session CSR (items[session_offsets[s] .. session_offsets[s+1]),
 * any order within a session) and the caller's norm factors a[i] = (supp_i + lmbd)^alpha, b[j] = (supp_j + lmbd)^(1 - alpha)
 * (finite, >= 0).  cnt(i, j) = sum over sessions s of (occurrences of i in s) * [j in s], cnt(i, i) = 0; sim = cnt / (a_i * b_j)
 * (a zero norm counts as 1), each product and quotient correctly rounded in float64; each row keeps its n_keep largest positive
 * sims by (sim desc, index asc).  Out (may be NULL): the pair work sum_s n_s d_s (events x distinct items per session), the
 * scratch bytes of the accumulators, the device time (CUDA events) from the first kernel that derives the per-session and per-item
 * lists from the uploaded events to the last kernel of the fit.  After the upload everything runs on the device. */
int g4r_bl_knn_fit(g4r_baselines* b, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_events,
                   const double* a, const double* bf, int64_t* pair_work, size_t* scratch_bytes, float* device_ms);
/* Pop / SessionPop scores (baselines.py:79-118,146-161): n = n_items float64, 0 past the top_n (at most top_n positive). */
int g4r_bl_set_pop(g4r_baselines* b, const double* scores, int64_t n);
/* ItemKNN rows: idx [n_items x n_keep] (-1 past len), sim [n_items x n_keep] float64 (0 past len), len [n_items].  Import checks
 * every row (indices, positive finite sims, (sim desc, index asc) order) before it changes anything. */
int g4r_bl_rows_export(g4r_baselines* b, int32_t* idx, double* sim, int32_t* len);
int g4r_bl_rows_import(g4r_baselines* b, const int32_t* idx, const double* sim, const int32_t* len);
/* evaluate_gpu / evaluate_events of a baseline.  Sessions as CSR of item indices; n_history (NULL: none) as in
 * g4r_schedule_build_history: an event is counted when its target lies past the session's first max(n_history, 1) events.  Each
 * counted event (input items[p], target items[p + 1], session items so far items[start .. p]) is ranked against the competitors:
 * the catalogue, or the multiset cand[0 .. n_cand) (the target competes only if listed).  exclude_seen: the session's items so
 * far leave the competitors and a target among them is a miss, (-1, -1).  mode 0 .. 3 as g4r_eval_schedule; 'tiebreaking' adds
 * U(0,1) * 1e-10 to every float64 score, a counter hash of (counted event, item).  recall_sum / mrr_sum: n_cut sums (a hit when
 * rank <= N); *n_counted: counted events.  out_counts (may be NULL): [n_counted x 2] (#greater, #equal incl. the target), in data
 * order.  k > 0: the k best eligible distinct competitors of each event by (score desc, index asc), zero scores included, into
 * out_items / out_scores [n_counted x k] (item -1, score NaN past the eligible ones).  G4R_ERR_INVALID unless
 * 0 <= k <= min(distinct competitors, 1024). */
int g4r_bl_evaluate(g4r_baselines* b, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                    const int32_t* n_history, int32_t mode, const int32_t* cut_off, int32_t n_cut, const int32_t* cand, int64_t n_cand,
                    int32_t exclude_seen, int32_t k, double* recall_sum, double* mrr_sum, int64_t* n_counted,
                    int32_t* out_counts, int32_t* out_items, double* out_scores);

/* ---- BPR-MF of the reference's baselines.py (BPR, baselines.py:303-418; DESIGN §3k) ---------------------------------------------
 * g4r_bl_create(G4R_BL_BPR, n_items, n_factors (1 .. 1024), ...).  The fit replays the caller's random draws and applies the
 * reference's SGD updates in its order, in float64; the result equals a strictly sequential run bit for bit. */
#define G4R_BL_BPR 3
/* Begins a fit: the training rows (the reference's merged frame, in its order) as session and item indices, and the initial
 * factors U [n_sessions x n_factors], I [n_items x n_factors] and biases bI [n_items] (bI is never updated, but scores add it).
 * n_items <= n_rows <= (2^31 - 1) / 3 (the negative draws index rows below n_items; a merged frame has a row per item at least)
 * and n_sessions + n_items < 2^32 - 1.  The device must hold U, I and 92 bytes per row; the call refuses with G4R_ERR_CUDA and a
 * message naming the sizes otherwise. */
int g4r_bl_bpr_begin(g4r_baselines* b, const int32_t* row_session, const int32_t* row_item, int64_t n_rows, int64_t n_sessions,
                     const double* U, const double* I, const double* bI);
/* One iteration: for t = 0 .. n_rows - 1, row e = perm[t] (a permutation of the rows), u, p its session and item, n the item of
 * row negrow[t] (0 <= negrow[t] < n_items <= n_rows), the update of baselines.py:349-358 with uF, I[p], I[n] read before it.  max_warps >= 1
 * bounds the warps that apply updates at once (1: one warp in order; the result is the same).  Out (may be NULL): the mean of
 * log(sigm) over the events (summed in a fixed order), the largest level (1 + the largest level of the event's predecessors on
 * its rows: the longest chain of dependent updates) and the device time (CUDA events) from the predecessor sort to the mean. */
int g4r_bl_bpr_iterate(g4r_baselines* b, const int32_t* perm, const int32_t* negrow, double learning_rate, double lambda_session,
                       double lambda_item, int32_t max_warps, double* mean_log_sigm, int64_t* max_level, float* device_ms);
/* The fit's U [n_sessions x n_factors] (NULL: skipped; G4R_ERR_STATE unless a fit has begun) and I [n_items x n_factors]. */
int g4r_bl_bpr_export(g4r_baselines* b, double* U, double* I);
/* The item factors and biases of a fitted model (a model loaded from a pickle); ends any fit in progress.  g4r_bl_evaluate of a
 * BPR handle scores item j after input p as (sum over f = 0 .. n_factors - 1 in order of I[j,f] * uF[f]) + bI[j], every product
 * and sum correctly rounded in float64, uF the mean of I over the session's items[start .. p]. */
int g4r_bl_bpr_import(g4r_baselines* b, const double* I, const double* bI);

/* ---- session-based kNN: S-KNN (cosine) and V-SKNN-style position weights (DESIGN §3o) -------------------------------------------
 * g4r_bl_create(G4R_BL_SKNN, n_items, k (1 .. 1024), ...).  Kind 4 is not used. */
#define G4R_BL_SKNN 5
/* The index: the training sessions' distinct items as CSR (items[session_offsets[s] .. session_offsets[s+1]) strictly ascending),
 * recency[s] the rank of session s in recency order (a permutation of 0 .. n_sessions - 1, 0 the most recent), sample_size
 * 1 .. 8192 (k <= sample_size), similarity 0 (cosine) or 1 (vector).  The library builds every item's sessions in recency order
 * and keeps both on the device; a later call replaces the index.  g4r_bl_evaluate of a SessionKNN handle ranks each counted
 * event by the scores of DESIGN §3o: the candidates are the first sample_size training sessions in recency order that share an
 * item with the session's items[start .. p]; the k most similar (ties: the more recent) are the neighbours, and item j scores
 * the sum, in float64 in neighbour order, of the similarities of the neighbours that contain j. */
int g4r_bl_sknn_fit(g4r_baselines* b, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_entries,
                    const int32_t* recency, int32_t sample_size, int32_t similarity);

/* ---- STAN-style time- and position-aware session kNN (DESIGN §3p) ---------------------------------------------------------------
 * g4r_bl_create(G4R_BL_STAN, n_items, k (1 .. 1024), ...).  The SessionKNN index plus three decay tables the caller computes, so
 * the device only multiplies, adds, divides and takes square roots (correctly rounded). */
#define G4R_BL_STAN 6
/* The index as g4r_bl_sknn_fit's, plus: positions[e] the 1-based position of items[e]'s last occurrence in its session (distinct
 * within a session, 1 .. n_w3), w2[s] session s's recency weight in [0, 1] (sessions in the order of session_offsets), and
 * w3[0 .. n_w3) the in-neighbour distance weights in [0, 1], n_w3 the longest training session's length in events.  Every
 * argument is checked before any device write; a later call replaces the index (not W1). */
int g4r_bl_stan_fit(g4r_baselines* b, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_entries,
                    const int32_t* positions, const int32_t* recency, const double* w2, const double* w3, int64_t n_w3,
                    int32_t sample_size);
/* W1[0 .. n_w1): the weight of a prefix item at distance d = t - p from the current input, entries in [0, 1]; replaces any
 * earlier table.  g4r_bl_evaluate of a STAN handle refuses (G4R_ERR_INVALID, before any device work) a frame with a counted event
 * whose prefix is longer than n_w1.  It ranks by DESIGN §3p: v(n) the sum of W1[t - p_i] over the shared items in ascending p_i,
 * sim(n) = v / sqrt(|I(c)| |I(n)|) * w2[n]; the k largest (ties: the more recent) are the neighbours; item j scores the sum, in
 * neighbour order, of sim(n) * w3[|q_n(j) - q_n(r(n))|], r(n) the shared item with the largest p_i; each product and sum
 * correctly rounded in float64.  Lists hold the positive scores first, then every zero-score item by index. */
int g4r_bl_stan_set_w1(g4r_baselines* b, const double* w1, int64_t n_w1);

/* ---- rule-based baselines: sequential rules (SR) and association rules (AR) (DESIGN §3q) --------------------------------------
 * g4r_bl_create(G4R_BL_SR or G4R_BL_AR, n_items, pruning (1 .. 1024), ...).  Kind 7 is not used.  The model is ItemKNN's rows:
 * g4r_bl_rows_export / g4r_bl_rows_import take SR and AR handles, and g4r_bl_evaluate ranks them as an ItemKNN (after input x,
 * item j scores its kept weight w(x, j), every other item 0). */
#define G4R_BL_SR 8
#define G4R_BL_AR 9
/* The fit, from the training events as session CSR in time order (items[session_offsets[s] .. session_offsets[s+1]) = x_1 .. x_n).
 * SR (steps 1 .. 20, weighting 0 'div' or 1 'same'): W(i, j) = sum over sessions and position pairs p < q <= p + steps with
 * x_p = i != j = x_q of L / (q - p) ('div', L = lcm(1 .. steps)) or 1 ('same', L = 1).  AR (steps = weighting = 0): W(i, j) =
 * sum over sessions of occ_s(i) * occ_s(j), i != j, L = 1.  W is counted in uint64; w = double(W) / L, each conversion and the
 * division correctly rounded.  Each row keeps its n_keep largest positive w by (w desc, index asc).  Every argument is checked
 * before any device write, and G4R_ERR_INVALID refuses a fit whose per-row bound (SR: occurrences * min(steps, longest session -
 * 1) * L; AR: the sum of n_s over the row item's occurrences) reaches 2^63.  Out (may be NULL): the pair work (the pairs the fit
 * visits), the scratch bytes of the accumulators, the device time (CUDA events) from the first kernel to the last. */
int g4r_bl_rules_fit(g4r_baselines* b, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_events,
                     int32_t steps, int32_t weighting, int64_t* pair_work, size_t* scratch_bytes, float* device_ms);

/* ---- VSTAN-style session kNN (DESIGN §3r) -----------------------------------------------------------------------------------------
 * g4r_bl_create(G4R_BL_VSTAN, n_items, k (1 .. 1024), ...); kind 10 is not used.  STAN plus a vector similarity, a neighbour weight by the prefix
 * distance of its most recent shared item and a per-item factor (IDF), all from tables the caller computes.  The index and W1 are
 * STAN's: g4r_bl_stan_fit and g4r_bl_stan_set_w1 take a VSTAN handle. */
#define G4R_BL_VSTAN 11
/* similarity 0 (cosine, STAN's sim) or 1 (vector: no norm), f[0 .. n_items) the item factors (finite, >= 0), w4[0 .. n_w4) the
 * neighbour weights by prefix distance, entries in [0, 1], n_w4 in 1 .. 2^30.  Every argument is checked before any device write;
 * a call replaces the earlier settings, and a fit clears them: g4r_bl_evaluate of a VSTAN handle returns G4R_ERR_STATE until this
 * has been called after the last fit, and refuses (G4R_ERR_INVALID, before any device work) a frame with a counted event whose
 * prefix is longer than n_w4 or n_w1.  It ranks by DESIGN §3r: sim1 = v (vector) or v / sqrt(|I(c)| |I(n)|) (cosine), sim2 =
 * sim1 * w2[n]; the neighbours are STAN's by sim2; g(n) = sim2 * w4[t - p_r(n)]; item j scores f[j] times the sum, in neighbour
 * order, of g(n) * w3[|q_n(j) - q_n(r(n))|]; each product and sum correctly rounded in float64. */
int g4r_bl_vstan_set(g4r_baselines* b, int32_t similarity, const double* f, int64_t n_f, const double* w4, int64_t n_w4);

/* ---- NARM neural session baseline (DESIGN §3s) -----------------------------------------------------------------------------------
 * g4r_bl_create(G4R_BL_NARM, n_items, d_e (1 .. 1024), ...).  The model is one flat float32 vector: E [n_items x d_e], Wx
 * [d_e x 3H], Wrz [H x 2H], Wh [H x H], Bh [3H], A1 [H x H], A2 [H x H], v [H], B [d_e x 2H], n_params = n_items d_e + 5 d_e H +
 * 5 H^2 + 4 H.  For inputs x_1 .. x_t: h_j the GRU of GRU4Rec's cell over E[x] from a zero state, alpha_j = v . sig(A1 h_t +
 * A2 h_j), c = [h_t ; sum_j alpha_j h_j], q = B c, score(i) = E[i] . q. */
#define G4R_BL_NARM 12
/* Begins a fit: hidden 1 .. 1024, max_len 2 .. 512, batch_size >= 1, the training pieces as CSR (items[piece_offsets[k] ..
 * piece_offsets[k+1]), 2 .. max_len events each: inputs are every event but the last, targets every event but the first) and the
 * initial parameters.  Adam's moments start at 0.  Every argument is checked before any device write; G4R_ERR_CUDA with a message
 * naming the sizes if the device cannot hold the largest batch's logits (positions x n_items floats) and scratch. */
int g4r_bl_narm_begin(g4r_baselines* b, int32_t hidden, int32_t max_len, int32_t batch_size, const int64_t* piece_offsets, int64_t n_pieces,
                      const int32_t* items, int64_t n_entries, const float* params, int64_t n_params);
/* One epoch: mini-batches of batch_size consecutive entries of order (piece indices; the last batch may be smaller), each the mean
 * full-catalogue cross-entropy over its positions and one Adam step (b1 0.9, b2 0.999, eps 1e-8, bias-corrected) on every
 * parameter, with dropout masks of global step = the steps since g4r_bl_narm_begin.  No host round trip inside.  A batch may
 * hold at most as many positions (inputs) as the batch_size longest distinct pieces, the scratch g4r_bl_narm_begin sized: a
 * batch that repeats a long piece past that bound refuses the call (G4R_ERR_INVALID) before any device write.  Out (may be
 * NULL): losses[ceil(n_order / batch_size)] and the device time (CUDA events). */
int g4r_bl_narm_epoch(g4r_baselines* b, const int32_t* order, int64_t n_order, uint32_t seed, float learning_rate, float dropout_emb,
                      float dropout_ct, float* losses, float* device_ms);
/* One mini-batch of n <= batch_size pieces at the current parameters, without an update: the mean loss and the gradient of every
 * parameter (n_params floats, the parameters' layout), dropout masks of global step `step`.  The pieces obey
 * g4r_bl_narm_epoch's bound on a batch's positions. */
int g4r_bl_narm_grads(g4r_baselines* b, const int32_t* pieces, int32_t n, uint32_t seed, int64_t step, float dropout_emb, float dropout_ct,
                      float* loss, float* grads);
/* The parameters (n_params floats). */
int g4r_bl_narm_export(g4r_baselines* b, float* params, int64_t n_params);
/* The parameters of a fitted model (a model loaded from a pickle); ends any fit in progress. */
int g4r_bl_narm_import(g4r_baselines* b, int32_t hidden, int32_t max_len, const float* params, int64_t n_params);
/* Every counted event's q (eval mode, the last max_len inputs of items[start .. p]) in g4r_bl_evaluate's order: q [n_q x d_e],
 * n_q the number of counted events.  g4r_bl_evaluate of a NARM handle ranks these q as a BPR handle ranks its session vectors,
 * with I = double(E) and bI = 0. */
int g4r_bl_narm_encode(g4r_baselines* b, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                       const int32_t* n_history, float* q, int64_t n_q);

/* ---- SASRec self-attentive session baseline (DESIGN §3t) -------------------------------------------------------------------------
 * g4r_bl_create(G4R_BL_SASREC, n_items, d (1 .. 1024), ...).  The model is one flat float32 vector: E [n_items x d] (the input
 * embedding and the output item side), Pe [max_len x d], per block g1, c1 [d], Wq, bq, Wk, bk, Wv, bv, Wo, bo ([d x d], [d]), g2,
 * c2 [d], W1, b1, W2, b2 ([d x d], [d]), then gf, cf [d]; n_params = n_items d + max_len d + n_blocks (6 d^2 + 10 d) + 2 d.  For
 * inputs x_0 .. x_(n-1): h_t = E[x_t] s_d + Pe[t]; per block u = LN1(h), causal multi-head softmax attention over u Wq + bq,
 * u Wk + bk, u Wv + bv with scale s_h, a = h + A Wo + bo, h = a + relu(LN2(a) W1 + b1) W2 + b2; q_t = LNf(h_t), score(i) = E[i] . q.
 * LN(x) = g (x - mean) / sqrt(var + 1e-8) + c over d; s_d and s_h the float32 of sqrt(d) and 1 / sqrt(d / n_heads). */
#define G4R_BL_SASREC 13
/* Begins a fit: n_blocks 1 .. 8, n_heads dividing d, max_len 1 .. 512, batch_size >= 1 with (n_blocks + 1) batch_size max_len d
 * < 2^32, the training pieces as CSR (2 .. max_len + 1 events each: inputs every event but the last, targets every event but the
 * first) and the initial parameters.  Adam's moments start at 0.  Every argument is checked before any device write; G4R_ERR_CUDA
 * with a message naming the sizes if the device cannot hold the largest batch's logits and activations. */
int g4r_bl_sasrec_begin(g4r_baselines* b, int32_t n_blocks, int32_t n_heads, int32_t max_len, int32_t batch_size, const int64_t* piece_offsets,
                        int64_t n_pieces, const int32_t* items, int64_t n_entries, const float* params, int64_t n_params);
/* One epoch, as g4r_bl_narm_epoch: mini-batches of batch_size consecutive entries of order, the mean full-catalogue cross-entropy
 * over the batch's positions and one Adam step each, dropout (rate in [0, 1)) on h0 and on both residual branches of every block.
 * A batch past the positions of the batch_size longest distinct pieces is refused before any device write. */
int g4r_bl_sasrec_epoch(g4r_baselines* b, const int32_t* order, int64_t n_order, uint32_t seed, float learning_rate, float dropout,
                        float* losses, float* device_ms);
/* One mini-batch of n <= batch_size pieces at the current parameters, without an update: the mean loss and every gradient. */
int g4r_bl_sasrec_grads(g4r_baselines* b, const int32_t* pieces, int32_t n, uint32_t seed, int64_t step, float dropout, float* loss,
                        float* grads);
int g4r_bl_sasrec_export(g4r_baselines* b, float* params, int64_t n_params);
/* The parameters of a fitted model (finite); ends any fit in progress. */
int g4r_bl_sasrec_import(g4r_baselines* b, int32_t n_blocks, int32_t n_heads, int32_t max_len, const float* params, int64_t n_params);
/* Every counted event's q (eval mode, the last max_len inputs of items[start .. p], positions counted from the first of them) in
 * g4r_bl_evaluate's order.  g4r_bl_evaluate of a SASRec handle ranks these q as NARM's, with I = double(E) and bI = 0. */
int g4r_bl_sasrec_encode(g4r_baselines* b, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                         const int32_t* n_history, float* q, int64_t n_q);

/* ---- SR-GNN session-graph baseline (DESIGN §3u) -----------------------------------------------------------------------------------
 * g4r_bl_create(G4R_BL_SRGNN, n_items, d (1 .. 1024), ...).  The model is one flat float32 vector: E [n_items x d] (the node
 * embedding and the scored item side), W_in, W_out [d x d], b_in, b_out, b_iah, b_oah [d], W_ih [2d x 3d], b_ih [3d], W_hh [d x 3d],
 * b_hh [3d], W1, W2 [d x d], b1, b2, q [d], W3 [2d x d], b3 [d]; n_params = n_items d + 15 d^2 + 14 d.  For the last max_len inputs
 * x_1 .. x_n of a prefix: the nodes are its distinct items ascending, edges u -> v for each consecutive pair (a repeat once,
 * self-loops kept), A_in[v][u] = 1 / indeg(v), A_out[u][v] = 1 / outdeg(u); from H = E[nodes], `step` times
 * a = [A_in (H W_in + b_in) + b_iah ; A_out (H W_out + b_out) + b_oah], gi = a W_ih + b_ih, gh = H W_hh + b_hh in (r, z, n) thirds,
 * r = sig(gi_r + gh_r), z = sig(gi_z + gh_z), n = tanh(gi_n + r gh_n), H = n + z (H - n); then h_t = H[node of x_t], s_l = h_n,
 * alpha_t = q . sig(s_l W1 + b1 + h_t W2 + b2), s_g = sum_t alpha_t h_t, s_h = [s_g ; s_l] W3 + b3 and score(i) = E[i] . s_h. */
#define G4R_BL_SRGNN 15
/* Begins a fit: step 1 .. 8, max_len 1 .. 512, batch_size >= 1 with batch_size max_len (step + 1) 3 d < 2^31, the training
 * sessions as CSR (events in time order) and the initial parameters.  The samples are every (prefix, next item) pair in session
 * order, the prefix cut to its last max_len inputs: sample k of g4r_bl_srgnn_epoch / _grads counts them from 0.  Adam's moments
 * start at 0.  Every argument is checked before any device write; G4R_ERR_CUDA with a message naming the sizes if the device
 * cannot hold the largest batch's logits and activations. */
int g4r_bl_srgnn_begin(g4r_baselines* b, int32_t step, int32_t max_len, int32_t batch_size, const int64_t* session_offsets, int64_t n_sessions,
                       const int32_t* items, int64_t n_entries, const float* params, int64_t n_params);
/* One epoch: mini-batches of batch_size consecutive samples of order, the mean full-catalogue cross-entropy over the batch's
 * samples and one Adam step each (NARM's constants) on gradient + l2 theta over every parameter.  A batch past the positions
 * of the batch_size longest samples is refused before any device write. */
int g4r_bl_srgnn_epoch(g4r_baselines* b, const int32_t* order, int64_t n_order, float learning_rate, float l2, float* losses, float* device_ms);
/* One mini-batch of n <= batch_size samples at the current parameters, without an update: the mean loss and its gradient (no L2). */
int g4r_bl_srgnn_grads(g4r_baselines* b, const int32_t* samples, int32_t n, float* loss, float* grads);
int g4r_bl_srgnn_export(g4r_baselines* b, float* params, int64_t n_params);
/* The parameters of a fitted model (finite); ends any fit in progress. */
int g4r_bl_srgnn_import(g4r_baselines* b, int32_t step, int32_t max_len, const float* params, int64_t n_params);
/* Every counted event's s_h (the graph of the last max_len inputs of items[start .. p]) in g4r_bl_evaluate's order.
 * g4r_bl_evaluate of an SR-GNN handle ranks these s_h as NARM's q, with I = double(E) and bI = 0. */
int g4r_bl_srgnn_encode(g4r_baselines* b, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                        const int32_t* n_history, float* q, int64_t n_q);

/* ---- STAMP short-term attention/memory baseline (DESIGN §3v) ----------------------------------------------------------------------
 * g4r_bl_create(G4R_BL_STAMP, n_items, d (1 .. 1024), ...).  The model is one flat float32 vector: E [n_items x d] (the input
 * embedding and the scored item side), W1, W2, W3 [d x d], b_a, w0 [d], Ws [d x d], bs [d], Wt [d x d], bt [d]; n_params =
 * n_items d + 5 d^2 + 4 d.  For the last max_len inputs x_1 .. x_n of a prefix (rows of E): m_s = (1/n) sum_i x_i, m_t = x_n,
 * a_i = w0 . sig(x_i W1 + m_t W2 + m_s W3 + b_a) (not normalised over i), m_a = sum_i a_i x_i, h_s = tanh(m_a Ws + bs),
 * h_t = tanh(m_t Wt + bt), q = h_s * h_t (elementwise) and score(i) = E[i] . q. */
#define G4R_BL_STAMP 17
/* Begins a fit: max_len 1 .. 512, batch_size >= 1 with batch_size max_len 2 d < 2^31, the training sessions as CSR (events in
 * time order) and the initial parameters.  The samples are every (prefix, next item) pair in session order, the prefix cut to its
 * last max_len inputs (SR-GNN's): sample k of g4r_bl_stamp_epoch / _grads counts them from 0.  Adam's moments start at 0.  Every
 * argument is checked before any device write; G4R_ERR_CUDA with a message naming the sizes if the device cannot hold the
 * largest batch's logits and activations. */
int g4r_bl_stamp_begin(g4r_baselines* b, int32_t max_len, int32_t batch_size, const int64_t* session_offsets, int64_t n_sessions,
                       const int32_t* items, int64_t n_entries, const float* params, int64_t n_params);
/* One epoch: mini-batches of batch_size consecutive samples of order, the mean full-catalogue cross-entropy over the batch's
 * samples and one Adam step each (NARM's constants, no L2).  A batch past the positions of the batch_size longest samples is
 * refused before any device write. */
int g4r_bl_stamp_epoch(g4r_baselines* b, const int32_t* order, int64_t n_order, float learning_rate, float* losses, float* device_ms);
/* One mini-batch of n <= batch_size samples at the current parameters, without an update: the mean loss and its gradient. */
int g4r_bl_stamp_grads(g4r_baselines* b, const int32_t* samples, int32_t n, float* loss, float* grads);
int g4r_bl_stamp_export(g4r_baselines* b, float* params, int64_t n_params);
/* The parameters of a fitted model (finite); ends any fit in progress. */
int g4r_bl_stamp_import(g4r_baselines* b, int32_t max_len, const float* params, int64_t n_params);
/* Every counted event's q (the last max_len inputs of items[start .. p]) in g4r_bl_evaluate's order.
 * g4r_bl_evaluate of a STAMP handle ranks these q as NARM's, with I = double(E) and bI = 0. */
int g4r_bl_stamp_encode(g4r_baselines* b, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                        const int32_t* n_history, float* q, int64_t n_q);

/* ---- NextItNet convolutional baseline (DESIGN §3w) -----------------------------------------------------------------------------
 * g4r_bl_create(G4R_BL_NEXTITNET, n_items, d (1 .. 1024), ...); kind 18 is not used.  The model is one flat float32 vector:
 * E [n_items x d] (the input embedding), per block b (one per dilation l_b) C1 [K d x d], c1, g1, n1 [d], C2 [K d x d], c2, g2,
 * n2 [d] (row k d + i of a kernel: tap k, input channel i), then W [n_items x d] and bW [n_items] (the scored item side);
 * n_params = 2 n_items d + n_items + n_dilations (2 K d^2 + 6 d).  For the inputs x_0 .. x_(n-1) of a piece or window, positions before 0 reading zeros: h_t = E[x_t];
 * per block u_t = c1 + sum_k h_(t - (K-1-k) l) C1[k], a = relu(LN1(u)), v_t = c2 + sum_k a_(t - (K-1-k) 2l) C2[k],
 * h'_t = h_t + relu(LN2(v)); q_t = h_t after the last block and score(i) = W[i] . q_t + bW[i].  LN is SASRec's (eps 1e-8). */
#define G4R_BL_NEXTITNET 19
/* Begins a fit: 1 .. 16 dilations each in 1 .. 256, kernel_size 1 .. 8, max_len 1 .. 512, batch_size >= 1, the training pieces as
 * CSR (2 .. max_len + 1 events each, inputs then the last target) and the initial parameters.  Adam's moments start at 0.  Every
 * argument is checked before any device write; G4R_ERR_CUDA with a message naming the sizes if the device cannot hold the largest
 * batch's logits and activations. */
int g4r_bl_nextitnet_begin(g4r_baselines* b, const int32_t* dilations, int32_t n_dilations, int32_t kernel_size, int32_t max_len,
                           int32_t batch_size, const int64_t* piece_offsets, int64_t n_pieces, const int32_t* items, int64_t n_entries,
                           const float* params, int64_t n_params);
/* One epoch: mini-batches of batch_size consecutive pieces of order, the mean full-catalogue cross-entropy over the batch's
 * positions and one Adam step each (NARM's constants).  A batch past the positions of the batch_size longest pieces is refused
 * before any device write. */
int g4r_bl_nextitnet_epoch(g4r_baselines* b, const int32_t* order, int64_t n_order, float learning_rate, float* losses, float* device_ms);
/* One mini-batch of n <= batch_size pieces at the current parameters, without an update: the mean loss and its gradient. */
int g4r_bl_nextitnet_grads(g4r_baselines* b, const int32_t* pieces, int32_t n, float* loss, float* grads);
int g4r_bl_nextitnet_export(g4r_baselines* b, float* params, int64_t n_params);
/* The parameters of a fitted model (finite); ends any fit in progress. */
int g4r_bl_nextitnet_import(g4r_baselines* b, const int32_t* dilations, int32_t n_dilations, int32_t kernel_size, int32_t max_len,
                            const float* params, int64_t n_params);
/* Every counted event's q (the last max_len inputs of items[start .. p]) in g4r_bl_evaluate's order.
 * g4r_bl_evaluate of a NextItNet handle ranks these q as NARM's, with I = double(W) and bI = double(bW). */
int g4r_bl_nextitnet_encode(g4r_baselines* b, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                            const int32_t* n_history, float* q, int64_t n_q);

/* ---- BERT4Rec bidirectional baseline (DESIGN §3x) ------------------------------------------------------------------------------
 * g4r_bl_create(G4R_BL_BERT4REC, n_items, d (1 .. 1024), ...); kind 20 is not used.  The model is one flat float32 vector:
 * E [(n_items + 1) x d] (row n_items the mask token; rows 0 .. n_items - 1 the input embedding and the scored item side),
 * Pe [max_len x d], g0, c0 [d], per block Wq, bq, Wk, bk, Wv, bv, Wo, bo ([d x d], [d]), g1, c1 [d], W1 [d x 4d], b1 [4d],
 * W2 [4d x d], b2, g2, c2 [d], then Wp [d x d], bp, gp, cp [d] and bO [n_items];
 * n_params = (n_items + 1) d + max_len d + 2 d + n_blocks (12 d^2 + 13 d) + d^2 + 3 d + n_items.
 * For inputs x_0 .. x_(n-1) (some of them the mask token): h = drop(LN0(E[x_t] + Pe[t])); per block a = LN1(h + drop(A Wo + bo)),
 * A multi-head softmax attention over all n positions (scale 1 / sqrt(d / n_heads)), h = LN2(a + drop(gelu(a W1 + b1) W2 + b2))
 * (exact-erf GELU); q_t = LNp(gelu(h_t Wp + bp)) and score(i) = E[i] . q_t + bO[i] over the n_items real items.  LN is SASRec's
 * (eps 1e-8). */
#define G4R_BL_BERT4REC 21
/* Begins a fit: n_blocks 1 .. 8, n_heads dividing d, max_len 2 .. 512, batch_size >= 1, the training pieces as CSR (2 .. max_len
 * events each, all of them inputs) and the initial parameters.  Adam's moments start at 0.  Every argument is checked before any
 * device write; G4R_ERR_CUDA with a message naming the sizes if the device cannot hold the largest batch's logits and activations. */
int g4r_bl_bert4rec_begin(g4r_baselines* b, int32_t n_blocks, int32_t n_heads, int32_t max_len, int32_t batch_size, const int64_t* piece_offsets,
                          int64_t n_pieces, const int32_t* items, int64_t n_entries, const float* params, int64_t n_params);
/* One epoch: mini-batches of batch_size consecutive pieces of order, masks one byte (0 or 1) per stored entry (n_masks = n_entries,
 * at least one masked entry in every piece used): each masked entry is replaced by the mask token, and the mean full-catalogue
 * cross-entropy over the batch's masked positions takes one Adam step (NARM's constants).  dropout in [0, 1) on h0 and both
 * residual branches of every block, keyed by (seed, global step).  A batch past the positions of the batch_size longest pieces is
 * refused before any device write. */
int g4r_bl_bert4rec_epoch(g4r_baselines* b, const int32_t* order, int64_t n_order, const uint8_t* masks, int64_t n_masks, uint32_t seed,
                          float learning_rate, float dropout, float* losses, float* device_ms);
/* One mini-batch of n <= batch_size pieces at the current parameters and the given step's dropout, without an update: the mean
 * loss and its gradient. */
int g4r_bl_bert4rec_grads(g4r_baselines* b, const int32_t* pieces, int32_t n, const uint8_t* masks, int64_t n_masks, uint32_t seed, int64_t step,
                          float dropout, float* loss, float* grads);
int g4r_bl_bert4rec_export(g4r_baselines* b, float* params, int64_t n_params);
/* The parameters of a fitted model (finite); ends any fit in progress. */
int g4r_bl_bert4rec_import(g4r_baselines* b, int32_t n_blocks, int32_t n_heads, int32_t max_len, const float* params, int64_t n_params);
/* Every counted event's q in g4r_bl_evaluate's order: the head's output at the mask token of the window of the last
 * min(p, max_len - 1) inputs of items[start .. p] followed by the mask token.  g4r_bl_evaluate of a BERT4Rec handle ranks these q
 * as NARM's, with I = double(E[0 .. n_items)) and bI = double(bO). */
int g4r_bl_bert4rec_encode(g4r_baselines* b, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                           const int32_t* n_history, float* q, int64_t n_q);

#ifdef __cplusplus
}
#endif
#endif
