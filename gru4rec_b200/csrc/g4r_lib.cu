// g4r_lib.cu -- host side of libg4r.so: handle, workspace carving, the session-parallel schedule builder,
// the per-step launch sequence, negative sampling, and the C ABI declared in include/g4r.h.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include "g4r_kernels.cuh"
#include "g4r_misc.cuh"

#define G4R_VERSION 102

static thread_local std::string g_create_error;
struct g4r_handle;
static void eval_release(g4r_handle* h);
static void sessions_release(g4r_handle* h);
static void mg_release(g4r_handle* h);
static void shard_release(g4r_handle* h);
static bool shard_eligible(const g4r_config& c, int n_sm);
static int shard_create(g4r_handle* h);
static bool tc_eligible(const g4r_config& c);
struct TensorInfo;
static int shard_set_tensor(g4r_handle* h, const TensorInfo& t, const float* host);
static int shard_get_tensor(g4r_handle* h, const TensorInfo& t, float* host);
static int mgs_run_window(g4r_handle* h, int64_t n);
static int mgs_plan_window(g4r_handle* h, int64_t n);
static int enqueue_full_step(g4r_handle* h, const int* base, int off);
static int64_t full_launches_per_step(const g4r_handle* h);
static void full_mark_inputs(g4r_handle* h, int64_t n);
static int full_opt_in(g4r_handle* h);
static bool wgmma_tiles(const g4r_config& cfg, int lanes, int n_comp, int n_items);

// sharded: row i of the logical [rows x cols] tensor lives on rank i % R at local row i / R; seg_off = byte offset of element
// (0, 0) inside every rank's peer-mapped segment (g4r_shard.cuh)
struct TensorInfo { float* ptr; int64_t rows, cols, ld; bool sharded = false; size_t seg_off = 0; };

struct g4r_schedule {
  int B = 0, mode = 0;
  int64_t n_steps = 0, n_events = 0;
  std::vector<int32_t> X, Y, slots, M;
  std::vector<uint8_t> F;
  std::vector<int64_t> P;       // recorded on request (mode | 2): index in data_items of every input X (target at P + 1), -1 on unused lanes
  bool has_pos = false;
  int64_t max_len = 1;          // events of the longest session walked (its inputs bound a lane's seen list, g4r_seen.cuh)
  bool hist = false;            // g4r_schedule_build_history: only lanes flagged 4 are counted events (g4r_history.cuh)
};

// window buffers of truncated BPTT (g4r_bptt.cuh): per-step slices [T][B][ld] of the forward saves and gradients, per-layer
// scratch of the backward, and the merged row list of the window
struct BpttDev {
  float *Hold[G4R_MAX_LAYERS], *R[G4R_MAX_LAYERS], *Z[G4R_MAX_LAYERS], *Ah[G4R_MAX_LAYERS], *Ht[G4R_MAX_LAYERS];   // forward saves
  float *In[G4R_MAX_LAYERS];       // layer inputs (layers with an input product)
  float *Dvec[G4R_MAX_LAYERS];     // [T][B][ld3] gate gradients (rows past a step's M stay zero)
  float *Carry[G4R_MAX_LAYERS];    // [B][ldL] gradient wrt the hidden state a step leaves, by physical slot
  float *Dyl[G4R_MAX_LAYERS], *Dh[G4R_MAX_LAYERS], *DHr[G4R_MAX_LAYERS];   // [B][ldL] scratch of the step being differentiated
  float *Dy;                       // [T][B][ldL] dL/dy of the top layer (chunk partials summed)
  float *DSY, *DBY; int* Item;     // [T][NP][ldL], [T][NP], [T][NP]: score-column gradients and their items in plan order
  float *DSx;                      // [T][B][ld_in0] gradients of the gathered input rows (embedding modes)
  int *M, *N, *X, *Slot; uint8_t* F; uint32_t* G;   // per step: lanes, columns, inputs, slots, flags, dropout step
  unsigned long long *keys, *keys2;                  // [T][B + NP] merged row list, unsorted / sorted
};

// full-softmax training (g4r_full.cuh): every step scores the whole catalogue, on fp32 tiles of FS_IT items or on the wgmma
// tiles of the evaluation path (FS_TC_M lanes x FS_TC_N items, K chunks of FS_TC_KC), whose statistics come per FS_TC_N / 2 items
constexpr int FS_IT = 64;          // items per fp32 score tile (== EV_IT of the fp32 evaluation tiles it reuses)
constexpr int FS_TC_M = 128, FS_TC_N = 256, FS_TC_KC = 32;   // == TC_M, TC_N, TC_KC (g4r_eval_tc.cuh)
struct FullDev {
  float* dO;                       // [n_items][Bld] dL/do of the step, item-major (lanes contiguous)
  float* stat;                     // [tiles][B][4] per-(tile, lane) max, sum-exp, target score, has-target
  int tiles, ks, kchunk;           // statistics tiles; K splits of dL/dy = dO . Wy and the items per split (a multiple of GK)
  bool tc;                         // score sweeps on the wgmma 3xTF32 tiles (chosen like the evaluation's, wgmma_tiles)
  int chunks;                      // wgmma: K chunks of L + 1 (the bias column)
  unsigned char *Asplit, *Bsplit;  // wgmma: [hi | lo] blocks of y (per step) and of Wy | By (per step: every row changes)
};
static FullDev full_shape(const g4r_config& c, int n_sm) {
  FullDev f; memset(&f, 0, sizeof(f));
  const int L = c.layers[c.n_layers - 1];
  f.tc = wgmma_tiles(c, c.batch_size, c.n_items, c.n_items);
  f.chunks = (L + 1 + FS_TC_KC - 1) / FS_TC_KC;
  f.tiles = f.tc ? 2 * ((c.n_items + FS_TC_N - 1) / FS_TC_N) : (c.n_items + FS_IT - 1) / FS_IT;
  const int mn = ((c.batch_size + GB - 1) / GB) * ((L + GB - 1) / GB);
  const int slabs = (c.n_items + GK - 1) / GK;
  int ks = std::max(1, std::min(slabs, (2 * n_sm + mn - 1) / mn));
  f.kchunk = ((slabs + ks - 1) / ks) * GK;
  f.ks = (c.n_items + f.kchunk - 1) / f.kchunk;          // no empty splits
  return f;
}

struct g4r_handle {
  g4r_config cfg;
  ModelDev md;
  std::string err;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  char* ws = nullptr; size_t ws_bytes = 0; bool own_ws = false;
  size_t ws_off = 0;
  std::map<std::string, TensorInfo> tensors;
  int Bmax = 0, n_sm = 132;
  int CAP = 0;
  // window staging (pinned host) and device arrays (non-const views of md.w*)
  int *hX = nullptr, *hY = nullptr, *hSlot = nullptr, *hM = nullptr, *hSti = nullptr; uint8_t* hF = nullptr; uint32_t* hG = nullptr;
  float* hCost = nullptr;
  int *dX = nullptr, *dY = nullptr, *dSlot = nullptr, *dM = nullptr, *dSti = nullptr, *dXnext = nullptr; uint8_t *dF = nullptr, *dXflag = nullptr; uint32_t* dG = nullptr;
  int* dStepBase = nullptr;
  // sampling
  float *dP = nullptr, *dLogP0t = nullptr, *dLogP0s = nullptr, *dU = nullptr;
  int* dST = nullptr; int gen_len = 0; int64_t sample_ptr = 0; bool have_store = false; bool have_cdf = false;
  int32_t* dMrgState = nullptr; int n_streams = 0; bool mrg_init = false; int64_t mrg_rstate[6];
  // evaluation hidden state
  float* He[G4R_MAX_LAYERS] = {};
  int* dRankCnt = nullptr; float* dTgt = nullptr;
  // bookkeeping
  uint32_t global_step = 0;
  int win_steps = 0;
  int64_t launches = 0;
  int npow2 = 0;
  // per-phase profiling (g4r_profile_uploaded)
  int slot = -1;
  cudaGraphExec_t graphU = nullptr, graph1 = nullptr; int graph_unroll = 16;
  bool use_graph = true;
  GridBar* dGridBar = nullptr; unsigned long long* dStamp = nullptr; int pk_blocks = 0; size_t pk_smem = 0;
  bool mg_alloc = false; MgDev mgdev; std::vector<MgTensor> mg_tensors;
  void* eval_ctx = nullptr;      // EvalCtx* (g4r_eval.cuh), owned by the handle
  void* sessions = nullptr;      // SessStore* (g4r_sessions.cuh), owned by the handle
  uint64_t wy_version = 0;       // bumped by everything that may change Wy / By (caches derived from them compare it)
  void* mg_host = nullptr;       // MgHost*  (g4r_multi.cuh), owned by the handle
  void* shard = nullptr;         // ShardHost* (g4r_shard.cuh): row-sharded item tables + in-kernel exchange, owned by the handle
  char* shard_ws = nullptr;      // workspace carve-outs of the sharded path (plans, device descriptor, counters, gathered input rows)
  size_t shard_ws_bytes = 0;
  FastSync* dFastSync = nullptr; bool fast_ok = false; bool fastc_ok = false; int fastc_grid = 0; int* hFlags = nullptr; int64_t fast_windows = 0, slow_windows = 0;
  bool prof = false; bool stamp_on = false;
  bool two_pass = false;         // grad_cap: gradients are exported, the global norm is taken, then a second pass applies them scaled
  bool phase_only = false;       // grad_cap / smoothing add phases that only the per-phase launch sequence has
  float* dGscale = nullptr;
  bool tc_ok = false; void* ts_buf = nullptr; unsigned long long* ts_dbg = nullptr; cudaStream_t side = nullptr, side2 = nullptr; cudaEvent_t ts_ev[12] = {};      // tensor-core training step (g4r_tcstep.cuh): TsBuf*
  std::vector<cudaEvent_t> prof_ev; std::vector<int> prof_phase;
  BpttDev bw = {}; void* bptt_cub = nullptr; size_t bptt_cub_bytes = 0; int64_t bptt_windows = 0;   // bptt > 1 (g4r_bptt.cuh)
  FullDev fs = {}; int64_t full_steps = 0;                                                            // full_softmax (g4r_full.cuh)
};

enum { PH_GATHER = 0, PH_F1, PH_F2, PH_SCORE, PH_STATS, PH_LOSSGRAD, PH_B1, PH_B2, PH_B3, PH_DENSE, PH_SPARSE_IN, PH_STATS2, PH_GRADCAP, PH_COUNT };
static const char* kPhaseNames[PH_COUNT] = {"gather_in", "gru_rz", "gru_h", "score", "stats", "lossgrad_update", "gru_bwd_elem", "gru_bwd_dHr", "gru_bwd_din", "dense_update", "sparse_in_update",
                                            "smoothing_stats", "grad_cap_norm_apply"};

// LAUNCH(phase, kernel<<<...>>>(...)): counts the launch and, when profiling, brackets it with CUDA events
#define LAUNCH_ON(strm, ph, ...) do { \
    cudaEvent_t e0_ = nullptr, e1_ = nullptr; \
    if (h->prof) { cudaEventCreate(&e0_); cudaEventCreate(&e1_); cudaEventRecord(e0_, (strm)); } \
    __VA_ARGS__; \
    h->launches++; \
    if (h->prof) { cudaEventRecord(e1_, (strm)); h->prof_ev.push_back(e0_); h->prof_ev.push_back(e1_); h->prof_phase.push_back(ph); } \
  } while (0)
#define LAUNCH(ph, ...) LAUNCH_ON(h->stream, ph, __VA_ARGS__)

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return G4R_ERR_CUDA; } } while (0)
#define FAIL(code, msg) do { h->err = (msg); return (code); } while (0)

static inline int round4(int x) { return (x + 3) & ~3; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------
// workspace layout: computed identically in a dry run (bytes) and for real (carving)
// ------------------------------------------------------------------------------------------------
struct Carver {
  char* base; size_t off; bool dry;
  template <class T> T* take(size_t n) {
    off = align_up(off, 256);
    T* p = dry ? nullptr : reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    return p;
  }
};

static int validate_config(const g4r_config& c, std::string& err) {
  if (c.n_items <= 0 || c.n_layers <= 0 || c.n_layers > G4R_MAX_LAYERS || c.batch_size <= 0) { err = "invalid sizes"; return G4R_ERR_INVALID; }
  for (int i = 0; i < c.n_layers; i++) if (c.layers[i] <= 0) { err = "invalid layer width"; return G4R_ERR_INVALID; }
  if (c.adapt < G4R_ADAPT_NONE || c.adapt > G4R_ADAPT_ADAM) { err = "adapt: unknown optimizer"; return G4R_ERR_INVALID; }
  if (c.adapt > G4R_ADAPT_ADAGRAD && c.constrained_embedding) {
    // the reference's duplicate-accurate state update couples the input and the output occurrences of an item in one scatter
    err = "adapt = rmsprop / adadelta / adam with constrained_embedding is not implemented on the device path"; return G4R_ERR_INVALID;
  }
  if (c.grad_cap < 0.f) { err = "grad_cap < 0"; return G4R_ERR_INVALID; }
  if ((c.adapt > G4R_ADAPT_ADAGRAD || c.grad_cap > 0.f || c.smoothing != 0.f) && c.world_size > 1) {
    err = "adapt other than adagrad, grad_cap and smoothing are single-GPU options"; return G4R_ERR_INVALID;
  }
  if (c.hidden_act < G4R_ACT_LINEAR || c.hidden_act > G4R_ACT_SELU) { err = "hidden_act unsupported"; return G4R_ERR_INVALID; }
  const bool elem = c.final_act >= G4R_ACT_LINEAR && c.final_act <= G4R_ACT_SELU;
  bool ok = false;
  if (c.loss == G4R_LOSS_XE && c.final_act == G4R_ACT_SOFTMAX) ok = true;
  if (c.loss == G4R_LOSS_XE_LOGIT && c.final_act == G4R_ACT_SOFTMAX_LOGIT) ok = true;
  if ((c.loss == G4R_LOSS_BPR_MAX || c.loss == G4R_LOSS_TOP1_MAX || c.loss == G4R_LOSS_BPR || c.loss == G4R_LOSS_TOP1) && elem) ok = true;
  if (!ok) { err = "loss / final_act combination not implemented on the device path"; return G4R_ERR_INVALID; }
  if (c.smoothing < 0.f) { err = "smoothing < 0"; return G4R_ERR_INVALID; }
  if (c.constrained_embedding && c.embedding) { /* reference: constrained wins (gru4rec.py:272) */ }
  if (c.n_sample < 0) { err = "n_sample < 0"; return G4R_ERR_INVALID; }
  if (c.bptt < 0 || c.bptt > 64) { err = "bptt must be in [1, 64]"; return G4R_ERR_INVALID; }
  if (c.bptt > 1 && c.world_size > 1) { err = "bptt > 1 is a single-GPU option"; return G4R_ERR_INVALID; }
  if (c.full_softmax != 0 && c.full_softmax != 1) { err = "full_softmax must be 0 or 1"; return G4R_ERR_INVALID; }
  if (c.full_softmax) {
    if (c.loss != G4R_LOSS_XE && c.loss != G4R_LOSS_XE_LOGIT) { err = "full_softmax: only loss cross-entropy / softmax and xe_logit / softmax_logit are implemented"; return G4R_ERR_INVALID; }
    if (c.smoothing > 0.f) { err = "full_softmax: label smoothing is not implemented"; return G4R_ERR_INVALID; }
    if (c.grad_cap > 0.f) { err = "full_softmax: grad_cap is not implemented"; return G4R_ERR_INVALID; }
    if (c.bptt > 1) { err = "full_softmax: bptt > 1 is not implemented"; return G4R_ERR_INVALID; }
    if (c.world_size > 1) { err = "full_softmax is a single-GPU option"; return G4R_ERR_INVALID; }
  }
  return G4R_OK;
}

static int model_mode(const g4r_config& c) { return c.constrained_embedding ? 2 : (c.embedding > 0 ? 1 : 0); }

static int next_pow2(int x) { int p = 1; while (p < x) p <<= 1; return p; }

static void layout(const g4r_config& c, Carver& cv, g4r_handle* h, int n_sm) {
  const bool shard = shard_eligible(c, n_sm);     // multi-GPU with row-sharded item tables: they live in the peer-mapped segment
  const int mode = model_mode(c);
  const int nl = c.n_layers;
  const int B = c.batch_size;
  const int Be = c.eval_batch_size > 0 ? c.eval_batch_size : B;
  const int Bmax = std::max(B, Be);
  const int Llast = c.layers[nl - 1], ldL = round4(Llast);
  const bool mom = c.momentum > 0.f;
  const bool ada = c.adapt != G4R_ADAPT_NONE;            // at least one adaptive state array ("acc")
  const int nacc = opt_states(c.adapt);                  // acc | acc, upd | acc, meang, countt -- stacked behind `*.acc`
  const bool full = c.full_softmax != 0;                 // the catalogue is the score column list: no sample store (DESIGN §3n)
  const int gen_len = (!full && c.n_sample > 0 && c.sample_store > 0) ? c.sample_store / c.n_sample : 0;
  const bool store = gen_len > 1;
  const int S = store ? c.n_sample : 0;
  const int NP = round4(B + S);
  const int NCH = std::max(1, std::min(shard ? n_sm - MGS_GRU_CTAS : n_sm, (NP + 3) / 4));   // sharded: the GRU CTAs own no columns
  const int R = c.world_size > 1 ? c.world_size : 1;
  const int CAP = std::max(c.max_resident_steps > 0 ? c.max_resident_steps : 2048, R > 1 ? MG_CAP : 1);
  ModelDev md; memset(&md, 0, sizeof(md));
  md.n_items = c.n_items; md.n_layers = nl; md.B = B; md.Bld = round4(Bmax); md.S = S; md.mode = mode; md.L = Llast; md.ldL = ldL;
  md.NP = NP; md.NCH = NCH; md.CAP = CAP; md.S_cfg = c.n_sample; md.shardR = shard ? R : 0;
  md.loss = c.loss; md.fact = {c.final_act, c.final_act_p1, c.final_act_p2}; md.hact = {c.hidden_act, c.hidden_act_p1, c.hidden_act_p2};
  md.p_drop_h = c.dropout_p_hidden; md.p_drop_e = c.dropout_p_embed; md.lr = c.learning_rate; md.mom = c.momentum; md.lmbd = c.lmbd;
  md.bpreg = c.bpreg; md.logq = full ? 0.f : c.logq; md.alpha = c.sample_alpha; md.adapt = c.adapt;   // logq corrects a sampled softmax only
  md.ap1 = c.adapt_p1; md.ap1c = c.adapt_p1c; md.ap2 = c.adapt_p2; md.ap2c = c.adapt_p2c; md.grad_cap = c.grad_cap;
  md.smoothing = (c.loss == G4R_LOSS_XE || c.loss == G4R_LOSS_XE_LOGIT) ? c.smoothing : 0.f;    // the other losses ignore it (gru4rec.py:237-248)
  md.drop_seed = c.dropout_seed + (c.world_size > 1 ? (uint32_t)c.rank * 0x9E3779B1u : 0u);   // multi-GPU: independent masks per rank
  md.in0_dim = mode == 2 ? Llast : (mode == 1 ? c.embedding : 0);
  md.ld_in0 = round4(md.in0_dim);
  auto reg = [&](const std::string& name, float* p, int64_t rows, int64_t cols, int64_t ld) { if (!cv.dry) h->tensors[name] = TensorInfo{p, rows, cols, ld}; };
  auto table3 = [&](const std::string& name, int64_t rows, int64_t cols, float** p, float** a, float** v, int64_t ld_override = 0) {
    const int64_t ld = ld_override > 0 ? ld_override : round4((int)cols);
    *p = cv.take<float>((size_t)rows * ld); reg(name, *p, rows, cols, ld);
    *a = ada ? cv.take<float>((size_t)rows * ld * nacc) : nullptr; if (ada) reg(name + ".acc", *a, rows, cols, ld);
    if (nacc > 1) reg(name + (c.adapt == G4R_ADAPT_ADAM ? ".meang" : ".upd"), *a + (size_t)rows * ld, rows, cols, ld);
    if (nacc > 2) reg(name + ".countt", *a + 2 * (size_t)rows * ld, rows, cols, ld);
    *v = mom ? cv.take<float>((size_t)rows * ld) : nullptr; if (mom) reg(name + ".vel", *v, rows, cols, ld);
  };
  // item tables
  if (!shard) {
    table3("Wy", c.n_items, Llast, &md.Wy, &md.Wy_acc, &md.Wy_vel);
    table3("By", c.n_items, 1, &md.By, &md.By_acc, &md.By_vel, 1);   // dense [I] vector
  }
  if (mode == 1) table3("E", c.n_items, c.embedding, &md.E, &md.E_acc, &md.E_vel);
  for (int i = 0; i < nl; i++) {
    LayerDev& ly = md.layer[i];
    const int L = c.layers[i];
    ly.L = L; ly.ldL = round4(L); ly.ld2 = round4(2 * L); ly.ld3 = round4(3 * L);
    int in_rows;
    if (i == 0) { in_rows = mode == 0 ? c.n_items : md.in0_dim; ly.in_dim = mode == 0 ? 0 : md.in0_dim; ly.ld_in = md.ld_in0; }
    else { in_rows = c.layers[i - 1]; ly.in_dim = c.layers[i - 1]; ly.ld_in = round4(c.layers[i - 1]); }
    const std::string si = std::to_string(i);
    if (!(shard && i == 0)) table3("Wx" + si, in_rows, 3 * L, &ly.Wx, &ly.Wx_acc, &ly.Wx_vel);
    table3("Wh" + si, L, L, &ly.Wh, &ly.Wh_acc, &ly.Wh_vel);
    table3("Wrz" + si, L, 2 * L, &ly.Wrz, &ly.Wrz_acc, &ly.Wrz_vel);
    table3("Bh" + si, 1, 3 * L, &ly.Bh, &ly.Bh_acc, &ly.Bh_vel);
    ly.H = cv.take<float>((size_t)B * ly.ldL); reg("H" + si, ly.H, B, L, ly.ldL);
    float* he = cv.take<float>((size_t)Be * ly.ldL); if (!cv.dry) h->He[i] = he;
    reg("He" + si, he, Be, L, ly.ldL);
    ly.Hold = cv.take<float>((size_t)Bmax * ly.ldL); ly.r = cv.take<float>((size_t)Bmax * ly.ldL); ly.z = cv.take<float>((size_t)Bmax * ly.ldL);
    ly.ah = cv.take<float>((size_t)Bmax * ly.ldL); ly.ht = cv.take<float>((size_t)Bmax * ly.ldL); ly.y = cv.take<float>((size_t)Bmax * ly.ldL);
    ly.dvec = cv.take<float>((size_t)Bmax * ly.ld3); ly.dy = cv.take<float>((size_t)Bmax * ly.ldL); ly.Hr = cv.take<float>((size_t)Bmax * ly.ldL);
    reg("y" + si, ly.y, Bmax, L, ly.ldL); reg("dvec" + si, ly.dvec, Bmax, 3 * L, ly.ld3);
  }
  if (mode != 0) {
    md.Sx = cv.take<float>((size_t)Bmax * md.ld_in0); md.in0 = cv.take<float>((size_t)Bmax * md.ld_in0); md.dSx = cv.take<float>((size_t)Bmax * md.ld_in0);
    if (mode == 2) { md.snapAcc = cv.take<float>((size_t)Bmax * md.ld_in0); md.snapVel = cv.take<float>((size_t)Bmax * md.ld_in0); }
    reg("dSx", md.dSx, Bmax, md.in0_dim, md.ld_in0);
  }
  for (int i = 0; i < nl; i++) md.layer[i].in = (i == 0) ? md.in0 : md.layer[i - 1].y;
  // step scratch
  md.O = cv.take<float>((size_t)NP * md.Bld);
  md.DSY = cv.take<float>((size_t)NP * ldL); md.DBY = cv.take<float>((size_t)NP);
  const FullDev fsh = full ? full_shape(c, n_sm) : FullDev{};
  md.part = cv.take<float>((size_t)std::max(NCH, fsh.ks) * B * ldL);    // full_softmax: the K-split partials of dL/dy
  md.stat = cv.take<float>((size_t)NCH * B * G4R_NSTAT);
  md.RS = cv.take<float>((size_t)Bmax * G4R_NSTAT);
  md.stat2 = md.smoothing > 0.f ? cv.take<float>((size_t)NCH * B * 2) : nullptr;
  float* gsc = c.grad_cap > 0.f ? cv.take<float>(8) : nullptr;
  md.gscale = gsc;
  md.cost = cv.take<float>((size_t)CAP);
  md.nanflag = cv.take<int>(4);
  reg("O", md.O, NP, Bmax, md.Bld); reg("DSY", md.DSY, NP, Llast, ldL);
  // schedule window + plans
  int* dX = cv.take<int>((size_t)CAP * B); int* dY = cv.take<int>((size_t)CAP * B); int* dSlot = cv.take<int>((size_t)CAP * B);
  int* dXnext = cv.take<int>((size_t)CAP * B);
  uint8_t* dF = cv.take<uint8_t>((size_t)CAP * B); uint8_t* dXflag = cv.take<uint8_t>((size_t)CAP * B);
  int* dM = cv.take<int>(CAP); int* dSti = cv.take<int>(CAP); uint32_t* dG = cv.take<uint32_t>(CAP);
  md.pItem = cv.take<int>((size_t)CAP * NP); md.pPos = cv.take<int>((size_t)CAP * NP);
  md.pTcol = cv.take<int>((size_t)CAP * B); md.pCbeg = cv.take<int>((size_t)CAP * (NCH + 1));
  md.pKey = shard ? cv.take<int>((size_t)CAP * NP) : nullptr;
  int* dStepBase = cv.take<int>(4);
  GridBar* dGridBar = cv.take<GridBar>(1);
  FastSync* dFastSync = cv.take<FastSync>(1);
  unsigned long long* dStamp = cv.take<unsigned long long>((size_t)CAP * 16);
  // sampling
  float* dP = cv.take<float>(c.n_items); float* dL0t = cv.take<float>(c.n_items); float* dL0s = cv.take<float>(c.n_items);
  int* dST = store ? cv.take<int>((size_t)gen_len * c.n_sample) : nullptr;
  float* dU = store ? cv.take<float>((size_t)gen_len * c.n_sample) : nullptr;
  int32_t* dMrg = cv.take<int32_t>((size_t)15360 * 6);
  // multi-GPU: dense-gradient twins (one flat all-reduce buffer) and the gathered / merged per-window state
  MgDev mgd; memset(&mgd, 0, sizeof(mgd));
  std::vector<MgTensor> mgt;
  const bool twins = R > 1 || c.grad_cap > 0.f || c.bptt > 1;      // dense gradients are exported (all-reduced / norm-capped / summed over a window) before they are applied
  if (twins) {
    size_t cnt = 0;
    for (int i = 0; i < nl; i++) {
      const LayerDev& ly = md.layer[i];
      if (ly.in_dim > 0) cnt += (size_t)ly.in_dim * ly.ld3;
      cnt += (size_t)ly.L * ly.ldL + (size_t)ly.L * ly.ld2 + ly.ld3;
    }
    float* gf = cv.take<float>(cnt);
    size_t off = 0;
    for (int i = 0; i < nl; i++) {
      LayerDev& ly = md.layer[i];
      if (ly.in_dim > 0) { ly.Wx_g = gf ? gf + off : nullptr; mgt.push_back(MgTensor{ly.Wx, ly.Wx_acc, ly.Wx_vel, off, ly.in_dim * ly.ld3}); off += (size_t)ly.in_dim * ly.ld3; }
      ly.Wh_g = gf ? gf + off : nullptr; mgt.push_back(MgTensor{ly.Wh, ly.Wh_acc, ly.Wh_vel, off, ly.L * ly.ldL}); off += (size_t)ly.L * ly.ldL;
      ly.Wrz_g = gf ? gf + off : nullptr; mgt.push_back(MgTensor{ly.Wrz, ly.Wrz_acc, ly.Wrz_vel, off, ly.L * ly.ld2}); off += (size_t)ly.L * ly.ld2;
      ly.Bh_g = gf ? gf + off : nullptr; mgt.push_back(MgTensor{ly.Bh, ly.Bh_acc, ly.Bh_vel, off, ly.ld3}); off += ly.ld3;
    }
    mgd.R = R; mgd.rank = c.rank; mgd.gradFlat = gf; mgd.gradCount = cnt;
  }
  if (R > 1) {
    mgd.gItem = cv.take<int>((size_t)R * MG_CAP * NP); mgd.gPos = nullptr;
    mgd.gM = cv.take<int>((size_t)R * MG_CAP); mgd.gX = cv.take<int>((size_t)R * MG_CAP * B);
    mgd.mEnt = cv.take<int>((size_t)MG_CAP * R * NP); mgd.mItem = cv.take<int>((size_t)MG_CAP * R * NP);
    mgd.mCbeg = cv.take<int>((size_t)MG_CAP * (n_sm + 1)); mgd.mTot = cv.take<int>(MG_CAP);
    mgd.xEnt = cv.take<int>((size_t)MG_CAP * R * B); mgd.xItem = cv.take<int>((size_t)MG_CAP * R * B); mgd.xTot = cv.take<int>(MG_CAP);
    if (!shard) {
      const int in_ld = mode == 0 ? md.layer[0].ld3 : md.ld_in0;
      mgd.DSYall = cv.take<float>((size_t)R * NP * ldL); mgd.DBYall = cv.take<float>((size_t)R * NP); mgd.INall = cv.take<float>((size_t)R * B * in_ld);
    }
  }
  // sharded path: owner bounds of the gathered lists, device descriptor, counters, gathered input rows
  char* shard_ws = nullptr; size_t shard_ws_bytes = 0;
  if (shard) {
    shard_ws_bytes = (size_t)2 * MG_CAP * R * sizeof(int) + 4096 + (size_t)B * md.layer[0].ld3 * sizeof(float) + 1024;
    shard_ws = cv.take<char>(shard_ws_bytes);
  }
  // tensor-core training step: hi|lo operand blocks (g4r_tcstep.cuh)
  TsBuf tsb; memset(&tsb, 0, sizeof(tsb));
  const bool tc = tc_eligible(c);
  if (tc) {
    auto r32 = [](int x) { return (x + 31) / 32 * 32; };
    auto r128 = [](int x) { return (x + 127) / 128 * 128; };
    const int L = Llast;
    tsb.Mpad = r128(B); tsb.Lk1 = r32(L); tsb.Lk2 = r32(2 * L); tsb.Lk3 = r32(3 * L); tsb.Nk = r128(NP); tsb.Bk = r32(B);
    tsb.ldO = tsb.Nk;
    auto op = [&](int rows, int K) { return cv.take<unsigned char>((size_t)((rows + 255) / 256 * 256) * K * 8); };   // hi + lo: 8 bytes per element; rows padded to a 256-wide N tile
    tsb.Lp = (L + 255) / 256 * 256;
    tsb.A1 = op(B, tsb.Lk2); tsb.A2 = op(B, tsb.Lk2); tsb.A3 = op(B, tsb.Lk1); tsb.A4 = op(NP, tsb.Bk); tsb.A5 = op(B, tsb.Nk);
    tsb.A6 = op(B, tsb.Lk1); tsb.A7 = op(B, tsb.Lk3); tsb.A8 = op(3 * L, tsb.Bk);
    tsb.W1 = op(2 * L, tsb.Lk2); tsb.W2 = op(L, tsb.Lk2); tsb.W3 = op(L, tsb.Lk1); tsb.W4 = op(L, tsb.Lk3);
    tsb.B3 = op(NP, tsb.Lk1); tsb.B4 = op(L, tsb.Bk); tsb.B5 = op(L, tsb.Nk); tsb.B8a = op(2 * tsb.Lp, tsb.Bk); tsb.B8b = op(L, tsb.Bk);
    size_t pf = 0;          // the main-stream products run one after the other: one buffer of the largest size (any cluster cap)
    for (const TsShape& t : {ts_shape(B, 2 * L, tsb.Lk2 / 32, n_sm, 16), ts_shape(B, L, tsb.Lk2 / 32, n_sm, 16), ts_shape(B, NP, tsb.Lk1 / 32, n_sm, 16),
                             ts_shape(B, L, tsb.Nk / 32, n_sm, 16), ts_shape(B, L, tsb.Lk1 / 32, n_sm, 16), ts_shape(B, L, tsb.Lk3 / 32, n_sm, 16)}) pf = std::max(pf, t.p_floats);
    tsb.P = cv.take<float>(pf);
    tsb.P1 = cv.take<float>(ts_shape(tsb.Nk, L, tsb.Bk / 32, n_sm, 16).p_floats);
    tsb.Pa = cv.take<float>(ts_shape(3 * L, 2 * tsb.Lp, tsb.Bk / 32, n_sm, 0).p_floats);
    tsb.Pb = cv.take<float>(ts_shape(3 * L, L, tsb.Bk / 32, n_sm, 0).p_floats);
    tsb.O = cv.take<float>((size_t)tsb.Mpad * tsb.ldO); tsb.bias = cv.take<float>(tsb.Nk);
  }
  // truncated BPTT: window slices
  BpttDev bw; memset(&bw, 0, sizeof(bw));
  if (c.bptt > 1) {
    const size_t TB = (size_t)c.bptt * B;
    for (int i = 0; i < nl; i++) {
      const LayerDev& ly = md.layer[i];
      bw.Hold[i] = cv.take<float>(TB * ly.ldL); bw.R[i] = cv.take<float>(TB * ly.ldL); bw.Z[i] = cv.take<float>(TB * ly.ldL);
      bw.Ah[i] = cv.take<float>(TB * ly.ldL); bw.Ht[i] = cv.take<float>(TB * ly.ldL);
      bw.In[i] = ly.in_dim > 0 ? cv.take<float>(TB * ly.ld_in) : nullptr;
      bw.Dvec[i] = cv.take<float>(TB * ly.ld3);
      bw.Carry[i] = cv.take<float>((size_t)B * ly.ldL); bw.Dyl[i] = cv.take<float>((size_t)B * ly.ldL);
      bw.Dh[i] = cv.take<float>((size_t)B * ly.ldL); bw.DHr[i] = cv.take<float>((size_t)B * ly.ldL);
    }
    bw.Dy = cv.take<float>(TB * ldL);
    bw.DSY = cv.take<float>((size_t)c.bptt * NP * ldL); bw.DBY = cv.take<float>((size_t)c.bptt * NP); bw.Item = cv.take<int>((size_t)c.bptt * NP);
    bw.DSx = mode != 0 ? cv.take<float>(TB * md.ld_in0) : nullptr;
    bw.M = cv.take<int>(c.bptt); bw.N = cv.take<int>(c.bptt); bw.X = cv.take<int>(TB); bw.Slot = cv.take<int>(TB);
    bw.F = cv.take<uint8_t>(TB); bw.G = cv.take<uint32_t>(c.bptt);
    bw.keys = cv.take<unsigned long long>((size_t)c.bptt * (B + NP)); bw.keys2 = cv.take<unsigned long long>((size_t)c.bptt * (B + NP));
  }
  // full-softmax training: dL/do of the step over the catalogue, per-tile row statistics
  FullDev fs = fsh;
  if (full) {
    fs.dO = cv.take<float>((size_t)c.n_items * md.Bld); fs.stat = cv.take<float>((size_t)fsh.tiles * B * 4);
    if (fsh.tc) {
      fs.Asplit = cv.take<unsigned char>((size_t)((B + FS_TC_M - 1) / FS_TC_M) * fsh.chunks * 2 * FS_TC_M * FS_TC_KC * 4);
      fs.Bsplit = cv.take<unsigned char>((size_t)((c.n_items + FS_TC_N - 1) / FS_TC_N) * fsh.chunks * 2 * FS_TC_N * FS_TC_KC * 4);
    }
  }
  // evaluation
  int* dRank = cv.take<int>((size_t)Be * 4); float* dTgt = cv.take<float>((size_t)Be * 3);   // target scores | lower | upper pre-activation thresholds (tensor-core ranking)
  if (!cv.dry) {
    md.wX = dX; md.wY = dY; md.wSlot = dSlot; md.wM = dM; md.wSti = dSti; md.wXnext = dXnext; md.wF = dF; md.wXflag = dXflag; md.wG = dG;
    md.ST = dST; md.logP0t = dL0t; md.logP0s = dL0s;
    h->md = md; h->Bmax = Bmax; h->CAP = CAP; h->mg_alloc = R > 1; h->mgdev = mgd; h->mg_tensors = mgt; h->gen_len = store ? gen_len : 0;
    h->dX = dX; h->dY = dY; h->dSlot = dSlot; h->dM = dM; h->dSti = dSti; h->dXnext = dXnext; h->dF = dF; h->dXflag = dXflag; h->dG = dG;
    h->dGridBar = dGridBar; h->dStamp = dStamp; h->dFastSync = dFastSync;
    h->dStepBase = dStepBase; h->dP = dP; h->dLogP0t = dL0t; h->dLogP0s = dL0s; h->dST = dST; h->dU = dU; h->dMrgState = dMrg;
    h->dRankCnt = dRank; h->dTgt = dTgt;
    h->npow2 = next_pow2(B + S);
    h->shard_ws = shard_ws; h->shard_ws_bytes = shard_ws_bytes;
    h->tc_ok = tc;
    if (tc) { if (!h->ts_buf) h->ts_buf = new TsBuf(); *static_cast<TsBuf*>(h->ts_buf) = tsb; }
    h->bw = bw; h->fs = fs;
    h->dGscale = gsc; h->two_pass = c.grad_cap > 0.f; h->phase_only = c.grad_cap > 0.f || md.smoothing > 0.f || full;
  }
}

// ------------------------------------------------------------------------------------------------
// kernels: one per phase (thin wrappers around the phase functions)
// ------------------------------------------------------------------------------------------------
// Model descriptors live in constant memory (one slot per handle / per scoring context) so that kernel launches
// carry a few scalars instead of a 2 KB by-value struct (the by-value launch cost 16 us of CPU time each).
#define G4R_MAX_SLOTS 24
__constant__ ModelDev c_models[G4R_MAX_SLOTS];
static bool g_slot_used[G4R_MAX_SLOTS] = {};
static std::mutex g_slot_mutex;      // handles are single-threaded, but several handles may live in several threads
static int slot_alloc() { std::lock_guard<std::mutex> lk(g_slot_mutex); for (int i = 0; i < G4R_MAX_SLOTS; i++) if (!g_slot_used[i]) { g_slot_used[i] = true; return i; } return -1; }
static void slot_free(int i) { std::lock_guard<std::mutex> lk(g_slot_mutex); if (i >= 0 && i < G4R_MAX_SLOTS) g_slot_used[i] = false; }
static cudaError_t slot_upload(int slot, const ModelDev& md, cudaStream_t st) {
  return cudaMemcpyToSymbolAsync(c_models, &md, sizeof(ModelDev), (size_t)slot * sizeof(ModelDev), cudaMemcpyHostToDevice, st);
}
#define MD (c_models[slot])
#define STEP_IDX (base ? (*base + off) : off)
__global__ void __launch_bounds__(256) k_gather_in(int slot, const int* base, int off, int train) { phase_gather_in(MD, STEP_IDX, train != 0, blockIdx.x, gridDim.x); }
__global__ void __launch_bounds__(GEMM_THREADS) k_f1(int slot, const int* base, int off, int li, float* Hsrc) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  phase_f1(MD, li, STEP_IDX, Hsrc, blockIdx.x, sA, sB);
}
__global__ void __launch_bounds__(GEMM_THREADS) k_f2(int slot, const int* base, int off, int li, float* Hsrc, int train) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  phase_f2(MD, li, STEP_IDX, Hsrc, train != 0, blockIdx.x, sA, sB);
}
__global__ void __launch_bounds__(SC_THREADS) k_score(int slot, const int* base, int off) {
  extern __shared__ __align__(16) float smem[];
  phase_score(MD, STEP_IDX, blockIdx.x, smem);
}
__global__ void __launch_bounds__(256) k_stats(int slot, const int* base, int off) {
  extern __shared__ __align__(16) float smem[];
  phase_stats(MD, STEP_IDX, blockIdx.x, gridDim.x, smem);
}
__global__ void __launch_bounds__(SC_THREADS) k_lossgrad(int slot, const int* base, int off) {
  extern __shared__ __align__(16) float smem[];
  phase_lossgrad(MD, STEP_IDX, blockIdx.x, smem);
}
__global__ void __launch_bounds__(256) k_b1(int slot, const int* base, int off, int li, int nch) { phase_b1(MD, li, STEP_IDX, blockIdx.x, gridDim.x, nch); }
__global__ void __launch_bounds__(GEMM_THREADS) k_b2(int slot, const int* base, int off, int li) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  phase_b2(MD, li, STEP_IDX, blockIdx.x, sA, sB);
}
__global__ void __launch_bounds__(GEMM_THREADS) k_b3(int slot, const int* base, int off, int li) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  phase_b3(MD, li, STEP_IDX, blockIdx.x, sA, sB);
}
__global__ void __launch_bounds__(GEMM_THREADS) k_dense(int slot, const int* base, int off, int li) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  phase_dense(MD, li, STEP_IDX, blockIdx.x, sA, sB);
}
__global__ void __launch_bounds__(128) k_sparse_in(int slot, const int* base, int off, int apply_pass) { phase_sparse_in(MD, STEP_IDX, blockIdx.x, apply_pass != 0); }
__global__ void __launch_bounds__(256) k_stats2a(int slot, const int* base, int off) { phase_stats2a(MD, STEP_IDX, blockIdx.x); }
__global__ void __launch_bounds__(256) k_stats2b(int slot, const int* base, int off) {
  __shared__ float smem[64];
  phase_stats2b(MD, STEP_IDX, blockIdx.x, gridDim.x, smem);
}
__global__ void __launch_bounds__(1024) k_gradnorm(int slot, const int* base, int off, const float* dense_flat, size_t dense_count, float* gscale) {
  __shared__ float smem[32];
  phase_gradnorm(MD, STEP_IDX, dense_flat, dense_count, gscale, smem);
}
__global__ void __launch_bounds__(SC_THREADS) k_apply_rows(int slot, const int* base, int off) { phase_apply_rows(MD, STEP_IDX, blockIdx.x); }
__global__ void __launch_bounds__(256) k_apply_dense(int slot, float* p, float* acc, float* vel, const float* g, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dense_update(MD, p + i, acc ? acc + i : nullptr, vel ? vel + i : nullptr, g[i], (size_t)n);
}
__global__ void k_advance(int* base, int n) { if (threadIdx.x == 0 && blockIdx.x == 0) *base += n; }

#include "g4r_persistent.cuh"
#include "g4r_fast.cuh"

// The shapes k_fast_t<false> (step_mode 2) takes, from the configuration alone: no-embedding mode, one GRU layer with
// L <= 120, batch <= 32, SGD / Adagrad (+momentum), none of the phases only the per-phase sequence has.  Its ldL / 4 GRU
// CTAs own no score columns, so this decides the chunk geometry before the workspace is laid out: such a handle has
// n_sm - ldL / 4 chunks (chunk c on CTA ldL / 4 + c) in every window, whichever kernel runs it, and needs at least one
// column CTA per lane (column CTA b combines the row statistics of lane b).
static bool fast_shape(const g4r_config& c, int n_sm) {
  const int L = c.layers[0], ldL = round4(L);
  const bool smoothing = (c.loss == G4R_LOSS_XE || c.loss == G4R_LOSS_XE_LOGIT) && c.smoothing > 0.f;
  return c.step_mode == 2 && c.bptt <= 1 && c.adapt <= G4R_ADAPT_ADAGRAD && !(c.grad_cap > 0.f) && !smoothing && model_mode(c) == 0 && c.n_layers == 1 &&
         ldL <= 128 && c.batch_size <= FK_B && 2 * L <= FK_W1 * FK_G && L <= FK_W2 * FK_G && n_sm >= FK_G + 1 &&
         n_sm - ldL / 4 >= c.batch_size && !tc_eligible(c) && !shard_eligible(c, n_sm);
}

// ---- cluster launch of the role-specialised kernel (step_mode 3) ----
constexpr int FC_CLUSTER = 8;      // portable cluster size; cRed in FastSmemC is sized for <= 8 ranks
static cudaError_t fastc_config(cudaLaunchConfig_t& lc, cudaLaunchAttribute* attrs, int n_attr_coop, int grid, cudaStream_t st) {
  lc = cudaLaunchConfig_t{};
  lc.gridDim = dim3(grid); lc.blockDim = dim3(FK_THREADS); lc.dynamicSmemBytes = sizeof(FastSmemC); lc.stream = st;
  attrs[0].id = cudaLaunchAttributeClusterDimension;
  attrs[0].val.clusterDim.x = FC_CLUSTER; attrs[0].val.clusterDim.y = 1; attrs[0].val.clusterDim.z = 1;
  attrs[1].id = cudaLaunchAttributeCooperative; attrs[1].val.cooperative = 1;
  lc.attrs = attrs; lc.numAttrs = 1 + n_attr_coop;
  return cudaSuccess;
}
// largest grid (multiple of the cluster size, at most one CTA per SM) whose clusters are all co-resident; 0 if unsupported
static int fastc_max_grid(int n_sm) {
  if (cudaFuncSetAttribute(k_fast_t<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastSmemC)) != cudaSuccess) { cudaGetLastError(); return 0; }
  cudaLaunchConfig_t lc; cudaLaunchAttribute attrs[2];
  fastc_config(lc, attrs, 0, (n_sm / FC_CLUSTER) * FC_CLUSTER, nullptr);
  int ncl = 0;
  if (cudaOccupancyMaxActiveClusters(&ncl, k_fast_t<true>, &lc) != cudaSuccess) { cudaGetLastError(); return 0; }
  return std::min(ncl, n_sm / FC_CLUSTER) * FC_CLUSTER;
}
static cudaError_t fastc_launch(int grid, cudaStream_t st, void** args) {
  static int coop_ok = 1;          // cooperative + cluster attributes together; dropped if the runtime rejects the pair
  cudaLaunchConfig_t lc; cudaLaunchAttribute attrs[2];
  if (coop_ok) {
    fastc_config(lc, attrs, 1, grid, st);
    cudaError_t e = cudaLaunchKernelExC(&lc, (const void*)k_fast_t<true>, args);
    if (e == cudaSuccess) return e;
    cudaGetLastError();
    coop_ok = 0;
  }
  // co-residency is still guaranteed: grid <= cudaOccupancyMaxActiveClusters * cluster size, one CTA per SM
  fastc_config(lc, attrs, 0, grid, st);
  return cudaLaunchKernelExC(&lc, (const void*)k_fast_t<true>, args);
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is per-function, process-global state: several handles (models of different shapes)
// may be alive at once, so the limit of a kernel is only ever raised (a smaller request of a later handle must not lower it)
static std::mutex g_smem_mutex;
static std::map<const void*, int> g_smem_limit;
static cudaError_t raise_smem_limit(const void* func, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_smem_mutex);
  int& cur = g_smem_limit[func];
  if ((int)bytes <= cur) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) cur = (int)bytes;
  return e;
}

static int tiles2(int cols, int rows) { return ((cols + GB - 1) / GB) * ((rows + GB - 1) / GB); }

#include "g4r_seen.cuh"
#include "g4r_eval_tc.cuh"
#include "g4r_tcstep.cuh"
// The shapes the tensor-core step takes: constrained embedding, one layer, batch <= 256, SGD / Adagrad (+momentum); chosen
// automatically for wide layers (L >= 160), or for any such model with step_mode 4.
static bool tc_eligible(const g4r_config& c) {
  if (!c.constrained_embedding || c.n_layers != 1 || c.batch_size > 256 || (c.layers[0] & 3)) return false;
  if (c.adapt > G4R_ADAPT_ADAGRAD || c.grad_cap > 0.f || c.smoothing != 0.f || c.world_size > 1 || c.bptt > 1 || c.full_softmax) return false;
  return c.step_mode == 4 || (c.step_mode >= 1 && c.step_mode <= 3 && c.layers[0] >= 160);
}
// G4R_TS_STAMP=1: per-product phase timeline of the last step (median / max over the CTAs, microseconds after the first CTA's entry)
static void ts_print_stamps(g4r_handle* h) {
  std::vector<unsigned long long> d(9 * 512 * 16);
  cudaDeviceSynchronize();
  cudaMemcpy(d.data(), h->ts_dbg, d.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
  for (int e = 0; e < 9; e++) {
    unsigned long long t0 = ~0ull; int n = 0;
    for (int c = 0; c < 512; c++) { const unsigned long long v = d[((size_t)e * 512 + c) * 16]; if (v && d[((size_t)e * 512 + c) * 16 + 1]) { t0 = std::min(t0, v); n++; } }
    if (!n) continue;
    fprintf(stderr, "[ts stamps] product %d, %d live CTAs:", e, n);
    for (int i = 0; i < 10; i++) {
      std::vector<double> v;
      for (int c = 0; c < 512; c++) { const unsigned long long* r = &d[((size_t)e * 512 + c) * 16]; if (r[0] && r[1] && r[i]) v.push_back((double)(r[i] - t0) / 1000.0); }
      if (v.empty()) { fprintf(stderr, " -"); continue; }
      std::sort(v.begin(), v.end());
      fprintf(stderr, " %d:%.1f/%.1f", i, v[v.size() / 2], v.back());
    }
    fprintf(stderr, "\n");
  }
}
// one mini-batch on the tensor cores (window-relative step = *base + off when base != nullptr).  Three streams (forked / joined
// with events, so the same code is captured into the step graph): the main stream carries the chain every product waits for;
// side stream 1 prepares operands that do not depend on it (weights, item-table rows, transposed operands) and runs the dSy
// product + the update of the scored rows; side stream 2 runs the dense-gradient products + dense update.
static int g_ts_pdl = 0;               // programmatic dependent launch along the main chain (G4R_TS_PDL=0 switches it off)
static int g_ts_cluster_big = 16;      // cluster size for the long-K products (non-portable size; G4R_TS_CLUSTER_BIG overrides)
static int g_ts_cluster_cap = 0;       // largest cluster the K splits may form (8 = portable limit; G4R_TS_CLUSTER overrides)
template <int EPI>
static int launch_ts_gemm(g4r_handle* h, cudaStream_t q, int ph, const int* base, int off, TsGemm g, const TsBuf& tb) {
  cudaLaunchConfig_t lc = {};
  cudaLaunchAttribute at[2];
  lc.gridDim = dim3(g.m_tiles * g.n_tiles * g.ksplit); lc.blockDim = dim3(TS_THREADS); lc.dynamicSmemBytes = sizeof(TsSmem); lc.stream = q;
  at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = g.fused ? g.ksplit : 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[1].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at; lc.numAttrs = (g_ts_pdl && q == h->stream) ? 2 : 1;
  int slot = h->slot;
  if (h->ts_dbg) g.dbg = h->ts_dbg + (size_t)EPI * 512 * 16;
  void* args[] = {&slot, (void*)&base, &off, &g, (void*)&tb};
  cudaError_t e = cudaSuccess;
  LAUNCH_ON(q, ph, e = cudaLaunchKernelExC(&lc, (const void*)k_ts_gemm<EPI>, args));
  if (e != cudaSuccess) { h->err = std::string("k_ts_gemm launch: ") + cudaGetErrorString(e); return G4R_ERR_CUDA; }
  return G4R_OK;
}
// main-stream elementwise kernel (slot, base, off[, tb]) as a programmatic dependent of its predecessor
static void launch_pdl(g4r_handle* h, int ph, const void* fn, dim3 grid, dim3 block, const int* base, int off, const TsBuf* tb) {
  cudaLaunchConfig_t lc = {};
  cudaLaunchAttribute at[1];
  lc.gridDim = grid; lc.blockDim = block; lc.dynamicSmemBytes = 0; lc.stream = h->stream;
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at; lc.numAttrs = g_ts_pdl ? 1 : 0;
  int slot = h->slot;
  void* args[] = {&slot, (void*)&base, &off, (void*)tb};
  LAUNCH(ph, cudaLaunchKernelExC(&lc, fn, args));
}
template <int EPI>
static void launch_ts_epi(g4r_handle* h, cudaStream_t st, int ph, const int* base, int off, const TsGemm& g, const TsBuf& tb, int rows, int cols) {
  LAUNCH_ON(st, ph, k_ts_epi<EPI><<<std::min(4 * h->n_sm, std::max(1, (rows * (cols / 4) + 255) / 256)), 256, 0, st>>>(h->slot, base, off, g, tb));
}
static int ts_opt_in(g4r_handle* h) {
  { const char* e = getenv("G4R_TS_PDL"); g_ts_pdl = e ? atoi(e) : 1; }
  if (getenv("G4R_TS_STAMP") && !h->ts_dbg) { cudaMalloc(&h->ts_dbg, 9 * 512 * 16 * sizeof(unsigned long long)); cudaMemset(h->ts_dbg, 0, 9 * 512 * 16 * sizeof(unsigned long long)); }
  { const char* e = getenv("G4R_TS_CLUSTER_BIG"); if (e) g_ts_cluster_big = std::max(1, std::min(16, atoi(e))); }
  if (!g_ts_cluster_cap) { const char* e = getenv("G4R_TS_CLUSTER"); g_ts_cluster_cap = e ? std::max(1, std::min(16, atoi(e))) : 8; }
  const void* fns[] = {(const void*)k_ts_gemm<TS_EPI_F1>, (const void*)k_ts_gemm<TS_EPI_F2>, (const void*)k_ts_gemm<TS_EPI_SCORE>, (const void*)k_ts_gemm<TS_EPI_DSY>,
                       (const void*)k_ts_gemm<TS_EPI_DH>, (const void*)k_ts_gemm<TS_EPI_B2>, (const void*)k_ts_gemm<TS_EPI_B3>,
                       (const void*)k_ts_gemm<TS_EPI_DENSE_A>, (const void*)k_ts_gemm<TS_EPI_DENSE_B>};
  for (const void* f : fns) {
    if (raise_smem_limit(f, sizeof(TsSmem)) != cudaSuccess) return G4R_ERR_CUDA;
    if (cudaFuncSetAttribute(f, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) return G4R_ERR_CUDA;
  }
  // a cluster larger than the portable 8 (one CTA per SM) must fit into one GPC: halve it until the device can schedule one
  while (g_ts_cluster_big > 8) {
    cudaLaunchConfig_t lc = {};
    cudaLaunchAttribute at[1];
    lc.gridDim = dim3(g_ts_cluster_big); lc.blockDim = dim3(TS_THREADS); lc.dynamicSmemBytes = sizeof(TsSmem);
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = g_ts_cluster_big; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    lc.attrs = at; lc.numAttrs = 1;
    int ncl = 0;
    if (cudaOccupancyMaxActiveClusters(&ncl, k_ts_gemm<TS_EPI_DH>, &lc) == cudaSuccess && ncl >= 1) break;
    cudaGetLastError();
    g_ts_cluster_big /= 2;
  }
  return G4R_OK;
}
static int enqueue_tc_step(g4r_handle* h, const int* base, int off) {
  const ModelDev& md = h->md;
  const TsBuf& tb = *static_cast<TsBuf*>(h->ts_buf);
  cudaStream_t st = h->stream, s1 = h->side, s2 = h->side2;
  cudaEvent_t* ev = h->ts_ev;
  const int L = md.L, B = md.B, slot = h->slot;
  const int fillg = 2 * h->n_sm;
  auto mk = [&](const unsigned char* A, const unsigned char* Bm, float* P, int chunks, int rows, int cols) -> TsGemm {
    const bool fused = P != tb.Pa && P != tb.Pb;
    int cap = g_ts_cluster_cap;
    if (chunks > 4 * cap) cap = std::max(cap, g_ts_cluster_big);       // long K (dL/dh, dL/d input): more, shorter splits
    const TsShape t = ts_shape(rows, cols, chunks, h->n_sm, fused ? cap : 0);
    TsGemm g; g.A = A; g.Bm = Bm; g.P = P; g.fused = fused; g.dbg = nullptr; g.chunks = chunks; g.m_tiles = t.m_tiles; g.n_tiles = t.n_tiles; g.NT = t.NT; g.ksplit = t.ksplit; g.ldP = t.ldP; g.epi = 0;
    return g;
  };
#define TS_GEMM(EPI, q, ph, g) do { const int rc_ = launch_ts_gemm<EPI>(h, q, ph, base, off, g, tb); if (rc_) return rc_; } while (0)
  auto fork = [&](int e, cudaStream_t from, cudaStream_t to) { cudaEventRecord(ev[e], from); cudaStreamWaitEvent(to, ev[e], 0); };
  fork(0, st, s1);
  // side 1: weight operands, item-table operands
  LAUNCH_ON(s1, PH_F1, k_ts_prep_w<<<dim3(fillg, 4), 256, 0, s1>>>(slot, tb));
  cudaEventRecord(ev[1], s1);
  LAUNCH_ON(s1, PH_SCORE, k_ts_prep_tab<<<dim3(fillg, 3), 256, 0, s1>>>(slot, base, off, tb));
  cudaEventRecord(ev[2], s1);
  // main: input rows, GRU forward
  LAUNCH(PH_GATHER, k_ts_prep_fwd<<<dim3(fillg, 2), 256, 0, st>>>(slot, base, off, tb));
  cudaStreamWaitEvent(st, ev[1], 0);
  TS_GEMM(TS_EPI_F1, st, PH_F1, mk(tb.A1, tb.W1, tb.P, tb.Lk2 / TC_KC, B, 2 * L));
  fork(3, st, s1);
  LAUNCH_ON(s1, PH_DENSE, k_ts_prep_a8<<<fillg, 256, 0, s1>>>(slot, base, off, tb));
  cudaEventRecord(ev[9], s1);
  TS_GEMM(TS_EPI_F2, st, PH_F2, mk(tb.A2, tb.W2, tb.P, tb.Lk2 / TC_KC, B, L));
  fork(4, st, s1);
  LAUNCH_ON(s1, PH_LOSSGRAD, k_ts_prep_yt<<<fillg, 256, 0, s1>>>(slot, base, off, tb));
  // main: scores, loss, dL/do
  cudaStreamWaitEvent(st, ev[2], 0);
  TS_GEMM(TS_EPI_SCORE, st, PH_SCORE, mk(tb.A3, tb.B3, tb.P, tb.Lk1 / TC_KC, B, md.NP));
  launch_pdl(h, PH_LOSSGRAD, (const void*)k_ts_loss, dim3(B), dim3(256), base, off, &tb);
  fork(5, st, s1);
  // side 1: dSy product and the update of the scored rows
  LAUNCH_ON(s1, PH_LOSSGRAD, k_ts_prep_g<<<dim3(fillg, 2), 256, 0, s1>>>(slot, base, off, tb));
  TS_GEMM(TS_EPI_DSY, s1, PH_LOSSGRAD, mk(tb.A4, tb.B4, tb.P1, tb.Bk / TC_KC, tb.Nk, L));
  LAUNCH_ON(s1, PH_LOSSGRAD, k_apply_rows<<<md.NCH, SC_THREADS, 0, s1>>>(slot, base, off));
  cudaEventRecord(ev[6], s1);
  // main: GRU backward (b1 is the epilogue of the dL/dh product)
  TS_GEMM(TS_EPI_DH, st, PH_B1, mk(tb.A5, tb.B5, tb.P, tb.Nk / TC_KC, B, L));
  fork(7, st, s2);
  // side 2: dense gradients of the da_h / da_z columns + update
  LAUNCH_ON(s2, PH_DENSE, k_ts_prep_b8<<<fillg, 256, 0, s2>>>(slot, base, off, tb, 0));
  cudaStreamWaitEvent(s2, ev[9], 0);       // A8 comes from side 1
  const TsGemm g8a = mk(tb.A8, tb.B8a, tb.Pa, tb.Bk / TC_KC, 3 * L, 2 * tb.Lp);
  TS_GEMM(TS_EPI_DENSE_A, s2, PH_DENSE, g8a);
  launch_ts_epi<TS_EPI_DENSE_A>(h, s2, PH_DENSE, base, off, g8a, tb, 3 * L, 2 * tb.Lp);
  TS_GEMM(TS_EPI_B2, st, PH_B2, mk(tb.A6, tb.W3, tb.P, tb.Lk1 / TC_KC, B, L));
  fork(8, st, s2);
  cudaStreamWaitEvent(s1, ev[8], 0);       // side 1 (idle by now): the bias gradient + update, dvec is complete
  LAUNCH_ON(s1, PH_DENSE, k_ts_bh<<<(3 * L + 31) / 32, 256, 0, s1>>>(slot, base, off));
  // side 2: the da_r columns
  LAUNCH_ON(s2, PH_DENSE, k_ts_prep_b8<<<fillg, 256, 0, s2>>>(slot, base, off, tb, 1));
  const TsGemm g8b = mk(tb.A8, tb.B8b, tb.Pb, tb.Bk / TC_KC, 3 * L, L);
  TS_GEMM(TS_EPI_DENSE_B, s2, PH_DENSE, g8b);
  launch_ts_epi<TS_EPI_DENSE_B>(h, s2, PH_DENSE, base, off, g8b, tb, 3 * L, L);
  // main: dL/d(input rows), then the input-row update (after the scored-row update: both touch the shared table)
  TS_GEMM(TS_EPI_B3, st, PH_B3, mk(tb.A7, tb.W4, tb.P, tb.Lk3 / TC_KC, B, L));
  cudaStreamWaitEvent(st, ev[6], 0);
  LAUNCH(PH_SPARSE_IN, k_sparse_in<<<B, 128, 0, st>>>(slot, base, off, 1));
  cudaEventRecord(ev[10], s2); cudaStreamWaitEvent(st, ev[10], 0);
  cudaEventRecord(ev[11], s1); cudaStreamWaitEvent(st, ev[11], 0);
#undef TS_GEMM
  return G4R_OK;
}

// the input gather and the GRU forward of one training step (window-relative index = *base + off when base != nullptr)
static void enqueue_forward(g4r_handle* h, const int* base, int off) {
  const ModelDev& md = h->md;
  cudaStream_t st = h->stream;
  const int B = md.B;
  if (md.mode != 0) LAUNCH(PH_GATHER, k_gather_in<<<std::max(1, (B + 7) / 8), 256, 0, st>>>(h->slot, base, off, 1));
  for (int li = 0; li < md.n_layers; li++) {
    const LayerDev& ly = md.layer[li];
    LAUNCH(PH_F1, k_f1<<<tiles2(2 * ly.L, B), GEMM_THREADS, 0, st>>>(h->slot, base, off, li, ly.H));
    LAUNCH(PH_F2, k_f2<<<tiles2(ly.L, B), GEMM_THREADS, 0, st>>>(h->slot, base, off, li, ly.H, 1));
  }
}
// the forward and score phases of one step, through the loss gradient
static void enqueue_forward_scores(g4r_handle* h, const int* base, int off) {
  const ModelDev& md = h->md;
  cudaStream_t st = h->stream;
  const int B = md.B;
  enqueue_forward(h, base, off);
  LAUNCH(PH_SCORE, k_score<<<md.NCH, SC_THREADS, score_smem_bytes(md.Bld), st>>>(h->slot, base, off));
  LAUNCH(PH_STATS, k_stats<<<B, 256, 256 * sizeof(float), st>>>(h->slot, base, off));
  if (md.smoothing > 0.f) {      // label smoothing: second statistics pass once the row maxima / normalisers are final
    LAUNCH(PH_STATS2, k_stats2a<<<md.NCH, 256, 0, st>>>(h->slot, base, off));
    LAUNCH(PH_STATS2, k_stats2b<<<B, 256, 0, st>>>(h->slot, base, off));
  }
  LAUNCH(PH_LOSSGRAD, k_lossgrad<<<md.NCH, SC_THREADS, lossgrad_smem_bytes(md.Bld, md.ldL), st>>>(h->slot, base, off));
}

// the backward phases and updates of one step once dL/dy of the top layer is in md.part (nch partials; 0: one per column chunk)
static void enqueue_backward(g4r_handle* h, const int* base, int off, int nch) {
  const ModelDev& md = h->md;
  cudaStream_t st = h->stream;
  const int B = md.B;
  for (int li = md.n_layers - 1; li >= 0; li--) {
    const LayerDev& ly = md.layer[li];
    LAUNCH(PH_B1, k_b1<<<std::max(1, std::min(h->n_sm, (B * ly.L * 8 + 255) / 256)), 256, 0, st>>>(h->slot, base, off, li, nch));
    LAUNCH(PH_B2, k_b2<<<tiles2(ly.L, B), GEMM_THREADS, 0, st>>>(h->slot, base, off, li));
    if (ly.in_dim > 0) LAUNCH(PH_B3, k_b3<<<tiles2(ly.in_dim, B), GEMM_THREADS, 0, st>>>(h->slot, base, off, li));
    const DenseJobs dj = dense_jobs(ly.L, ly.in_dim);
    LAUNCH(PH_DENSE, k_dense<<<dj.nWh + dj.nWrz + dj.nWx + dj.nBh, GEMM_THREADS, 0, st>>>(h->slot, base, off, li));
  }
  LAUNCH(PH_SPARSE_IN, k_sparse_in<<<B, 128, 0, st>>>(h->slot, base, off, 0));
  if (h->two_pass) {
    // grad_cap: the phases above ran in export mode (gradients only); global norm, then the updates with the scaled gradients
    const MgDev& mg = h->mgdev;
    LAUNCH(PH_GRADCAP, k_gradnorm<<<1, 1024, 0, st>>>(h->slot, base, off, mg.gradFlat, mg.gradCount, h->dGscale));
    LAUNCH(PH_GRADCAP, k_apply_rows<<<md.NCH, SC_THREADS, 0, st>>>(h->slot, base, off));
    for (const MgTensor& t : h->mg_tensors) LAUNCH(PH_GRADCAP, k_apply_dense<<<(t.count + 255) / 256, 256, 0, st>>>(h->slot, t.p, t.acc, t.vel, mg.gradFlat + t.goff, t.count));
    LAUNCH(PH_GRADCAP, k_sparse_in<<<B, 128, 0, st>>>(h->slot, base, off, 1));
  }
}

// enqueue the kernels of one training step (window-relative index = *base + off when base != nullptr)
static int enqueue_train_step(g4r_handle* h, const int* base, int off) {
  if (h->tc_ok) return enqueue_tc_step(h, base, off);
  if (h->cfg.full_softmax) return enqueue_full_step(h, base, off);
  enqueue_forward_scores(h, base, off);
  enqueue_backward(h, base, off, 0);
  return G4R_OK;
}

// ------------------------------------------------------------------------------------------------
// C ABI: lifecycle
// ------------------------------------------------------------------------------------------------
extern "C" int g4r_version(void) { return G4R_VERSION; }

extern "C" const char* g4r_last_error(const g4r_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

extern "C" int g4r_workspace_bytes(const g4r_config* cfg, size_t* bytes) {
  if (!cfg || !bytes) return G4R_ERR_INVALID;
  std::string err;
  int rc = validate_config(*cfg, err);
  if (rc) { g_create_error = err; return rc; }
  int n_sm = 132;
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) == cudaSuccess && dev_count > cfg->device) {
    cudaDeviceProp p; if (cudaGetDeviceProperties(&p, cfg->device) == cudaSuccess) n_sm = p.multiProcessorCount;
  }
  Carver cv{nullptr, 0, true};
  layout(*cfg, cv, nullptr, n_sm);
  *bytes = align_up(cv.off, 256) + 256;
  return G4R_OK;
}

extern "C" int g4r_destroy(g4r_handle* h) {
  if (!h) return G4R_OK;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  sessions_release(h);
  eval_release(h);
  if (h->ts_buf) { delete static_cast<TsBuf*>(h->ts_buf); h->ts_buf = nullptr; }
  shard_release(h);
  mg_release(h);
  if (h->graphU) cudaGraphExecDestroy(h->graphU);
  if (h->graph1) cudaGraphExecDestroy(h->graph1);
  slot_free(h->slot);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->hX) cudaFreeHost(h->hX);
  if (h->hY) cudaFreeHost(h->hY);
  if (h->hSlot) cudaFreeHost(h->hSlot);
  if (h->hM) cudaFreeHost(h->hM);
  if (h->hSti) cudaFreeHost(h->hSti);
  if (h->hF) cudaFreeHost(h->hF);
  if (h->hG) cudaFreeHost(h->hG);
  if (h->hCost) cudaFreeHost(h->hCost);
  if (h->hFlags) cudaFreeHost(h->hFlags);
  if (h->own_ws && h->ws) cudaFree(h->ws);
  if (h->bptt_cub) cudaFree(h->bptt_cub);
  if (h->ts_dbg) { ts_print_stamps(h); cudaFree(h->ts_dbg); }
  if (h->side) cudaStreamDestroy(h->side);
  if (h->side2) cudaStreamDestroy(h->side2);
  for (cudaEvent_t e : h->ts_ev) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return G4R_OK;
}

extern "C" int g4r_create(const g4r_config* cfg, void* device_workspace, size_t workspace_bytes, g4r_handle** out) {
  if (!cfg || !out) { g_create_error = "null argument"; return G4R_ERR_INVALID; }
  std::string err;
  int rc = validate_config(*cfg, err);
  if (rc) { g_create_error = err; return rc; }
  int dev_count = 0;
  cudaError_t ce = cudaGetDeviceCount(&dev_count);
  if (ce != cudaSuccess || dev_count <= cfg->device) {
    g_create_error = "no CUDA device available: libg4r has no CPU path";
    return G4R_ERR_CUDA;
  }
  g4r_handle* h = new g4r_handle();
  h->cfg = *cfg;
  auto bail = [&](int code, const std::string& m) { g_create_error = m; g4r_destroy(h); return code; };
  if (cudaSetDevice(cfg->device) != cudaSuccess) return bail(G4R_ERR_CUDA, "cudaSetDevice failed");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess) return bail(G4R_ERR_CUDA, "cudaGetDeviceProperties failed");
  h->n_sm = prop.multiProcessorCount;
  // step_mode 3: the role-specialised kernel is launched as thread-block clusters of FC_CLUSTER CTAs; the number of
  // co-resident clusters bounds the grid and therefore the number of column chunks (one chunk per CTA)
  int chunk_cap = h->n_sm;
  if (cfg->step_mode == 3) {
    h->fastc_grid = fastc_max_grid(h->n_sm);
    if (h->fastc_grid >= FC_CLUSTER * 2) chunk_cap = std::min(chunk_cap, h->fastc_grid);
  }
  if (fast_shape(*cfg, h->n_sm)) chunk_cap = h->n_sm - round4(cfg->layers[0]) / 4;   // step_mode 2: no chunks on the GRU CTAs
  size_t need = 0;
  { Carver cv{nullptr, 0, true}; layout(*cfg, cv, nullptr, chunk_cap); need = align_up(cv.off, 256) + 256; }
  if (device_workspace) {
    if (workspace_bytes < need) return bail(G4R_ERR_INVALID, "workspace too small");
    h->ws = (char*)device_workspace; h->own_ws = false;
  } else {
    if (cudaMalloc(&h->ws, need) != cudaSuccess) {
      if (cfg->full_softmax) return bail(G4R_ERR_INVALID, "full_softmax: the workspace of " + std::to_string(need) + " bytes does not fit in device memory");
      return bail(G4R_ERR_CUDA, "cudaMalloc of workspace failed");
    }
    h->own_ws = true;
  }
  h->ws_bytes = need;
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(G4R_ERR_CUDA, "stream create failed");
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1);
  if (cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&h->side2, cudaStreamNonBlocking) != cudaSuccess) return bail(G4R_ERR_CUDA, "stream create failed");
  for (cudaEvent_t& e : h->ts_ev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  if (cudaMemsetAsync(h->ws, 0, need, h->stream) != cudaSuccess) return bail(G4R_ERR_CUDA, "memset failed");
  // 256-byte align the carve base
  char* base = (char*)align_up((size_t)h->ws, 256);
  Carver cv{base, 0, false};
  layout(*cfg, cv, h, chunk_cap);
  h->slot = slot_alloc();
  if (h->slot < 0) return bail(G4R_ERR_STATE, "too many live g4r handles in this process");
  if (h->two_pass || cfg->bptt > 1) h->md.export_only = 1;       // grad_cap: every update waits for the global gradient norm; bptt: for the window
  if (cfg->bptt > 1) {
    const int nk = cfg->bptt * (h->md.B + h->md.NP);
    if (cub::DeviceRadixSort::SortKeys(nullptr, h->bptt_cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, nk, 0, 64, h->stream) != cudaSuccess ||
        cudaMalloc(&h->bptt_cub, std::max<size_t>(h->bptt_cub_bytes, 256)) != cudaSuccess)
      return bail(G4R_ERR_CUDA, "bptt: sort scratch allocation failed");
  }
  if (slot_upload(h->slot, h->md, h->stream) != cudaSuccess) return bail(G4R_ERR_CUDA, "constant upload failed");
  const int B = cfg->batch_size, CAP = h->CAP;
  bool ok = true;
  ok &= cudaMallocHost(&h->hX, (size_t)CAP * B * sizeof(int)) == cudaSuccess;
  ok &= cudaMallocHost(&h->hY, (size_t)CAP * B * sizeof(int)) == cudaSuccess;
  ok &= cudaMallocHost(&h->hSlot, (size_t)CAP * B * sizeof(int)) == cudaSuccess;
  ok &= cudaMallocHost(&h->hF, (size_t)CAP * B) == cudaSuccess;
  ok &= cudaMallocHost(&h->hM, (size_t)CAP * sizeof(int)) == cudaSuccess;
  ok &= cudaMallocHost(&h->hSti, (size_t)CAP * sizeof(int)) == cudaSuccess;
  ok &= cudaMallocHost(&h->hG, (size_t)CAP * sizeof(uint32_t)) == cudaSuccess;
  ok &= cudaMallocHost(&h->hCost, (size_t)CAP * sizeof(float)) == cudaSuccess;
  if (!ok) return bail(G4R_ERR_CUDA, "pinned host allocation failed");
  // opt in to large dynamic shared memory where needed
  h->pk_smem = std::max(std::max(score_smem_bytes(h->md.Bld), lossgrad_smem_bytes(h->md.Bld, h->md.ldL)), (size_t)2 * GK * (GB + 1) * sizeof(float));
  if (raise_smem_limit((const void*)k_score, score_smem_bytes(h->md.Bld)) != cudaSuccess ||
      raise_smem_limit((const void*)k_lossgrad, lossgrad_smem_bytes(h->md.Bld, h->md.ldL)) != cudaSuccess ||
      raise_smem_limit((const void*)k_plan, (size_t)h->npow2 * 8 + 1024) != cudaSuccess ||
      raise_smem_limit((const void*)k_persistent, h->pk_smem) != cudaSuccess)
    return bail(G4R_ERR_INVALID, "this shape needs more shared memory per block than the device offers (batch_size / layer width / n_sample too large for the step scratch)");
  {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_persistent, PK_THREADS, h->pk_smem);
    int coop = 0; cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, cfg->device);
    h->pk_blocks = (per_sm >= 1 && coop) ? h->n_sm : 0;
  }
  {
    const ModelDev& m = h->md;
    raise_smem_limit((const void*)k_fast_t<false>, sizeof(FastSmemR));
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fast_t<false>, FK_THREADS, sizeof(FastSmemR));
    const bool plain_opt = m.adapt <= G4R_ADAPT_ADAGRAD && !h->phase_only;    // the role-specialised kernels implement SGD / Adagrad (+momentum) only
    // k_fast_t<false>: ldL / 4 GRU CTAs, then one column CTA per chunk (the grid is n_sm CTAs, fast_shape chose
    // NCH = n_sm - ldL / 4); the first B of them also update the input rows.  fk_b1 sums at most 160 chunk
    // partials.  Otherwise these shapes run on the generic kernels with the same chunks; g4r_fast_windows() reports such
    // windows as slow ones.
    h->fast_ok = plain_opt && fast_shape(*cfg, h->n_sm) && h->pk_blocks == h->n_sm && per_sm >= 1 && m.NCH <= h->pk_blocks - m.ldL / 4 && m.NCH <= 160 &&
                 (m.adapt == G4R_ADAPT_ADAGRAD ? m.Wy_acc != nullptr : true);
    h->fastc_ok = plain_opt && cfg->step_mode == 3 && h->fastc_grid >= FC_CLUSTER * 2 && m.mode == 0 && m.n_layers == 1 && m.ldL <= 128 && m.B <= FK_B &&
                  m.NCH <= h->fastc_grid && (m.adapt == G4R_ADAPT_ADAGRAD ? m.Wy_acc != nullptr : true);
    cudaMallocHost(&h->hFlags, 4 * sizeof(int));
  }
  if (h->tc_ok) {
    if (ts_opt_in(h) != G4R_OK) return bail(G4R_ERR_CUDA, "k_ts_gemm: shared memory / cluster opt-in failed");
    h->fast_ok = false; h->fastc_ok = false;
  }
  if (cfg->full_softmax && full_opt_in(h) != G4R_OK) return bail(G4R_ERR_INVALID, "full_softmax: this batch size needs more shared memory per block than the device offers");
  if (cfg->step_mode == 1 && h->pk_blocks == 0) return bail(G4R_ERR_INVALID, "persistent mode unavailable (cooperative launch / shared memory)");
  if (h->md.shardR > 0) {
    const int src = shard_create(h);
    if (src) return bail(src, h->err);
    h->fast_ok = false; h->fastc_ok = false;       // the single-GPU kernels never run on a sharded handle
  }
  if (cudaStreamSynchronize(h->stream) != cudaSuccess) return bail(G4R_ERR_CUDA, "init sync failed");
  *out = h;
  return G4R_OK;
}

extern "C" void* g4r_stream(g4r_handle* h) { return h ? (void*)h->stream : nullptr; }
extern "C" int64_t g4r_kernel_launches(const g4r_handle* h) { return h ? h->launches : 0; }

// ------------------------------------------------------------------------------------------------
// tensors
// ------------------------------------------------------------------------------------------------
static TensorInfo* find_tensor(g4r_handle* h, const char* name) {
  auto it = h->tensors.find(name ? name : "");
  return it == h->tensors.end() ? nullptr : &it->second;
}
extern "C" int g4r_tensor_shape(g4r_handle* h, const char* name, int64_t* rows, int64_t* cols) {
  if (!h) return G4R_ERR_INVALID;
  TensorInfo* t = find_tensor(h, name);
  if (!t) FAIL(G4R_ERR_INVALID, std::string("unknown tensor ") + (name ? name : "(null)"));
  if (rows) *rows = t->rows;
  if (cols) *cols = t->cols;
  return G4R_OK;
}
extern "C" int g4r_set_tensor(g4r_handle* h, const char* name, const float* host, int64_t rows, int64_t cols) {
  if (!h || !host) return G4R_ERR_INVALID;
  TensorInfo* t = find_tensor(h, name);
  if (!t) FAIL(G4R_ERR_INVALID, std::string("unknown tensor ") + (name ? name : "(null)"));
  if (rows != t->rows || cols != t->cols) FAIL(G4R_ERR_INVALID, std::string("shape mismatch for ") + name);
  cudaSetDevice(h->cfg.device);
  if (t->ptr == h->md.Wy || t->ptr == h->md.By) h->wy_version++;
  if (t->sharded) return shard_set_tensor(h, *t, host);
  CK(cudaMemcpy2DAsync(t->ptr, t->ld * sizeof(float), host, cols * sizeof(float), cols * sizeof(float), rows, cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}
extern "C" int g4r_get_tensor(g4r_handle* h, const char* name, float* host, int64_t rows, int64_t cols) {
  if (!h || !host) return G4R_ERR_INVALID;
  TensorInfo* t = find_tensor(h, name);
  if (!t) FAIL(G4R_ERR_INVALID, std::string("unknown tensor ") + (name ? name : "(null)"));
  if (rows != t->rows || cols != t->cols) FAIL(G4R_ERR_INVALID, std::string("shape mismatch for ") + name);
  cudaSetDevice(h->cfg.device);
  if (t->sharded) return shard_get_tensor(h, *t, host);
  CK(cudaMemcpy2DAsync(host, cols * sizeof(float), t->ptr, t->ld * sizeof(float), cols * sizeof(float), rows, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}
extern "C" int g4r_reset_hidden(g4r_handle* h) {
  if (!h) return G4R_ERR_INVALID;
  cudaSetDevice(h->cfg.device);
  for (int i = 0; i < h->md.n_layers; i++) CK(cudaMemsetAsync(h->md.layer[i].H, 0, (size_t)h->md.B * h->md.layer[i].ldL * sizeof(float), h->stream));
  return G4R_OK;
}

// ------------------------------------------------------------------------------------------------
// negative sampling
// ------------------------------------------------------------------------------------------------
extern "C" int g4r_set_sampling_cdf(g4r_handle* h, const float* P, int64_t n) {
  if (!h || !P) return G4R_ERR_INVALID;
  if (n != h->cfg.n_items) FAIL(G4R_ERR_INVALID, "cdf length != n_items");
  cudaSetDevice(h->cfg.device);
  CK(cudaMemcpyAsync(h->dP, P, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->have_cdf = true;
  return G4R_OK;
}
extern "C" int g4r_set_logq_support(g4r_handle* h, const float* P0, int64_t n) {
  if (!h || !P0) return G4R_ERR_INVALID;
  if (n != h->cfg.n_items) FAIL(G4R_ERR_INVALID, "support length != n_items");
  // gru4rec.py:495: logq * log(concat(P0[targets], P0[samples] ** sample_alpha)), float32 arithmetic
  std::vector<float> lt(n), ls(n);
  for (int64_t i = 0; i < n; i++) {
    lt[i] = h->cfg.logq * logf(P0[i]);
    ls[i] = h->cfg.logq * logf(powf(P0[i], h->cfg.sample_alpha));
  }
  cudaSetDevice(h->cfg.device);
  CK(cudaMemcpyAsync(h->dLogP0t, lt.data(), n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->dLogP0s, ls.data(), n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}
extern "C" int g4r_sample_store_rows(g4r_handle* h) { return h ? h->gen_len : 0; }
extern "C" int g4r_set_sample_pointer(g4r_handle* h, int64_t p) { if (!h) return G4R_ERR_INVALID; h->sample_ptr = p; return G4R_OK; }
extern "C" int64_t g4r_get_sample_pointer(g4r_handle* h) { return h ? h->sample_ptr : -1; }

static void mrg_host_init(g4r_handle* h);

static int launch_search_store(g4r_handle* h) {
  const int64_t n = (int64_t)h->gen_len * h->cfg.n_sample;
  k_searchsorted<int><<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(h->dP, h->cfg.n_items, h->dU, n, h->dST);
  h->launches++;
  CK(cudaGetLastError());
  h->sample_ptr = 0; h->have_store = true;
  return G4R_OK;
}

extern "C" int g4r_generate_samples(g4r_handle* h) {
  if (!h) return G4R_ERR_INVALID;
  if (h->gen_len <= 0) FAIL(G4R_ERR_STATE, "no sample store configured");
  if (!h->have_cdf) FAIL(G4R_ERR_STATE, "sampling cdf not set");
  cudaSetDevice(h->cfg.device);
  const int64_t n = (int64_t)h->gen_len * h->cfg.n_sample;
  if (!h->mrg_init) { mrg_host_init(h); }
  // Each uniform() call takes a block of substreams once (graph construction); the compiled function then keeps
  // advancing the same streams (rstate is a shared-variable update) -- SURVEY Appendix B.
  k_mrg_uniform<<<(h->n_streams + 127) / 128, 128, 0, h->stream>>>(h->dMrgState, h->n_streams, h->dU, n);
  h->launches++;
  CK(cudaGetLastError());
  return launch_search_store(h);
}
extern "C" int g4r_mrg_uniform(g4r_handle* h, float* out, int64_t n) {
  if (!h || !out) return G4R_ERR_INVALID;
  if (h->gen_len <= 0 || n > (int64_t)h->gen_len * h->cfg.n_sample) FAIL(G4R_ERR_INVALID, "n exceeds uniform scratch");
  cudaSetDevice(h->cfg.device);
  if (!h->mrg_init) mrg_host_init(h);
  k_mrg_uniform<<<(h->n_streams + 127) / 128, 128, 0, h->stream>>>(h->dMrgState, h->n_streams, h->dU, n);
  h->launches++;
  CK(cudaMemcpyAsync(out, h->dU, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}
extern "C" int g4r_generate_samples_from_uniform(g4r_handle* h, const float* u, int64_t n) {
  if (!h || !u) return G4R_ERR_INVALID;
  if (h->gen_len <= 0) FAIL(G4R_ERR_STATE, "no sample store configured");
  if (!h->have_cdf) FAIL(G4R_ERR_STATE, "sampling cdf not set");
  if (n != (int64_t)h->gen_len * h->cfg.n_sample) FAIL(G4R_ERR_INVALID, "uniform count != generate_length * n_sample");
  cudaSetDevice(h->cfg.device);
  CK(cudaMemcpyAsync(h->dU, u, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  return launch_search_store(h);
}
extern "C" int g4r_set_sample_store(g4r_handle* h, const int64_t* st, int64_t rows) {
  if (!h || !st) return G4R_ERR_INVALID;
  if (h->gen_len <= 0 || rows != h->gen_len) FAIL(G4R_ERR_INVALID, "rows != generate_length");
  const int64_t n = rows * h->cfg.n_sample;
  std::vector<int> tmp(n);
  for (int64_t i = 0; i < n; i++) {
    if (st[i] < 0 || st[i] >= h->cfg.n_items) FAIL(G4R_ERR_INDEX, "Index out of bounds");
    tmp[i] = (int)st[i];
  }
  cudaSetDevice(h->cfg.device);
  CK(cudaMemcpyAsync(h->dST, tmp.data(), n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->sample_ptr = 0; h->have_store = true;
  return G4R_OK;
}
extern "C" int g4r_get_sample_store(g4r_handle* h, int64_t* st, int64_t rows) {
  if (!h || !st) return G4R_ERR_INVALID;
  if (h->gen_len <= 0 || rows != h->gen_len) FAIL(G4R_ERR_INVALID, "rows != generate_length");
  const int64_t n = rows * h->cfg.n_sample;
  std::vector<int> tmp(n);
  cudaSetDevice(h->cfg.device);
  CK(cudaMemcpyAsync(tmp.data(), h->dST, n * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int64_t i = 0; i < n; i++) st[i] = tmp[i];
  return G4R_OK;
}

// ---- MRG31k3p substream set-up on the host (theano.sandbox.rng_mrg restatement; SURVEY Appendix B) ----
static const int64_t MRG_M1 = 2147483647LL, MRG_M2 = 2147462579LL;
static const int64_t A1p72[3][3] = {{1516919229, 758510237, 499121365}, {1884998244, 1516919229, 335398200}, {601897748, 1884998244, 358115744}};
static const int64_t A2p72[3][3] = {{1228857673, 1496414766, 954677935}, {1133297478, 1407477216, 1496414766}, {2002613992, 1639496704, 1407477216}};
static const int64_t A1p134[3][3] = {{1702500920, 1849582496, 1656874625}, {828554832, 1702500920, 1512419905}, {1143731069, 828554832, 102237247}};
static const int64_t A2p134[3][3] = {{796789021, 1464208080, 607337906}, {1241679051, 1431130166, 1464208080}, {1401213391, 1178684362, 1431130166}};
static void matvec_mod(const int64_t A[3][3], const int64_t* v, int64_t m, int64_t* o) {
  for (int i = 0; i < 3; i++) {
    unsigned __int128 s = 0;
    for (int j = 0; j < 3; j++) s += (unsigned __int128)A[i][j] * (unsigned __int128)v[j];
    o[i] = (int64_t)(s % (unsigned __int128)m);
  }
}
static void mrg_ff(const int64_t* s, const int64_t A1[3][3], const int64_t A2[3][3], int64_t* o) {
  matvec_mod(A1, s, MRG_M1, o); matvec_mod(A2, s + 3, MRG_M2, o + 3);
}
// substreams a handle's uniform() draws from: fixed by the size of its sample store
static int mrg_stream_count(const g4r_handle* h) {
  const int64_t n = (int64_t)h->gen_len * h->cfg.n_sample;
  int64_t r = n; if (r > 6) r = r / 6;
  return (int)std::min<int64_t>(r, 15360);
}
static void mrg_host_init(g4r_handle* h) {
  h->n_streams = mrg_stream_count(h);
  for (int i = 0; i < 6; i++) h->mrg_rstate[i] = h->cfg.mrg_seed ? h->cfg.mrg_seed : 12345;
  // multi-GPU: every rank draws its own negatives -- rank r takes the r-th block of substreams (the block a further
  // uniform() call of the same generator would have taken: the base state advances by 2^134 per call, SURVEY appendix B)
  for (int r = 0; r < (h->cfg.world_size > 1 ? h->cfg.rank : 0); r++) { int64_t nb[6]; mrg_ff(h->mrg_rstate, A1p134, A2p134, nb); memcpy(h->mrg_rstate, nb, sizeof(nb)); }
  std::vector<int32_t> st((size_t)h->n_streams * 6);
  int64_t cur[6]; memcpy(cur, h->mrg_rstate, sizeof(cur));
  for (int i = 0; i < h->n_streams; i++) {
    for (int k = 0; k < 6; k++) st[(size_t)i * 6 + k] = (int32_t)cur[k];
    int64_t nx[6]; mrg_ff(cur, A1p72, A2p72, nx); memcpy(cur, nx, sizeof(cur));
  }
  int64_t nb[6]; mrg_ff(h->mrg_rstate, A1p134, A2p134, nb); memcpy(h->mrg_rstate, nb, sizeof(nb));
  cudaMemcpyAsync(h->dMrgState, st.data(), st.size() * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream);
  cudaStreamSynchronize(h->stream);
  h->mrg_init = true;
}

// ------------------------------------------------------------------------------------------------
// stand-alone custom ops
// ------------------------------------------------------------------------------------------------
extern "C" int g4r_searchsorted(g4r_handle* h, const float* d, int64_t n_d, const float* x, int64_t n_x, int64_t* y) {
  if (!h || !d || !x || !y || n_d <= 0 || n_x < 0) return G4R_ERR_INVALID;
  if (n_x == 0) return G4R_OK;
  cudaSetDevice(h->cfg.device);
  float *dd = nullptr, *dx = nullptr; long long* dy = nullptr;
  CK(cudaMalloc(&dd, n_d * sizeof(float))); CK(cudaMalloc(&dx, n_x * sizeof(float))); CK(cudaMalloc(&dy, n_x * sizeof(long long)));
  CK(cudaMemcpyAsync(dd, d, n_d * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(dx, x, n_x * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  k_searchsorted<long long><<<(unsigned)((n_x + 255) / 256), 256, 0, h->stream>>>(dd, (int)n_d, dx, n_x, dy);
  h->launches++;
  CK(cudaMemcpyAsync(y, dy, n_x * sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  cudaFree(dd); cudaFree(dx); cudaFree(dy);
  return G4R_OK;
}
extern "C" int g4r_gather_rows(g4r_handle* h, const float* table, int64_t rows, int64_t cols, const int64_t* idx, int64_t n_idx, float* out) {
  if (!h || !table || !idx || !out || rows <= 0 || cols <= 0 || n_idx < 0) return G4R_ERR_INVALID;
  if (n_idx == 0) return G4R_OK;
  cudaSetDevice(h->cfg.device);
  float *dt = nullptr, *dout = nullptr; long long* di = nullptr; int* derr = nullptr;
  CK(cudaMalloc(&dt, rows * cols * sizeof(float))); CK(cudaMalloc(&dout, n_idx * cols * sizeof(float)));
  CK(cudaMalloc(&di, n_idx * sizeof(long long))); CK(cudaMalloc(&derr, sizeof(int)));
  CK(cudaMemcpyAsync(dt, table, rows * cols * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(di, idx, n_idx * sizeof(long long), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemsetAsync(derr, 0, sizeof(int), h->stream));
  k_gather_rows<<<(unsigned)std::min<int64_t>(n_idx, (int64_t)h->n_sm * 8), 128, 0, h->stream>>>(dt, rows, cols, di, n_idx, dout, derr);
  h->launches++;
  int herr = 0;
  CK(cudaMemcpyAsync(out, dout, n_idx * cols * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(&herr, derr, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  cudaFree(dt); cudaFree(dout); cudaFree(di); cudaFree(derr);
  if (herr) FAIL(G4R_ERR_INDEX, "Index out of bounds");
  return G4R_OK;
}

// ------------------------------------------------------------------------------------------------
// schedule builder (gru4rec.py:594-651; evaluation.py:90-139), host C++
// ------------------------------------------------------------------------------------------------
// n_hist (evaluation only, g4r_schedule_build_history): per session id, its leading events that are history -- a lane's target
// is counted (flag bit 2) only past them, and n_events counts only those lanes
static int schedule_build(const int64_t* data_items, int64_t n_events, const int32_t* offs, int64_t n_sessions,
                          const int64_t* order, int32_t B, int32_t n_sample, int32_t mode, const int32_t* n_hist, g4r_schedule** out) {
  if (!data_items || !offs || !out || B <= 0 || n_sessions < 0) return G4R_ERR_INVALID;
  if (n_sessions < B) { g_create_error = "index out of bounds: fewer sessions than batch_size (reference: IndexError at gru4rec.py:596)"; return G4R_ERR_INDEX; }
  const bool want_pos = mode == (1 | G4R_SCHED_POSITIONS);   // evaluation schedule that also records input positions
  if (want_pos) mode = 1;
  g4r_schedule* s = new g4r_schedule();
  s->B = B; s->mode = mode; s->has_pos = want_pos; s->hist = n_hist != nullptr;
  auto sess_of = [&](int64_t it) -> int64_t { return order ? order[it] : it; };
  std::vector<int64_t> iters(B), start(B), end(B), hend(B);   // hend: first counted target position of the lane's session
  std::vector<int32_t> slots(B);
  std::vector<uint8_t> zero_next(B, 0), fin(B), valid(B);
  auto hist_end = [&](int64_t ss) -> int64_t { return n_hist ? (int64_t)offs[ss] + n_hist[ss] : 0; };
  for (int b = 0; b < B; b++) { iters[b] = b; start[b] = offs[sess_of(b)]; end[b] = offs[sess_of(b) + 1]; slots[b] = b; hend[b] = hist_end(sess_of(b)); }
  {
    // capacity up front.  While sessions are left every step runs all B lanes and consumes B (input, target) pairs; once the
    // supply is exhausted the remaining lanes finish their sessions within max_len steps.  A session of length l holds l - 1
    // pairs, so steps <= pairs / B + max_len.  At RSC15 size the arrays are ~270 MB: growing them by doubling would touch that
    // memory twice (page faults dominate the build time).
    int64_t pairs = 0, max_len = 1;
    for (int64_t i = 0; i < n_sessions; i++) {
      const int64_t ss = sess_of(i), len = (int64_t)offs[ss + 1] - offs[ss];
      if (len > 1) pairs += len - 1;
      max_len = std::max(max_len, len);
    }
    s->max_len = max_len;
    const size_t guess = (size_t)(pairs / B + max_len + 2);
    s->X.reserve(guess * B); s->Y.reserve(guess * B); s->slots.reserve(guess * B); s->F.reserve(guess * B); s->M.reserve(guess);
    if (want_pos) s->P.reserve(guess * B);
  }
  int64_t maxiter = B - 1;
  int M = B;
  while (true) {
    int64_t minlen = end[0] - start[0];
    for (int b = 1; b < M; b++) minlen = std::min(minlen, end[b] - start[b]);
    const int64_t nst = minlen - 1;        // mini-batches all M lanes can take before the shortest running session ends
    if (nst > 0) {
      for (int b = 0; b < M; b++)
        if (start[b] + nst >= n_events) { delete s; g_create_error = "schedule: event index out of range"; return G4R_ERR_INDEX; }
      const size_t base = s->X.size(), add = (size_t)nst * B;
      s->X.resize(base + add); s->Y.resize(base + add); s->slots.resize(base + add); s->F.resize(base + add);      // zero-filled
      int32_t* X = s->X.data() + base; int32_t* Y = s->Y.data() + base; int32_t* SL = s->slots.data() + base; uint8_t* F = s->F.data() + base;
      for (int64_t i = 0; i < nst; i++) {
        int32_t* x = X + i * B; int32_t* y = Y + i * B; int32_t* sl = SL + i * B;
        for (int b = 0; b < M; b++) {
          const int64_t p = start[b] + i;
          x[b] = (int32_t)data_items[p]; y[b] = (int32_t)data_items[p + 1]; sl[b] = slots[b];
        }
        for (int b = M; b < B; b++) { x[b] = -1; y[b] = -1; }
      }
      if (want_pos) {
        s->P.resize(base + add, -1);
        for (int64_t i = 0; i < nst; i++) for (int b = 0; b < M; b++) s->P[base + i * B + b] = start[b] + i;
      }
      if (mode == 0) {       // bit 0: the step that consumes a session's last event -- the lane's state is reset after it (gru4rec.py:647-651)
        uint8_t* f = F + (nst - 1) * B;
        for (int b = 0; b < M; b++) if (end[b] - start[b] == minlen) f[b] = 1;
      } else {               // bit 1: the lane starts a new session with this step -- its state is zeroed before it (evaluation.py:136-139)
        for (int b = 0; b < M; b++) if (zero_next[b]) { F[b] = 2; zero_next[b] = 0; }
      }
      s->M.insert(s->M.end(), (size_t)nst, M);
      if (n_hist) {          // bit 2: the lane's target (position start + i + 1) is past its session's history
        for (int64_t i = 0; i < nst; i++)
          for (int b = 0; b < M; b++) if (start[b] + i + 1 >= hend[b]) { F[i * B + b] |= 4; s->n_events++; }
      } else {
        s->n_events += nst * M;
      }
    }
    int n_finished = 0;
    for (int b = 0; b < M; b++) { start[b] += minlen - 1; fin[b] = (end[b] - start[b] <= 1); }
    for (int b = 0; b < M; b++) if (fin[b]) { n_finished++; iters[b] = maxiter + n_finished; }
    maxiter += n_finished;
    int n_valid = 0;
    for (int b = 0; b < M; b++) { valid[b] = iters[b] < n_sessions; n_valid += valid[b]; }
    if (n_valid == 0 || (mode == 0 && n_valid < 2 && n_sample == 0)) break;
    for (int b = 0; b < M; b++) if (fin[b] && valid[b]) {
      const int64_t ss = sess_of(iters[b]);
      start[b] = offs[ss]; end[b] = offs[ss + 1]; hend[b] = hist_end(ss);
      if (mode == 1) zero_next[b] = 1;
    }
    if (n_valid < M) {
      int w = 0;
      for (int b = 0; b < M; b++) if (valid[b]) {
        iters[w] = iters[b]; start[w] = start[b]; end[w] = end[b]; slots[w] = slots[b]; zero_next[w] = zero_next[b]; hend[w] = hend[b]; w++;
      }
      M = w;
    }
  }
  s->n_steps = (int64_t)s->M.size();
  *out = s;
  return G4R_OK;
}
extern "C" int g4r_schedule_build(const int64_t* data_items, int64_t n_events, const int32_t* offs, int64_t n_sessions,
                                  const int64_t* order, int32_t B, int32_t n_sample, int32_t mode, g4r_schedule** out) {
  return schedule_build(data_items, n_events, offs, n_sessions, order, B, n_sample, mode, nullptr, out);
}
extern "C" int g4r_schedule_build_history(const int64_t* data_items, int64_t n_events, const int32_t* offs, int64_t n_sessions,
                                          const int64_t* order, const int32_t* n_history, int32_t B, int32_t mode, g4r_schedule** out) {
  if (!n_history) { g_create_error = "g4r_schedule_build_history: n_history is NULL"; return G4R_ERR_INVALID; }
  if (mode != 1 && mode != (1 | G4R_SCHED_POSITIONS)) {
    g_create_error = "g4r_schedule_build_history: mode must be 1 or 1 | G4R_SCHED_POSITIONS (an evaluation schedule)";
    return G4R_ERR_INVALID;
  }
  if (offs && n_sessions > 0) {
    for (int64_t i = 0; i < n_sessions; i++) {
      const int64_t ss = order ? order[i] : i;
      if (n_history[ss] < 0 || n_history[ss] > offs[ss + 1] - offs[ss]) {
        g_create_error = "g4r_schedule_build_history: n_history of a session is negative or longer than the session";
        return G4R_ERR_INVALID;
      }
    }
  }
  return schedule_build(data_items, n_events, offs, n_sessions, order, B, 0, mode, n_history, out);
}
extern "C" int g4r_schedule_free(g4r_schedule* s) { delete s; return G4R_OK; }
extern "C" int64_t g4r_schedule_steps(const g4r_schedule* s) { return s ? s->n_steps : 0; }
extern "C" int64_t g4r_schedule_events(const g4r_schedule* s) { return s ? s->n_events : 0; }
extern "C" int g4r_schedule_export(const g4r_schedule* s, int32_t* X, int32_t* Y, uint8_t* flags, int32_t* M, int32_t* slots) {
  if (!s) return G4R_ERR_INVALID;
  const size_t n = s->X.size();
  if (X) memcpy(X, s->X.data(), n * sizeof(int32_t));
  if (Y) memcpy(Y, s->Y.data(), n * sizeof(int32_t));
  if (flags) memcpy(flags, s->F.data(), n);
  if (slots) memcpy(slots, s->slots.data(), n * sizeof(int32_t));
  if (M) memcpy(M, s->M.data(), s->M.size() * sizeof(int32_t));
  return G4R_OK;
}
extern "C" int g4r_schedule_positions(const g4r_schedule* s, int64_t* pos) {
  if (!s || !pos) return G4R_ERR_INVALID;
  if (!s->has_pos) { g_create_error = "g4r_schedule_positions: the schedule was not built with mode 1 | G4R_SCHED_POSITIONS"; return G4R_ERR_STATE; }
  memcpy(pos, s->P.data(), s->P.size() * sizeof(int64_t));
  return G4R_OK;
}

// ------------------------------------------------------------------------------------------------
// window upload + plan
// ------------------------------------------------------------------------------------------------
// copies steps [first, first+n) of the schedule into the pinned staging buffers; assigns sample-store rows
// and global step counters; stops early at a sample-store wrap.  Returns the number of steps staged.
static int64_t stage_window(g4r_handle* h, const g4r_schedule* s, int64_t first, int64_t n) {
  const int B = h->md.B;
  n = std::min<int64_t>(n, h->CAP);
  const bool store = h->gen_len > 0;
  if (store && h->sample_ptr >= h->gen_len) return 0;   // caller must regenerate first
  if (store) n = std::min<int64_t>(n, h->gen_len - h->sample_ptr);
  memcpy(h->hX, s->X.data() + first * B, (size_t)n * B * sizeof(int));
  memcpy(h->hY, s->Y.data() + first * B, (size_t)n * B * sizeof(int));
  memcpy(h->hSlot, s->slots.data() + first * B, (size_t)n * B * sizeof(int));
  memcpy(h->hF, s->F.data() + first * B, (size_t)n * B);
  memcpy(h->hM, s->M.data() + first, (size_t)n * sizeof(int));
  for (int64_t i = 0; i < n; i++) {
    h->hSti[i] = store ? (int)(h->sample_ptr + i) : -1;
    h->hG[i] = h->global_step + (uint32_t)i;
  }
  return n;
}

static int validate_window(g4r_handle* h, int64_t n) {
  const int B = h->md.B, I = h->md.n_items;
  for (int64_t i = 0; i < n; i++) {
    const int M = h->hM[i];
    if (M <= 0 || M > B) FAIL(G4R_ERR_INVALID, "batch size out of range");
    for (int b = 0; b < M; b++) {
      const int x = h->hX[i * B + b], y = h->hY[i * B + b], sl = h->hSlot[i * B + b];
      if (x < 0 || x >= I || y < 0 || y >= I) FAIL(G4R_ERR_INDEX, "Index out of bounds");
      if (sl < 0 || sl >= B) FAIL(G4R_ERR_INDEX, "lane slot out of bounds");
    }
  }
  return G4R_OK;
}

static int upload_window(g4r_handle* h, int64_t n) {
  const int B = h->md.B;
  int rc = validate_window(h, n);
  if (rc) return rc;
  if (h->gen_len > 0 && !h->have_store) FAIL(G4R_ERR_STATE, "sample store not generated");
  cudaStream_t st = h->stream;
  CK(cudaMemcpyAsync(h->dX, h->hX, (size_t)n * B * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dY, h->hY, (size_t)n * B * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dSlot, h->hSlot, (size_t)n * B * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dF, h->hF, (size_t)n * B, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dM, h->hM, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dSti, h->hSti, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dG, h->hG, (size_t)n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(h->md.nanflag + 2, 0, sizeof(int), st));
  k_plan<<<(unsigned)n, 256, (size_t)h->npow2 * 8 + 1024, st>>>(h->md, h->dXnext, h->dXflag, h->npow2);
  h->launches++;
  if (h->cfg.full_softmax) full_mark_inputs(h, n);
  CK(cudaGetLastError());
  h->win_steps = (int)n;
  if (h->shard) return mgs_plan_window(h, n);
  return G4R_OK;
}

static int build_graph(g4r_handle* h, int unroll, cudaGraphExec_t* out) {
  cudaGraph_t g = nullptr;
  CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
  const int64_t l0 = h->launches;
  for (int i = 0; i < unroll; i++) enqueue_train_step(h, h->dStepBase, i);
  k_advance<<<1, 32, 0, h->stream>>>(h->dStepBase, unroll);
  h->launches = l0;
  CK(cudaStreamEndCapture(h->stream, &g));
  CK(cudaGraphInstantiate(out, g, 0));
  cudaGraphDestroy(g);
  return G4R_OK;
}
static int64_t launches_per_step(const g4r_handle* h) {
  const ModelDev& md = h->md;
  if (h->tc_ok) return 25;
  if (h->cfg.full_softmax) return full_launches_per_step(h);
  int64_t n = (md.mode != 0 ? 1 : 0) + 4;        // gather + score/stats/lossgrad + sparse_in
  for (int li = 0; li < md.n_layers; li++) n += 2 + 2 + (md.layer[li].in_dim > 0 ? 1 : 0) + 1;
  if (md.smoothing > 0.f) n += 2;
  if (h->two_pass) n += 3 + (int64_t)h->mg_tensors.size();
  return n;
}

static int run_window(g4r_handle* h, int64_t n) {
  bool fast = false, fastc = false;
  if ((h->cfg.step_mode == 3 && h->fastc_ok) || (h->cfg.step_mode == 2 && h->fast_ok)) {
    if (!h->prof) {
      // the plan kernel recorded the widest chunk of the window; the role-specialised kernels handle <= FK_CT columns per chunk
      CK(cudaMemcpyAsync(h->hFlags, h->md.nanflag, 4 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      const bool fits = h->hFlags[2] <= FK_CT;
      fastc = fits && h->cfg.step_mode == 3;
      fast = fits && h->cfg.step_mode == 2;
    }
  }
  if (fastc) {
    int slot = h->slot, nst = (int)n; FastSync* fsp = h->dFastSync; unsigned long long* ts = h->stamp_on ? h->dStamp : nullptr;
    void* args[] = {&slot, &nst, &fsp, &ts};
    CK(cudaMemsetAsync(h->dFastSync, 0, sizeof(FastSync), h->stream));
    CK(fastc_launch(h->fastc_grid, h->stream, args));
    h->launches += 1; h->fast_windows++;
  } else if (fast) {
    int slot = h->slot, nst = (int)n; FastSync* fsp = h->dFastSync; unsigned long long* ts = h->stamp_on ? h->dStamp : nullptr;
    void* args[] = {&slot, &nst, &fsp, &ts};
    CK(cudaMemsetAsync(h->dFastSync, 0, sizeof(FastSync), h->stream));
    CK(cudaLaunchCooperativeKernel((void*)k_fast_t<false>, dim3(h->pk_blocks), dim3(FK_THREADS), args, sizeof(FastSmemR), h->stream));
    h->launches += 1; h->fast_windows++;
  } else if (h->cfg.step_mode >= 1 && !h->prof && h->pk_blocks > 0 && !h->phase_only && !h->tc_ok) {
    if (h->cfg.step_mode >= 2) h->slow_windows++;
    int slot = h->slot, nst = (int)n; GridBar* gb = h->dGridBar; unsigned long long* ts = h->stamp_on ? h->dStamp : nullptr;
    void* args[] = {&slot, &nst, &gb, &ts};
    CK(cudaMemsetAsync(h->dGridBar, 0, sizeof(GridBar), h->stream));
    CK(cudaLaunchCooperativeKernel((void*)k_persistent, dim3(h->pk_blocks), dim3(PK_THREADS), args, h->pk_smem, h->stream));
    h->launches += 1;
  } else if (h->prof || !h->use_graph) {
    for (int64_t i = 0; i < n; i++) enqueue_train_step(h, nullptr, (int)i);
  } else {
    if (!h->graphU) { int rc = build_graph(h, h->graph_unroll, &h->graphU); if (rc) return rc; rc = build_graph(h, 1, &h->graph1); if (rc) return rc; }
    CK(cudaMemsetAsync(h->dStepBase, 0, sizeof(int), h->stream));
    int64_t i = 0;
    for (; i + h->graph_unroll <= n; i += h->graph_unroll) CK(cudaGraphLaunch(h->graphU, h->stream));
    for (; i < n; i++) CK(cudaGraphLaunch(h->graph1, h->stream));
    h->launches += n * launches_per_step(h) + (n / h->graph_unroll) + (n % h->graph_unroll);
  }
  CK(cudaGetLastError());
  if (h->gen_len > 0) h->sample_ptr += n;
  h->global_step += (uint32_t)n;
  if (h->cfg.full_softmax) h->full_steps += n;
  return G4R_OK;
}

#include "g4r_multi.cuh"
#include "g4r_shard.cuh"
#include "g4r_bptt.cuh"
static bool mg_is_ready(g4r_handle* h) { return h->mg_host && static_cast<MgHost*>(h->mg_host)->ready; }

extern "C" int g4r_upload_steps(g4r_handle* h, const g4r_schedule* s, int64_t first, int64_t n) {
  if (!h || !s) return G4R_ERR_INVALID;
  if (h->shard && n > MG_CAP) FAIL(G4R_ERR_INVALID, "row-sharded handle: at most MG_CAP steps per uploaded window");
  if (s->B != h->md.B) FAIL(G4R_ERR_INVALID, "schedule batch size != model batch size");
  if (first < 0 || n <= 0 || first + n > s->n_steps) FAIL(G4R_ERR_INVALID, "step range out of schedule");
  if (n > h->CAP) FAIL(G4R_ERR_INVALID, "n exceeds the resident window capacity");
  if (h->cfg.bptt > 1 && !bptt_aligned(h, s, first, n)) FAIL(G4R_ERR_INVALID, "bptt: the range must start at a multiple of bptt and hold whole windows unless it runs to the schedule's end");
  cudaSetDevice(h->cfg.device);
  if (h->gen_len > 0 && h->sample_ptr + n > h->gen_len) FAIL(G4R_ERR_STATE, "window would wrap the sample store; regenerate or shorten");
  const int64_t got = stage_window(h, s, first, n);
  if (got != n) FAIL(G4R_ERR_STATE, "could not stage the window");
  return upload_window(h, n);
}

extern "C" int g4r_run_uploaded(g4r_handle* h, float* cost_out, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  if (h->win_steps <= 0) FAIL(G4R_ERR_STATE, "no uploaded window");
  cudaSetDevice(h->cfg.device);
  h->wy_version++;
  const int n = h->win_steps;
  if (h->cfg.world_size > 1 && !mg_is_ready(h)) FAIL(G4R_ERR_STATE, "multi-GPU handle: call g4r_mg_init first");
  if (h->cfg.world_size > 1 && !h->shard) FAIL(G4R_ERR_STATE, "g4r_run_uploaded on a multi-GPU handle needs the row-sharded path");
  CK(cudaEventRecord(h->ev0, h->stream));
  int rc = h->shard ? mgs_run_window(h, n) : (h->cfg.bptt > 1 ? bptt_run_uploaded(h, n) : run_window(h, n));
  if (rc) return rc;
  CK(cudaEventRecord(h->ev1, h->stream));
  if (cost_out) CK(cudaMemcpyAsync(h->hCost, h->md.cost, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (h->shard) CK(cudaMemcpyAsync(h->hFlags, h->md.nanflag, 4 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (h->shard && h->hFlags[3]) FAIL(G4R_ERR_STATE, "multi-GPU: a cross-GPU wait timed out (a peer rank stopped or never started its window)");
  if (cost_out) memcpy(cost_out, h->hCost, (size_t)n * sizeof(float));
  if (device_ms) CK(cudaEventElapsedTime(device_ms, h->ev0, h->ev1));
  // re-running the same window is allowed for benchmarking: undo the pointer advance only on request (not here)
  return G4R_OK;
}

extern "C" int g4r_profile_uploaded(g4r_handle* h, float* phase_ms, int32_t* phase_launches, int32_t n_phases) {
  if (!h || !phase_ms || !phase_launches || n_phases < PH_COUNT) return G4R_ERR_INVALID;
  if (h->shard) FAIL(G4R_ERR_STATE, "per-phase profiling is a single-GPU measurement (row-sharded handle)");
  if (h->cfg.bptt > 1) FAIL(G4R_ERR_STATE, "per-phase profiling measures one-step updates (bptt > 1 handle)");
  if (h->win_steps <= 0) FAIL(G4R_ERR_STATE, "no uploaded window");
  cudaSetDevice(h->cfg.device);
  h->wy_version++;
  h->prof = true; h->prof_ev.clear(); h->prof_phase.clear();
  int rc = run_window(h, h->win_steps);
  h->prof = false;
  if (rc) return rc;
  CK(cudaStreamSynchronize(h->stream));
  for (int i = 0; i < n_phases; i++) { phase_ms[i] = 0.f; phase_launches[i] = 0; }
  for (size_t k = 0; k < h->prof_phase.size(); k++) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->prof_ev[2 * k], h->prof_ev[2 * k + 1]);
    phase_ms[h->prof_phase[k]] += ms; phase_launches[h->prof_phase[k]]++;
    cudaEventDestroy(h->prof_ev[2 * k]); cudaEventDestroy(h->prof_ev[2 * k + 1]);
  }
  h->prof_ev.clear(); h->prof_phase.clear();
  return G4R_OK;
}
// persistent mode: globaltimer stamps at phase boundaries of every step of the last window (6 per step, ns)
extern "C" int g4r_persistent_stamps(g4r_handle* h, int32_t enable, unsigned long long* out, int64_t n_steps) {
  if (!h) return G4R_ERR_INVALID;
  h->stamp_on = enable != 0;
  if (out && n_steps > 0) {
    if (n_steps > h->CAP) FAIL(G4R_ERR_INVALID, "n_steps exceeds window capacity");
    cudaSetDevice(h->cfg.device);
    CK(cudaMemcpyAsync(out, h->dStamp, (size_t)n_steps * 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return G4R_OK;
}
extern "C" int g4r_uses_tensor_cores(const g4r_handle* h) { return (h && h->tc_ok) ? 1 : 0; }
extern "C" int64_t g4r_fast_windows(const g4r_handle* h, int64_t* fallback_windows) {
  if (!h) return 0;
  if (fallback_windows) *fallback_windows = h->slow_windows;
  return h->fast_windows;
}
extern "C" int64_t g4r_bptt_windows(const g4r_handle* h) { return h ? h->bptt_windows : 0; }
extern "C" int64_t g4r_full_steps(const g4r_handle* h) { return h ? h->full_steps : 0; }
extern "C" const char* g4r_phase_name(int32_t i) { return (i >= 0 && i < PH_COUNT) ? kPhaseNames[i] : ""; }
extern "C" int g4r_phase_count(void) { return PH_COUNT; }

extern "C" int g4r_train_steps(g4r_handle* h, const g4r_schedule* s, int64_t first, int64_t n, float* cost_out, int64_t* nan_step) {
  if (!h || !s) return G4R_ERR_INVALID;
  if (s->B != h->md.B) FAIL(G4R_ERR_INVALID, "schedule batch size != model batch size");
  if (first < 0 || n < 0 || first + n > s->n_steps) FAIL(G4R_ERR_INVALID, "step range out of schedule");
  if (h->cfg.bptt > 1 && n > 0 && !bptt_aligned(h, s, first, n)) FAIL(G4R_ERR_INVALID, "bptt: the range must start at a multiple of bptt and hold whole windows unless it runs to the schedule's end");
  cudaSetDevice(h->cfg.device);
  h->wy_version++;
  if (nan_step) *nan_step = -1;
  if (h->cfg.bptt > 1) return bptt_train_steps(h, s, first, n, cost_out, nan_step);
  int64_t done = 0;
  while (done < n) {
    if (h->gen_len > 0 && (!h->have_store || h->sample_ptr >= h->gen_len)) {   // gru4rec.py:618-621
      int rc = g4r_generate_samples(h);
      if (rc) return rc;
    }
    const bool multi = h->cfg.world_size > 1;
    const int64_t w = stage_window(h, s, first + done, multi ? std::min<int64_t>(n - done, MG_CAP) : n - done);
    if (w <= 0) FAIL(G4R_ERR_STATE, "empty window");
    int rc = upload_window(h, w);
    if (rc) return rc;
    if (multi) {
      if (!mg_is_ready(h)) FAIL(G4R_ERR_STATE, "multi-GPU handle: call g4r_mg_init first");
      rc = h->shard ? mgs_run_window(h, w) : mg_run_window(h, w);
    } else rc = run_window(h, w);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h->hCost, h->md.cost, (size_t)w * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (h->shard) CK(cudaMemcpyAsync(h->hFlags, h->md.nanflag, 4 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (h->shard && h->hFlags[3]) FAIL(G4R_ERR_STATE, "multi-GPU: a cross-GPU wait timed out (a peer rank stopped or never started its window)");
    for (int64_t i = 0; i < w; i++) {
      if (cost_out) cost_out[done + i] = h->hCost[i];
      if (h->hCost[i] != h->hCost[i]) {
        if (nan_step) *nan_step = first + done + i;
        FAIL(G4R_ERR_NAN, "NaN error!");
      }
    }
    done += w;
  }
  return G4R_OK;
}

extern "C" int g4r_train_step(g4r_handle* h, const int32_t* X, const int32_t* Y, int32_t M, const int8_t* R, float* cost) {
  if (!h || !X || !Y) return G4R_ERR_INVALID;
  const int B = h->md.B;
  if (M <= 0 || M > B) FAIL(G4R_ERR_INVALID, "M out of range");
  if (h->shard) FAIL(G4R_ERR_STATE, "g4r_train_step: not available on a row-sharded multi-GPU handle (use g4r_train_steps)");
  if (h->cfg.bptt > 1) FAIL(G4R_ERR_STATE, "g4r_train_step: a bptt > 1 handle trains whole windows (use g4r_train_steps)");
  cudaSetDevice(h->cfg.device);
  h->wy_version++;
  if (h->gen_len > 0 && (!h->have_store || h->sample_ptr >= h->gen_len)) {
    int rc = g4r_generate_samples(h);
    if (rc) return rc;
  }
  for (int b = 0; b < B; b++) {
    h->hX[b] = b < M ? X[b] : -1; h->hY[b] = b < M ? Y[b] : -1; h->hSlot[b] = b;
    h->hF[b] = (b < M && R && R[b]) ? 1 : 0;
  }
  h->hM[0] = M; h->hSti[0] = h->gen_len > 0 ? (int)h->sample_ptr : -1; h->hG[0] = h->global_step;
  int rc = upload_window(h, 1);
  if (rc) return rc;
  rc = run_window(h, 1);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h->hCost, h->md.cost, sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (cost) *cost = h->hCost[0];
  if (h->hCost[0] != h->hCost[0]) FAIL(G4R_ERR_NAN, "NaN error!");
  return G4R_OK;
}

// ------------------------------------------------------------------------------------------------
// training state: checkpoint / resume and catalogue growth (DESIGN §3i)
// ------------------------------------------------------------------------------------------------
// Everything a training handle holds besides its named tensors and the sample store, in one flat blob: the header below, then
// n_streams x 6 int32 MRG31k3p stream states (zero until the first uniform() call seeds them).
#define G4R_STATE_MAGIC 0x53523447u      /* "G4RS" */
#define G4R_STATE_VERSION 1u
struct TrainStateHdr {
  uint32_t magic, version;
  uint64_t bytes;
  // the configuration the state is valid for
  int32_t n_sample, store_rows; uint32_t mrg_seed, dropout_seed; int32_t world_size, rank;
  // the state
  uint32_t global_step; int32_t mrg_init, n_streams, reserved;
  int64_t sample_ptr, mrg_rstate[6];
};
static TrainStateHdr train_state_header(const g4r_handle* h) {
  TrainStateHdr d; memset(&d, 0, sizeof(d));
  d.magic = G4R_STATE_MAGIC; d.version = G4R_STATE_VERSION;
  d.n_streams = mrg_stream_count(h);
  d.bytes = sizeof(TrainStateHdr) + (size_t)d.n_streams * 6 * sizeof(int32_t);
  d.n_sample = h->cfg.n_sample; d.store_rows = h->gen_len; d.mrg_seed = h->cfg.mrg_seed; d.dropout_seed = h->cfg.dropout_seed;
  d.world_size = h->cfg.world_size; d.rank = h->cfg.rank;
  return d;
}
extern "C" int g4r_train_state_bytes(g4r_handle* h, size_t* bytes) {
  if (!h || !bytes) return G4R_ERR_INVALID;
  if (h->cfg.world_size > 1) FAIL(G4R_ERR_STATE, "training state export / import is single-GPU only");
  *bytes = (size_t)train_state_header(h).bytes;
  return G4R_OK;
}
extern "C" int g4r_train_state_export(g4r_handle* h, void* host, size_t bytes) {
  if (!h || !host) return G4R_ERR_INVALID;
  if (h->cfg.world_size > 1) FAIL(G4R_ERR_STATE, "training state export / import is single-GPU only");
  TrainStateHdr d = train_state_header(h);
  if (bytes != d.bytes) FAIL(G4R_ERR_INVALID, "g4r_train_state_export: buffer size != g4r_train_state_bytes");
  d.global_step = h->global_step; d.mrg_init = h->mrg_init ? 1 : 0; d.sample_ptr = h->sample_ptr;
  if (h->mrg_init) memcpy(d.mrg_rstate, h->mrg_rstate, sizeof(d.mrg_rstate));
  char* out = static_cast<char*>(host);
  memcpy(out, &d, sizeof(d));
  const size_t sb = (size_t)d.n_streams * 6 * sizeof(int32_t);
  cudaSetDevice(h->cfg.device);
  if (h->mrg_init && sb) {
    CK(cudaMemcpyAsync(out + sizeof(d), h->dMrgState, sb, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  } else memset(out + sizeof(d), 0, sb);
  return G4R_OK;
}
extern "C" int g4r_train_state_import(g4r_handle* h, const void* host, size_t bytes) {
  if (!h || !host) return G4R_ERR_INVALID;
  if (h->cfg.world_size > 1) FAIL(G4R_ERR_STATE, "training state export / import is single-GPU only");
  // every check comes before the first write: a refused blob leaves the handle as it was
  const TrainStateHdr want = train_state_header(h);
  if (bytes < sizeof(TrainStateHdr)) FAIL(G4R_ERR_INVALID, "g4r_train_state_import: truncated blob");
  TrainStateHdr d; memcpy(&d, host, sizeof(d));
  if (d.magic != G4R_STATE_MAGIC) FAIL(G4R_ERR_INVALID, "g4r_train_state_import: not a training-state blob");
  if (d.version != G4R_STATE_VERSION) FAIL(G4R_ERR_INVALID, "g4r_train_state_import: unknown blob version");
  if (d.bytes != bytes || bytes != want.bytes) FAIL(G4R_ERR_INVALID, "g4r_train_state_import: truncated blob or a blob of another sample-store size");
  if (d.n_sample != want.n_sample || d.store_rows != want.store_rows || d.n_streams != want.n_streams)
    FAIL(G4R_ERR_INVALID, "g4r_train_state_import: the blob was exported with another n_sample / sample-store size");
  if (d.mrg_seed != want.mrg_seed || d.dropout_seed != want.dropout_seed || d.world_size != want.world_size || d.rank != want.rank)
    FAIL(G4R_ERR_INVALID, "g4r_train_state_import: the blob was exported with other seeds");
  if (d.sample_ptr < 0 || d.sample_ptr > std::max(want.store_rows, 0) || (d.mrg_init != 0 && d.mrg_init != 1))
    FAIL(G4R_ERR_INVALID, "g4r_train_state_import: sample pointer / flags out of range");
  const size_t sb = (size_t)d.n_streams * 6 * sizeof(int32_t);
  cudaSetDevice(h->cfg.device);
  if (d.mrg_init && sb) {
    CK(cudaMemcpyAsync(h->dMrgState, static_cast<const char*>(host) + sizeof(d), sb, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  h->global_step = d.global_step; h->sample_ptr = d.sample_ptr; h->mrg_init = d.mrg_init != 0; h->n_streams = d.mrg_init ? d.n_streams : 0;
  memcpy(h->mrg_rstate, d.mrg_rstate, sizeof(d.mrg_rstate));
  return G4R_OK;
}

// The tensors a trained model consists of: parameters, their optimizer state ("<name>.<slot>") and the training hidden state.
// *item_table: rows are catalogue items (Wy, By, E; Wx0 without an embedding).
static bool model_tensor(const g4r_handle* h, const std::string& name, bool* item_table) {
  const std::string base = name.substr(0, name.find('.'));
  const std::string kind = base.substr(0, base.find_first_of("0123456789"));
  *item_table = base == "Wy" || base == "By" || base == "E" || (base == "Wx0" && h->md.mode == 0);
  return *item_table || kind == "Wx" || kind == "Wh" || kind == "Wrz" || kind == "Bh" || (kind == "H" && name == base);
}
extern "C" int g4r_copy_item_tables(g4r_handle* h, g4r_handle* src, const float* new_Wy, const float* new_By, const float* new_in) {
  if (!h || !src) return G4R_ERR_INVALID;
  if (h == src) FAIL(G4R_ERR_INVALID, "g4r_copy_item_tables: source and destination are the same handle");
  const g4r_config &a = h->cfg, &b = src->cfg;
  if (a.world_size > 1 || b.world_size > 1) FAIL(G4R_ERR_STATE, "g4r_copy_item_tables is single-GPU only");
  bool same = a.device == b.device && a.n_layers == b.n_layers && a.batch_size == b.batch_size && a.embedding == b.embedding &&
              a.constrained_embedding == b.constrained_embedding && a.adapt == b.adapt && (a.momentum > 0.f) == (b.momentum > 0.f);
  for (int i = 0; same && i < a.n_layers; i++) same = a.layers[i] == b.layers[i];
  if (!same) FAIL(G4R_ERR_INVALID, "g4r_copy_item_tables: the handles differ in more than n_items (layers, batch size, embedding mode, optimizer state)");
  if (a.n_items < b.n_items) FAIL(G4R_ERR_INVALID, "g4r_copy_item_tables: the destination has fewer items than the source");
  const int64_t n_old = b.n_items, n_new = a.n_items;
  // the same names with matching shapes on both sides, before anything is written
  for (const auto& kv : src->tensors) {
    bool item = false;
    if (!model_tensor(src, kv.first, &item)) continue;
    const TensorInfo* t = find_tensor(h, kv.first.c_str());
    if (!t || t->cols != kv.second.cols || t->ld != kv.second.ld || t->rows != (item ? n_new : kv.second.rows) || kv.second.rows != (item ? n_old : t->rows))
      FAIL(G4R_ERR_INVALID, "g4r_copy_item_tables: tensor " + kv.first + " does not match between the handles");
  }
  cudaSetDevice(a.device);
  CK(cudaStreamSynchronize(src->stream));
  // new rows of the weights: one device block per table, freed after the copy
  struct Fill { const char* name; const float* host; float* dev; };
  Fill fills[3] = {{"Wy", new_Wy, nullptr}, {"By", new_By, nullptr}, {h->md.mode == 1 ? "E" : "Wx0", h->md.mode == 2 ? nullptr : new_in, nullptr}};
  int rc = G4R_OK;
  auto release = [&]() { for (Fill& f : fills) if (f.dev) { cudaFree(f.dev); f.dev = nullptr; } };
  if (n_new > n_old) for (Fill& f : fills) {
    if (!f.host) continue;
    const size_t nb = (size_t)(n_new - n_old) * find_tensor(h, f.name)->cols * sizeof(float);
    if (cudaMalloc(&f.dev, nb) != cudaSuccess || cudaMemcpyAsync(f.dev, f.host, nb, cudaMemcpyHostToDevice, h->stream) != cudaSuccess) { rc = G4R_ERR_CUDA; break; }
  }
  if (rc) { release(); FAIL(rc, "g4r_copy_item_tables: staging the new rows failed"); }
  for (const auto& kv : src->tensors) {
    bool item = false;
    if (!model_tensor(src, kv.first, &item)) continue;
    const TensorInfo& s = kv.second; const TensorInfo& d = *find_tensor(h, kv.first.c_str());
    if (!item) {
      if (cudaMemcpyAsync(d.ptr, s.ptr, (size_t)s.rows * s.ld * sizeof(float), cudaMemcpyDeviceToDevice, h->stream) != cudaSuccess) { rc = G4R_ERR_CUDA; break; }
      continue;
    }
    const float* fill = nullptr;
    for (const Fill& f : fills) if (kv.first == f.name) fill = f.dev;
    const int64_t n = n_new * d.ld;
    k_rows_extend<<<(unsigned)std::min<int64_t>((n + 255) / 256, (int64_t)h->n_sm * 16), 256, 0, h->stream>>>(d.ptr, s.ptr, n_old, n_new, d.ld, d.cols, fill);
    h->launches++;
  }
  if (!rc && (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(h->stream) != cudaSuccess)) rc = G4R_ERR_CUDA;
  release();
  h->wy_version++;
  if (rc) FAIL(rc, "g4r_copy_item_tables: device copy failed");
  return G4R_OK;
}

#include "g4r_eval.cuh"
#include "g4r_full.cuh"
#include "g4r_baselines.cuh"
#include "g4r_rules.cuh"
#include "g4r_bpr.cuh"
#include "g4r_sknn.cuh"
#include "g4r_narm.cuh"
#include "g4r_sasrec.cuh"
#include "g4r_srgnn.cuh"
#include "g4r_stamp.cuh"
#include "g4r_nextitnet.cuh"
#include "g4r_bert4rec.cuh"
