// g4r_baselines.cuh -- the session baselines of the reference's baselines.py (ItemKNN, Pop, SessionPop) on the device
// (DESIGN §3j): the item-kNN fit (co-occurrence counts, normalisation, top n_sims per row) and the event-parallel ranking that
// evaluate_gpu / evaluate_events run for a baseline.  Included at the end of g4r_lib.cu, after g4r_eval.cuh (sorted_lb, mix32);
// nothing here touches a g4r_handle.
#pragma once

constexpr int BL_POP = 0, BL_SESSIONPOP = 1, BL_ITEMKNN = 2, BL_BPR = 3, BL_SKNN = 5, BL_STAN = 6, BL_SR = 8, BL_AR = 9,
              BL_VSTAN = 11, BL_NARM = 12, BL_SASREC = 13, BL_SRGNN = 15, BL_STAMP = 17,
              BL_NEXTITNET = 19, BL_BERT4REC = 21;       // 4, 7, 10, 14, 16, 18 and 20 stay unused
constexpr int BPR_F_MAX = 1024;                        // n_factors bound of a BPR handle (g4r_bpr.cuh)
constexpr int KF_THREADS = 256;
constexpr int KF_KEEP_MAX = 1024;                       // n_sims bound: the kept entries of a row are sorted in shared memory
constexpr size_t KF_SCRATCH = (size_t)512 << 20;        // dense accumulators of the fit's resident CTAs
constexpr unsigned BL_TIE_SEED = 0x6A09E667U;           // key of the tiebreaking noise (fixed: evaluations are reproducible)

// NARM's device scratch (g4r_narm.cuh): per position indices, the carved float arrays, the logits, split partials, the
// sort of the input embeddings' rows, per slot the plan
struct NmScratch {
  int *PX = nullptr, *PY = nullptr, *PS = nullptr;
  float* f = nullptr; float* S = nullptr; float* part = nullptr;
  unsigned long long *keys = nullptr, *keys2 = nullptr; unsigned char* cub = nullptr; size_t cub_bytes = 0;
  long long* pstart = nullptr; int *plen = nullptr, *poff = nullptr;
};

struct g4r_baselines {
  int kind = 0, n_items = 0, n_keep = 0, device = 0, n_sm = 132;
  std::string err;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool ready = false;                                   // rows fitted / imported, or Pop scores set
  // ItemKNN, SR and AR: [n_items x n_keep] rows by (sim desc, index asc) and the same rows by index asc (lookups); len [n_items]
  int *dIdx = nullptr, *dIdxI = nullptr, *dLen = nullptr;
  double *dSim = nullptr, *dSimI = nullptr;
  // Pop / SessionPop: dense scores [n_items] (0 past top_n) and the positive ones by (score desc, index asc)
  double *dPop = nullptr, *dTopS = nullptr;
  int* dTop = nullptr;
  std::vector<int> hTop;
  std::vector<double> hPop;
  // BPR: item factors [n_items x n_keep] and biases float64; the fit's session factors and per-iteration buffers (bpr_mem, from
  // g4r_bl_bpr_begin until an import or the destroy)
  double *dI = nullptr, *dBI = nullptr, *dU = nullptr, *dLsig = nullptr;
  int *dRowS = nullptr, *dRowI = nullptr, *dPerm = nullptr, *dNeg = nullptr, *dPred = nullptr, *dLevel = nullptr, *dCtr = nullptr;
  unsigned long long *dKeys = nullptr, *dKeys2 = nullptr;
  unsigned* dFlag = nullptr;
  unsigned char* dCub = nullptr;
  std::vector<void*> bpr_mem;
  int64_t bpr_rows = 0, bpr_sessions = 0;
  size_t bpr_cub_bytes = 0;
  int bpr_end_bit = 64;
  unsigned bpr_tag = 0;                                 // the iteration's done-flag value (flags are never cleared)
  // SessionKNN (g4r_sknn.cuh): training sessions by recency rank (distinct items ascending), every item's sessions by rank
  int64_t *dSkOff = nullptr, *dSkIoff = nullptr;
  int *dSkItem = nullptr, *dSkIsess = nullptr;
  std::vector<void*> sknn_mem;
  int64_t sk_sessions = 0, sk_zmax = 0;                 // sk_zmax: distinct items of the n_keep longest training sessions
  int sk_sample = 0, sk_sim = 0;
  // STAN (the SessionKNN index above plus): each entry's last position in its session, W2 by rank and W3 (freed with the index);
  // W1 by prefix distance (g4r_bl_stan_set_w1, kept across index replacements)
  int* dStPos = nullptr;
  double *dStW2 = nullptr, *dStW3 = nullptr, *dStW1 = nullptr;
  int64_t st_n_w1 = 0;
  // VSTAN (the STAN index and W1 above plus): F per item and W4 by prefix distance, with the similarity (sk_sim) set by
  // g4r_bl_vstan_set; a fit clears them, and evaluation needs them set (vs_set)
  double *dVsF = nullptr, *dVsW4 = nullptr;
  int64_t vs_n_w4 = 0;
  bool vs_set = false;
  // NARM (g4r_narm.cuh): the flat float32 parameters, a device 1.0f, and dI = double(E), dBI = 0 for bpr_blocks; the fit's
  // gradient, Adam moments, training pieces and scratch (nm_mem, from g4r_bl_narm_begin until an import or the destroy)
  float *dNmTh = nullptr, *dNmOne = nullptr, *dNmG = nullptr, *dNmM = nullptr, *dNmV = nullptr, *dNmLoss = nullptr;
  int* dNmItems = nullptr;
  int nm_H = 0, nm_len = 0, nm_bs = 0;
  size_t nm_n = 0;
  long long nm_Pmax = 0;
  int64_t nm_step = 0;                                  // Adam steps since the fit began
  bool nm_fit = false;
  std::vector<int64_t> nm_off;                          // the training pieces' offsets (host)
  std::vector<void*> nm_mem;
  NmScratch nm_s;
  // SASRec (g4r_sasrec.cuh) keeps its parameters, fit, plan and scratch in the NARM fields above (nm_H unused, nm_len its
  // max_len), plus its shape and its per-position activations (sa_f, in nm_mem)
  int sa_blocks = 0, sa_heads = 0;
  float* sa_f = nullptr;
  // SR-GNN (g4r_srgnn.cuh) keeps its parameters, fit and scratch in the NARM fields above (nm_len its max_len), plus its step
  // count, its samples (host: first input, inputs) and its per-position float and int scratch (sg_f, sg_i, in nm_mem)
  int sg_step = 0;
  long long sg_icap = 0;
  std::vector<int64_t> sg_start;
  std::vector<int> sg_len;
  float* sg_f = nullptr;
  int* sg_i = nullptr;
  // STAMP (g4r_stamp.cuh) keeps its parameters, fit and scratch in the NARM fields above (nm_len its max_len), and its samples
  // and its per-position and per-sample float and int scratch in SR-GNN's (sg_start, sg_len, sg_f, sg_i; sg_icap its positions)
  // NextItNet (g4r_nextitnet.cuh) keeps its parameters, fit, plan and scratch in the NARM fields above (nm_len its max_len), plus
  // its dilations, kernel size and per-position activations (ni_f, in nm_mem)
  std::vector<int> ni_dil;
  int ni_K = 0;
  float* ni_f = nullptr;
  // BERT4Rec (g4r_bert4rec.cuh) keeps its parameters, fit, plan and scratch in the NARM fields above (nm_len its max_len, nm_off
  // the device's padded piece offsets) and its n_blocks / n_heads in SASRec's, plus its per-position activations, the masked rows'
  // targets and the device copy of the mask bytes (b4_f, b4_my, b4_mk, in nm_mem)
  float* b4_f = nullptr;
  int* b4_my = nullptr;
  unsigned char* b4_mk = nullptr;
};

// ---------------------------------------------------------------------------------------------------------------------------
// item-kNN fit
// ---------------------------------------------------------------------------------------------------------------------------
struct KnnFitDev {
  const int64_t* s_off; const int* s_item;              // per session its distinct items
  const int64_t* i_off; const int* i_sess; const int* i_mult;   // per item its (session, multiplicity) occurrences
  const int* order; int* next;                          // rows by decreasing pair work; the queue head
  const double* a; const double* b;                     // (supp_i + lmbd)^alpha, (supp_j + lmbd)^(1 - alpha)
  unsigned* acc; int* touched; double* sims;            // per CTA: dense counts [n_items], touched columns, their sims
  int n_items, n_keep;
  int* out_idx; double* out_sim; int* out_len;
};

// what g4r_bl_create and g4r_bl_evaluate know of each kind: its n_keep bound, the model storage the handle allocates at its
// creation (NONE: at the fit) and the function that ranks an evaluation (null: no such kind)
struct BlCall;
static int bl_rank_list(g4r_baselines* h, BlCall& c);  // k_bl_rank (below)
static int bpr_rank(g4r_baselines* h, BlCall& c);      // g4r_bpr.cuh
static int sknn_rank(g4r_baselines* h, BlCall& c);     // g4r_sknn.cuh
static int narm_rank(g4r_baselines* h, BlCall& c);     // g4r_narm.cuh
static int sasrec_rank(g4r_baselines* h, BlCall& c);   // g4r_sasrec.cuh
static int srgnn_rank(g4r_baselines* h, BlCall& c);    // g4r_srgnn.cuh
static int stamp_rank(g4r_baselines* h, BlCall& c);    // g4r_stamp.cuh
static int nextitnet_rank(g4r_baselines* h, BlCall& c);   // g4r_nextitnet.cuh
static int bert4rec_rank(g4r_baselines* h, BlCall& c);    // g4r_bert4rec.cuh
enum BlStore { BL_STORE_NONE, BL_STORE_ROWS, BL_STORE_POP, BL_STORE_BPR };
struct BlKind { int keep_max; BlStore store; int (*rank)(g4r_baselines*, BlCall&); };
constexpr BlKind BL_KINDS[] = {
    {INT32_MAX, BL_STORE_POP, bl_rank_list},            // 0 Pop
    {INT32_MAX, BL_STORE_POP, bl_rank_list},            // 1 SessionPop
    {KF_KEEP_MAX, BL_STORE_ROWS, bl_rank_list},         // 2 ItemKNN
    {BPR_F_MAX, BL_STORE_BPR, bpr_rank},                // 3 BPR
    {0, BL_STORE_NONE, nullptr},
    {KF_KEEP_MAX, BL_STORE_NONE, sknn_rank},            // 5 SessionKNN
    {KF_KEEP_MAX, BL_STORE_NONE, sknn_rank},            // 6 STAN
    {0, BL_STORE_NONE, nullptr},
    {KF_KEEP_MAX, BL_STORE_ROWS, bl_rank_list},         // 8 SR (g4r_rules.cuh; its rows rank as ItemKNN's)
    {KF_KEEP_MAX, BL_STORE_ROWS, bl_rank_list},         // 9 AR
    {0, BL_STORE_NONE, nullptr},
    {KF_KEEP_MAX, BL_STORE_NONE, sknn_rank},            // 11 VSTAN
    {BPR_F_MAX, BL_STORE_NONE, narm_rank},              // 12 NARM
    {BPR_F_MAX, BL_STORE_NONE, sasrec_rank},            // 13 SASRec
    {0, BL_STORE_NONE, nullptr},
    {BPR_F_MAX, BL_STORE_NONE, srgnn_rank},             // 15 SR-GNN
    {0, BL_STORE_NONE, nullptr},
    {BPR_F_MAX, BL_STORE_NONE, stamp_rank},             // 17 STAMP
    {0, BL_STORE_NONE, nullptr},
    {BPR_F_MAX, BL_STORE_NONE, nextitnet_rank},         // 19 NextItNet
    {0, BL_STORE_NONE, nullptr},
    {BPR_F_MAX, BL_STORE_NONE, bert4rec_rank},          // 21 BERT4Rec
};
static bool bl_kind_ok(int kind) { return kind >= 0 && kind < (int)(sizeof(BL_KINDS) / sizeof(BL_KINDS[0])) && BL_KINDS[kind].rank; }
// the kinds whose model is ItemKNN's rows
static bool bl_has_rows(int kind) { return BL_KINDS[kind].store == BL_STORE_ROWS; }

// (score desc, index asc): the order of every kept row and list
__device__ __forceinline__ bool bl_before(double sa, int ia, double sb, int ib) { return sa > sb || (sa == sb && ia < ib); }

// in-place bitonic sort of P (a power of two) shared (key, index) pairs; BYIDX: by index asc, else by bl_before
template <bool BYIDX>
__device__ void cta_bitonic(double* ks, int* ki, int P) {
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < P; t += blockDim.x) {
        const int u = t ^ stride;
        if (u <= t) continue;
        const bool up = (t & size) == 0;
        const bool u_first = BYIDX ? ki[u] < ki[t] : bl_before(ks[u], ki[u], ks[t], ki[t]);
        if (u_first == up) {
          const double s = ks[t]; ks[t] = ks[u]; ks[u] = s;
          const int i = ki[t]; ki[t] = ki[u]; ki[u] = i;
        }
      }
    }
  __syncthreads();
}

// row i of a fit (KF_THREADS threads): of the T touched columns tl[t] with values sv[t], the K largest by (value desc, index
// asc) -- a radix select on (value bits, then index) and a bitonic sort of the kept entries -- into out_idx / out_sim (-1 / 0
// past the kept ones) and out_len.  Only integer and bit operations: the values are copied, never computed.
__device__ void bl_keep_row(const double* sv, const int* tl, int T, int K, int i, int* out_idx, double* out_sim, int* out_len) {
  __shared__ double sKs[KF_KEEP_MAX];
  __shared__ int sKi[KF_KEEP_MAX];
  __shared__ unsigned sHist[256];
  __shared__ int sKn, sBin, sNeed, sFull;
  const int tid = threadIdx.x;
  if (tid == 0) sKn = 0;
  __syncthreads();
  {
    // every value is positive and finite, so its bits order like its value
    unsigned long long prefix = 0ull, mask = 0ull;
    int need = K, full = 1;
    unsigned jprefix = 0u, jmask = 0u;
    if (T > K) {
      full = 0;
      for (int shift = 56; shift >= 0 && !full; shift -= 8) {
        for (int q = tid; q < 256; q += KF_THREADS) sHist[q] = 0u;
        __syncthreads();
        for (int t = tid; t < T; t += KF_THREADS) {
          const unsigned long long key = (unsigned long long)__double_as_longlong(sv[t]);
          if ((key & mask) == prefix) atomicAdd(&sHist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
          int cum = 0, bin = 255;
          for (; bin > 0 && cum + (int)sHist[bin] < need; bin--) cum += (int)sHist[bin];
          sBin = bin; sNeed = need - cum; sFull = (int)sHist[bin] == need - cum;
        }
        __syncthreads();
        prefix |= (unsigned long long)sBin << shift; mask |= 255ull << shift; need = sNeed; full = sFull;
        __syncthreads();
      }
      if (!full) {          // sims equal to the boundary value: the `need` smallest indices
        for (int shift = 24; shift >= 0 && !full; shift -= 8) {
          for (int q = tid; q < 256; q += KF_THREADS) sHist[q] = 0u;
          __syncthreads();
          for (int t = tid; t < T; t += KF_THREADS) {
            const unsigned j = (unsigned)tl[t];
            if ((unsigned long long)__double_as_longlong(sv[t]) == prefix && (j & jmask) == jprefix) atomicAdd(&sHist[(j >> shift) & 255u], 1u);
          }
          __syncthreads();
          if (tid == 0) {
            int cum = 0, bin = 0;
            for (; bin < 255 && cum + (int)sHist[bin] < need; bin++) cum += (int)sHist[bin];
            sBin = bin; sNeed = need - cum; sFull = (int)sHist[bin] == need - cum;
          }
          __syncthreads();
          jprefix |= (unsigned)sBin << shift; jmask |= 255u << shift; need = sNeed; full = sFull;
          __syncthreads();
        }
      }
    }
    for (int t = tid; t < T; t += KF_THREADS) {
      bool keep = true;
      if (T > K) {
        const unsigned long long key = (unsigned long long)__double_as_longlong(sv[t]) & mask;
        keep = key > prefix || (key == prefix && (jmask == 0u || ((unsigned)tl[t] & jmask) <= jprefix));
      }
      if (keep) { const int q = atomicAdd(&sKn, 1); sKs[q] = sv[t]; sKi[q] = tl[t]; }
    }
    __syncthreads();
    const int n = sKn;
    int P = 1;
    while (P < n) P <<= 1;
    for (int q = n + tid; q < P; q += KF_THREADS) { sKs[q] = -1.0; sKi[q] = 0x7fffffff; }
    cta_bitonic<false>(sKs, sKi, P);
    for (int q = tid; q < K; q += KF_THREADS) {
      out_idx[(size_t)i * K + q] = q < n ? sKi[q] : -1;
      out_sim[(size_t)i * K + q] = q < n ? sKs[q] : 0.0;
    }
    if (tid == 0) out_len[i] = n;
    __syncthreads();
  }
}

// one CTA per row from the work queue: cnt(i, .) accumulated in the CTA's dense slice (a column enters the touched list when its
// count leaves 0), sims of the touched columns, the kept entries by bl_keep_row, and the slice cleared on the way (atomicExch
// reads and zeroes each touched count)
__global__ void __launch_bounds__(KF_THREADS) k_knn_fit(KnnFitDev d) {
  __shared__ int sRow, sT;
  unsigned* acc = d.acc + (size_t)blockIdx.x * d.n_items;
  int* tl = d.touched + (size_t)blockIdx.x * d.n_items;
  double* sv = d.sims + (size_t)blockIdx.x * d.n_items;
  const int tid = threadIdx.x;
  for (;;) {
    if (tid == 0) { sRow = atomicAdd(d.next, 1); sT = 0; }
    __syncthreads();
    if (sRow >= d.n_items) break;
    const int i = d.order[sRow];
    for (int64_t o = d.i_off[i] + tid; o < d.i_off[i + 1]; o += KF_THREADS) {
      const int s = d.i_sess[o];
      const unsigned c = (unsigned)d.i_mult[o];
      for (int64_t e = d.s_off[s]; e < d.s_off[s + 1]; e++) {
        const int j = d.s_item[e];
        if (j != i && atomicAdd(&acc[j], c) == 0u) tl[atomicAdd(&sT, 1)] = j;
      }
    }
    __syncthreads();
    const int T = sT;
    const double ai = d.a[i];
    for (int t = tid; t < T; t += KF_THREADS) {
      const int j = tl[t];
      const unsigned c = atomicExch(&acc[j], 0u);
      double nrm = __dmul_rn(ai, d.b[j]);
      if (nrm == 0.0) nrm = 1.0;
      sv[t] = __ddiv_rn((double)c, nrm);
    }
    __syncthreads();
    bl_keep_row(sv, tl, T, d.n_keep, i, d.out_idx, d.out_sim, d.out_len);
  }
}

// the rows again, by index asc (binary-search lookups of a column's sim)
__global__ void __launch_bounds__(KF_THREADS) k_knn_by_index(const int* idx, const double* sim, const int* len, int K, int* oidx, double* osim) {
  __shared__ double sKs[KF_KEEP_MAX];
  __shared__ int sKi[KF_KEEP_MAX];
  const int i = blockIdx.x, n = len[i], tid = threadIdx.x;
  int P = 1;
  while (P < n) P <<= 1;
  for (int q = tid; q < P; q += KF_THREADS) {
    sKs[q] = q < n ? sim[(size_t)i * K + q] : 0.0;
    sKi[q] = q < n ? idx[(size_t)i * K + q] : 0x7fffffff;
  }
  cta_bitonic<true>(sKs, sKi, P);
  for (int q = tid; q < K; q += KF_THREADS) {
    oidx[(size_t)i * K + q] = q < n ? sKi[q] : 0x7fffffff;
    osim[(size_t)i * K + q] = q < n ? sKs[q] : 0.0;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// the fit's inputs, derived on the device from the session CSR of the training events: every session sorted, its distinct
// items with multiplicities, every item's (session, multiplicity) occurrences, and the rows ordered by decreasing work
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int KP_SHORT = 64;        // sessions up to this length are sorted by one warp, longer ones by a CTA
constexpr int SCAN_B = 1024;

// warp per session: a session of <= KP_SHORT events is sorted into srt by rank (value, then position); a longer one is listed
// for k_kp_sort_long
__global__ void __launch_bounds__(256) k_kp_sort_short(const int64_t* off, int64_t S, const int* items, int* srt, int* long_list, int* n_long) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  const int64_t st = off[s];
  const int n = (int)(off[s + 1] - st);
  if (n > KP_SHORT) {
    if (lane == 0) long_list[atomicAdd(n_long, 1)] = (int)s;
    return;
  }
  for (int q = lane; q < n; q += 32) {
    const int v = items[st + q];
    int r = 0;
    for (int f = 0; f < n; f++) { const int u = items[st + f]; r += (u < v || (u == v && f < q)) ? 1 : 0; }
    srt[st + r] = v;
  }
}

// CTA per listed session: bitonic sort of the session, padded to a power of two, in the CTA's slice of `cap` ints of scratch
__global__ void __launch_bounds__(KF_THREADS) k_kp_sort_long(const int64_t* off, const int* items, int* srt, const int* long_list, const int* n_long,
                                                             int* scratch, int cap) {
  int* buf = scratch + (size_t)blockIdx.x * cap;
  const int tid = threadIdx.x;
  for (int q = blockIdx.x; q < *n_long; q += gridDim.x) {
    const int s = long_list[q];
    const int64_t st = off[s];
    const int n = (int)(off[s + 1] - st);
    int P = 1;
    while (P < n) P <<= 1;
    for (int t = tid; t < P; t += KF_THREADS) buf[t] = t < n ? items[st + t] : 0x7fffffff;
    for (int size = 2; size <= P; size <<= 1)
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        __syncthreads();
        for (int t = tid; t < P; t += KF_THREADS) {
          const int u = t ^ stride;
          if (u <= t) continue;
          const int x = buf[t], y = buf[u];
          if ((y < x) == ((t & size) == 0)) { buf[t] = y; buf[u] = x; }
        }
      }
    __syncthreads();
    for (int t = tid; t < n; t += KF_THREADS) srt[st + t] = buf[t];
    __syncthreads();
  }
}

// warp per session: its number of distinct items (the runs of its sorted events)
__global__ void __launch_bounds__(256) k_kp_count(const int64_t* off, int64_t S, const int* srt, long long* s_cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  const int64_t st = off[s], en = off[s + 1];
  int c = 0;
  for (int64_t e = st + lane; e < en; e += 32) c += (e == st || srt[e] != srt[e - 1]) ? 1 : 0;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) s_cnt[s] = c;
}

// exclusive scan out[0 .. n] of in[0 .. n) in three launches: blocks of SCAN_B, the block totals (one thread), the carries
__global__ void __launch_bounds__(SCAN_B) k_scan_block(const long long* in, int64_t n, long long* out, long long* tot) {
  __shared__ long long w[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * SCAN_B + threadIdx.x;
  long long v = i < n ? in[i] : 0;
  for (int o = 1; o < 32; o <<= 1) { const long long u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
  if (lane == 31) w[warp] = v;
  __syncthreads();
  if (warp == 0) {
    long long x = w[lane];
    for (int o = 1; o < 32; o <<= 1) { const long long u = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += u; }
    w[lane] = x;
  }
  __syncthreads();
  if (warp > 0) v += w[warp - 1];
  if (i < n) out[i + 1] = v;
  if (threadIdx.x == SCAN_B - 1) tot[blockIdx.x] = v;
}
__global__ void k_scan_tot(long long* tot, int64_t nb) {
  long long acc = 0;
  for (int64_t b = 0; b < nb; b++) { const long long v = tot[b]; tot[b] = acc; acc += v; }
}
__global__ void __launch_bounds__(SCAN_B) k_scan_add(long long* out, int64_t n, const long long* tot) {
  const int64_t i = (int64_t)blockIdx.x * SCAN_B + threadIdx.x;
  if (i < n) out[i + 1] += tot[blockIdx.x];
  if (i == 0) out[0] = 0;
}

// warp per session: its distinct items (ascending) and multiplicities into the session CSR; per item the number of sessions it
// occurs in and its pair work (the distinct items of those sessions); the total pair work sum_s n_s d_s
__global__ void __launch_bounds__(256) k_kp_emit(const int64_t* off, int64_t S, const int* srt, const int64_t* s_off, int* s_item, int* s_mult,
                                                 unsigned long long* i_cnt, unsigned long long* work, unsigned long long* pairs) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  const int64_t st = off[s], en = off[s + 1], o = s_off[s], d = s_off[s + 1] - o;
  int64_t base = 0;
  for (int64_t e0 = st; e0 < en; e0 += 32) {
    const int64_t e = e0 + lane;
    const bool head = e < en && (e == st || srt[e] != srt[e - 1]);
    const unsigned m = __ballot_sync(0xffffffffu, head);
    if (head) {
      const int j = srt[e];
      int64_t f = e + 1;
      while (f < en && srt[f] == j) f++;
      const int64_t q = o + base + __popc(m & ((1u << lane) - 1u));
      s_item[q] = j; s_mult[q] = (int)(f - e);
      atomicAdd(&i_cnt[j], 1ull);
      atomicAdd(&work[j], (unsigned long long)d);
    }
    base += __popc(m);
  }
  if (lane == 0) atomicAdd(pairs, (unsigned long long)((en - st) * d));
}

// warp per session: (session, multiplicity) into the occurrence list of each of its items.  The order inside a list depends on
// the atomics; the fit only sums integers over it, so the rows do not.
__global__ void __launch_bounds__(256) k_kp_occ(const int64_t* s_off, int64_t S, const int* s_item, const int* s_mult, const int64_t* i_off,
                                                unsigned* i_fill, int* i_sess, int* i_mult) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  for (int64_t q = s_off[s] + lane; q < s_off[s + 1]; q += 32) {
    const int j = s_item[q];
    const int64_t p = i_off[j] + atomicAdd(&i_fill[j], 1u);
    i_sess[p] = (int)s; i_mult[p] = s_mult[q];
  }
}

// rows by decreasing work to within a factor of two: bucket 64 - clz(work) (0 for no work), buckets in descending order
__global__ void k_kp_bucket_count(const unsigned long long* work, int NI, unsigned* cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NI) atomicAdd(&cnt[work[i] ? 64 - __clzll((long long)work[i]) : 0], 1u);
}
__global__ void k_kp_bucket_start(unsigned* cnt) {
  unsigned acc = 0;
  for (int b = 64; b >= 0; b--) { const unsigned v = cnt[b]; cnt[b] = acc; acc += v; }
}
__global__ void k_kp_bucket_place(const unsigned long long* work, int NI, unsigned* start, int* order) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < NI) order[atomicAdd(&start[work[i] ? 64 - __clzll((long long)work[i]) : 0], 1u)] = i;
}

// ---------------------------------------------------------------------------------------------------------------------------
// event-parallel ranking: one warp per session walks its events in order, keeping the session's input items so far (sorted,
// with counts) in the session's own slice of a scratch array; every counted event gets (#greater, #equal) over the competitors
// and, on request, its top-k list
// ---------------------------------------------------------------------------------------------------------------------------
struct BlEvalDev {
  int n_items, K, n_top, mode, k, exclude;
  const int* items; const int64_t* off; const int* nh; const int64_t* ev0;
  int* pl_item; int* pl_cnt;
  const int* rIdx; const double* rSim; const int* rLen; const int* rIdxI; const double* rSimI;
  const double* pop; const int* top; const double* topS; const long long* topW;   // topW[r]: competitor weight of top[0 .. r)
  const int* mult; long long wtot; const int* cdist; int n_cdist;                 // candidates: multiplicities, distinct ascending
  int* counts; int* out_items; double* out_scores;
};

// U(0,1) * 1e-10 of competitor `item` in counted event `e`
__device__ __forceinline__ double bl_noise(long long e, int item) {
  unsigned k = mix32(BL_TIE_SEED ^ (0x9E3779B9U * (unsigned)(e + 1)));
  k = mix32(k + (unsigned)((unsigned long long)e >> 32) * 0x85EBCA6BU);
  return __dmul_rn((double)(mix32(k + (unsigned)item) >> 8) * (1.0 / 16777216.0), 1e-10);
}

__device__ __forceinline__ int bl_plcount(const int* pl, const int* pc, int n, int j) {
  const int p = sorted_lb(pl, n, j);
  return (p < n && pl[p] == j) ? pc[p] : 0;
}
__device__ __forceinline__ double bl_knn(const BlEvalDev& d, int x, int j) {
  const int* r = d.rIdxI + (size_t)x * d.K;
  const int p = sorted_lb(r, d.rLen[x], j);
  return (p < d.rLen[x] && r[p] == j) ? d.rSimI[(size_t)x * d.K + p] : 0.0;
}
template <int KIND>
__device__ __forceinline__ double bl_score(const BlEvalDev& d, int x, const int* pl, const int* pc, int n, int j) {
  if (KIND == BL_ITEMKNN) return bl_knn(d, x, j);
  if (KIND == BL_POP) return d.pop[j];
  return __dadd_rn(d.pop[j], (double)bl_plcount(pl, pc, n, j));
}
__device__ __forceinline__ long long bl_w(const BlEvalDev& d, int j) { return d.mult ? (long long)d.mult[j] : 1ll; }
// a competitor that may enter a list: listed among the candidates (if any), not excluded as seen
__device__ __forceinline__ bool bl_eligible(const BlEvalDev& d, const int* pl, const int* pc, int n, int j) {
  return (!d.mult || d.mult[j] > 0) && !(d.exclude && bl_plcount(pl, pc, n, j) > 0);
}
// the competitors outside a scored set all score 0: they tie a target that scores 0 (sx: weight of the competitors the caller
// accounted for itself, the scored ones and the excluded zeros)
__device__ __forceinline__ long long bl_zero_eq(const BlEvalDev& d, double t, long long sx) { return t == 0.0 ? d.wtot - sx : 0ll; }
// first r of the descending topS[0 .. n) with topS[r] <= t (STRICT: < t)
template <bool STRICT>
__device__ __forceinline__ int bl_top_pos(const double* s, int n, double t) {
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (STRICT ? s[m] >= t : s[m] > t) lo = m + 1; else hi = m; }
  return lo;
}

// warp-wide: append the eligible entries of a candidate stream to list row `o` at *base (ballot order = stream order)
__device__ __forceinline__ void bl_emit(bool ok, int j, double sc, int* o_i, double* o_s, int k, int& base) {
  const unsigned m = __ballot_sync(0xffffffffu, ok);
  const int lane = threadIdx.x & 31, pos = base + __popc(m & ((1u << lane) - 1u));
  if (ok && pos < k) { o_i[pos] = j; o_s[pos] = sc; }
  base += __popc(m);
}

template <int KIND, bool LISTS>
__global__ void __launch_bounds__(256, 1) k_bl_rank(BlEvalDev d, int64_t n_sessions) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= n_sessions) return;
  const int64_t st = d.off[s], en = d.off[s + 1];
  if (en - st < 2) return;
  const int64_t p0 = st + max(d.nh ? d.nh[s] : 0, 1) - 1;
  int* pl = d.pl_item + st;
  int* pc = d.pl_cnt + st;
  int npl = 0;
  long long e = d.ev0[s];
  for (int64_t p = st; p + 1 < en; p++) {
    const int x = d.items[p];
    int nn = npl;
    if (lane == 0) {                                     // the input joins the session's items
      const int q = sorted_lb(pl, npl, x);
      if (q < npl && pl[q] == x) pc[q]++;
      else { for (int r = npl; r > q; r--) { pl[r] = pl[r - 1]; pc[r] = pc[r - 1]; } pl[q] = x; pc[q] = 1; nn++; }
    }
    __syncwarp();
    npl = __shfl_sync(0xffffffffu, nn, 0);
    if (p < p0) continue;
    const int y = d.items[p + 1];
    const bool miss = d.exclude && bl_plcount(pl, pc, npl, y) > 0;
    const double t = bl_score<KIND>(d, x, pl, pc, npl, y);
    long long gt = 0, eq = 0;
    if (d.mode == 3) {
      const double tn = __dadd_rn(t, bl_noise(e, y));
      const int n_comp = d.mult ? d.n_cdist : d.n_items;
      for (int q = lane; q < n_comp; q += 32) {
        const int j = d.mult ? d.cdist[q] : q;
        if (d.exclude && bl_plcount(pl, pc, npl, j) > 0) continue;
        const double sn = __dadd_rn(bl_score<KIND>(d, x, pl, pc, npl, j), bl_noise(e, j));
        const long long w = bl_w(d, j);
        gt += sn > tn ? w : 0; eq += sn == tn ? w : 0;
      }
    } else {
      long long sx = 0;                                  // weight of competitors outside the positive set that leave the zeros
      if (KIND == BL_ITEMKNN) {
        const int L = d.rLen[x];
        for (int q = lane; q < L; q += 32) {
          const int j = d.rIdx[(size_t)x * d.K + q];
          const double sc = d.rSim[(size_t)x * d.K + q];
          const long long w = bl_w(d, j);
          sx += w;                                       // kept entries are not zeros
          if (d.exclude && bl_plcount(pl, pc, npl, j) > 0) continue;
          gt += sc > t ? w : 0; eq += sc == t ? w : 0;
        }
        if (d.exclude)
          for (int q = lane; q < npl; q += 32) if (bl_knn(d, x, pl[q]) == 0.0) sx += bl_w(d, pl[q]);
      } else {
        const int ng = bl_top_pos<false>(d.topS, d.n_top, t), nge = bl_top_pos<true>(d.topS, d.n_top, t);
        if (lane == 0) { gt = d.topW[ng]; eq = d.topW[nge] - d.topW[ng]; sx = d.topW[d.n_top]; }
        if (KIND == BL_SESSIONPOP || d.exclude)
          for (int q = lane; q < npl; q += 32) {
            const int j = pl[q];
            const double pj = d.pop[j];
            const long long w = bl_w(d, j);
            if (pj > 0.0) { gt -= pj > t ? w : 0; eq -= pj == t ? w : 0; }
            else sx += w;
            if (KIND == BL_SESSIONPOP && !d.exclude) {
              const double sc = __dadd_rn(pj, (double)pc[q]);
              gt += sc > t ? w : 0; eq += sc == t ? w : 0;
            }
          }
      }
      for (int o = 16; o > 0; o >>= 1) sx += __shfl_xor_sync(0xffffffffu, sx, o);
      if (lane == 0) eq += bl_zero_eq(d, t, sx);
    }
    for (int o = 16; o > 0; o >>= 1) { gt += __shfl_xor_sync(0xffffffffu, gt, o); eq += __shfl_xor_sync(0xffffffffu, eq, o); }
    if (lane == 0) {
      d.counts[2 * e] = miss ? -1 : (int)gt;
      d.counts[2 * e + 1] = miss ? -1 : (int)eq;
    }
    if (LISTS) {
      int* o_i = d.out_items + (size_t)e * d.k;
      double* o_s = d.out_scores + (size_t)e * d.k;
      int base = 0;
      if (KIND == BL_ITEMKNN) {
        const int L = d.rLen[x];
        for (int q0 = 0; q0 < L && base < d.k; q0 += 32) {
          const int q = q0 + lane;
          const int j = q < L ? d.rIdx[(size_t)x * d.K + q] : 0;
          bl_emit(q < L && bl_eligible(d, pl, pc, npl, j), j, q < L ? d.rSim[(size_t)x * d.K + q] : 0.0, o_i, o_s, d.k, base);
        }
      } else {
        if (KIND == BL_SESSIONPOP && !d.exclude) {     // the session's items first: their scores are >= 1 > every Pop score
          int nel = 0;
          for (int q = lane; q < npl; q += 32) {
            const int j = pl[q];
            if (!bl_eligible(d, pl, pc, npl, j)) continue;
            const double sc = __dadd_rn(d.pop[j], (double)pc[q]);
            int r = 0;
            for (int f = 0; f < npl; f++)
              if (f != q && bl_eligible(d, pl, pc, npl, pl[f]) && bl_before(__dadd_rn(d.pop[pl[f]], (double)pc[f]), pl[f], sc, j)) r++;
            if (r < d.k) { o_i[r] = j; o_s[r] = sc; }
            nel++;
          }
          for (int o = 16; o > 0; o >>= 1) nel += __shfl_xor_sync(0xffffffffu, nel, o);
          base = nel;
        }
        for (int q0 = 0; q0 < d.n_top && base < d.k; q0 += 32) {
          const int q = q0 + lane;
          const int j = q < d.n_top ? d.top[q] : 0;
          const bool ok = q < d.n_top && bl_eligible(d, pl, pc, npl, j) && !(KIND == BL_SESSIONPOP && bl_plcount(pl, pc, npl, j) > 0);
          bl_emit(ok, j, q < d.n_top ? d.topS[q] : 0.0, o_i, o_s, d.k, base);
        }
      }
      const int n_comp = d.mult ? d.n_cdist : d.n_items;   // then the zero-score items, by index
      for (int q0 = 0; q0 < n_comp && base < d.k; q0 += 32) {
        const int q = q0 + lane;
        const int j = q < n_comp ? (d.mult ? d.cdist[q] : q) : 0;
        const bool ok = q < n_comp && bl_eligible(d, pl, pc, npl, j) && bl_score<KIND>(d, x, pl, pc, npl, j) == 0.0;
        bl_emit(ok, j, 0.0, o_i, o_s, d.k, base);
      }
      for (int q = base + lane; q < d.k; q += 32) { o_i[q] = -1; o_s[q] = __longlong_as_double(0x7ff8000000000000ll); }
    }
    __syncwarp();
    e++;
  }
}

// Recall / MRR sums over the counted events, in a fixed order (one block): rank by the mode's formula, a hit when rank <= N
__global__ void __launch_bounds__(1024) k_bl_sums(const int* counts, int64_t n, const int* cut, int n_cut, int mode, double* sums) {
  __shared__ double red[32][2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int c = 0; c < n_cut; c++) {
    double hit = 0.0, rr = 0.0;
    for (int64_t e = tid; e < n; e += 1024) {
      const int gt = counts[2 * e], eq = counts[2 * e + 1];
      if (gt < 0) continue;
      double rank;
      if (mode == 1) rank = (double)gt + (double)eq;
      else if (mode == 2) rank = (double)gt + 0.5 * (double)(eq - 1) + 1.0;
      else rank = (double)gt + 1.0;
      if (rank <= (double)cut[c]) { hit += 1.0; rr += 1.0 / rank; }
    }
    for (int o = 16; o > 0; o >>= 1) { hit += __shfl_xor_sync(0xffffffffu, hit, o); rr += __shfl_xor_sync(0xffffffffu, rr, o); }
    __syncthreads();
    if (lane == 0) { red[warp][0] = hit; red[warp][1] = rr; }
    __syncthreads();
    if (tid == 0) {
      double h = 0.0, r = 0.0;
      for (int w = 0; w < 32; w++) { h += red[w][0]; r += red[w][1]; }
      sums[c] = h; sums[n_cut + c] = r;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// C ABI (include/g4r.h)
// ---------------------------------------------------------------------------------------------------------------------------
static thread_local std::string g_bl_create_error;

template <class T>
static cudaError_t bl_alloc(T** p, size_t n) { return cudaMalloc((void**)p, std::max<size_t>(n, 1) * sizeof(T)); }

extern "C" const char* g4r_bl_last_error(const g4r_baselines* h) { return h ? h->err.c_str() : g_bl_create_error.c_str(); }

extern "C" int g4r_bl_destroy(g4r_baselines* h) {
  if (!h) return G4R_OK;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (void* p : {(void*)h->dIdx, (void*)h->dIdxI, (void*)h->dLen, (void*)h->dSim, (void*)h->dSimI, (void*)h->dPop, (void*)h->dTopS, (void*)h->dTop,
                  (void*)h->dI, (void*)h->dBI, (void*)h->dStW1, (void*)h->dVsF, (void*)h->dVsW4, (void*)h->dNmTh, (void*)h->dNmOne})
    if (p) cudaFree(p);
  for (void* p : h->bpr_mem) cudaFree(p);
  for (void* p : h->nm_mem) cudaFree(p);
  for (void* p : h->sknn_mem) cudaFree(p);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return G4R_OK;
}

extern "C" int g4r_bl_create(int32_t kind, int32_t n_items, int32_t n_keep, int32_t device, g4r_baselines** out) {
  if (!out) { g_bl_create_error = "null argument"; return G4R_ERR_INVALID; }
  if (!bl_kind_ok(kind)) {
    g_bl_create_error = "kind must be 0 (Pop), 1 (SessionPop), 2 (ItemKNN), 3 (BPR), 5 (SessionKNN), 6 (STAN), 8 (SR), 9 (AR), 11 (VSTAN), 12 (NARM), 13 (SASRec), 15 (SR-GNN), 17 (STAMP), 19 (NextItNet) or 21 (BERT4Rec)";
    return G4R_ERR_INVALID;
  }
  const BlStore store = BL_KINDS[kind].store;
  if (n_items < 1 || n_keep < 1 || n_keep > BL_KINDS[kind].keep_max) {
    g_bl_create_error = "need n_items >= 1 and 1 <= n_keep (<= " + std::to_string(KF_KEEP_MAX) + " for ItemKNN, SessionKNN, STAN, SR, AR and VSTAN, <= " +
                        std::to_string(BPR_F_MAX) + " n_factors for BPR and embedding for NARM, SASRec, SR-GNN, STAMP, NextItNet and BERT4Rec)";
    return G4R_ERR_INVALID;
  }
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count <= device || device < 0) {
    g_bl_create_error = "no CUDA device available: libg4r has no CPU path";
    return G4R_ERR_CUDA;
  }
  g4r_baselines* h = new g4r_baselines();
  h->kind = kind; h->n_items = n_items; h->n_keep = store == BL_STORE_POP ? std::min(n_keep, n_items) : n_keep; h->device = device;
  auto bail = [&](const char* m) { g_bl_create_error = m; g4r_bl_destroy(h); return G4R_ERR_CUDA; };
  if (cudaSetDevice(device) != cudaSuccess) return bail("cudaSetDevice failed");
  cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return bail("stream create failed");
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1);
  const size_t rows = (size_t)n_items * h->n_keep;
  bool ok = true;
  if (store == BL_STORE_BPR) {
    ok &= bl_alloc(&h->dI, rows) == cudaSuccess && bl_alloc(&h->dBI, n_items) == cudaSuccess;
  } else if (store == BL_STORE_ROWS) {
    ok &= bl_alloc(&h->dIdx, rows) == cudaSuccess && bl_alloc(&h->dIdxI, rows) == cudaSuccess && bl_alloc(&h->dLen, n_items) == cudaSuccess;
    ok &= bl_alloc(&h->dSim, rows) == cudaSuccess && bl_alloc(&h->dSimI, rows) == cudaSuccess;
  } else if (store == BL_STORE_POP) {
    ok &= bl_alloc(&h->dPop, n_items) == cudaSuccess && bl_alloc(&h->dTopS, h->n_keep) == cudaSuccess && bl_alloc(&h->dTop, h->n_keep) == cudaSuccess;
  }
  if (!ok) return bail("device allocation failed");
  *out = h;
  return G4R_OK;
}

// device buffers of one call, freed on every return path
struct BlBufs {
  std::vector<void*> p;
  template <class T> cudaError_t take(T** q, size_t n) { cudaError_t e = bl_alloc(q, n); if (e == cudaSuccess) p.push_back(*q); else *q = nullptr; return e; }
  template <class T> cudaError_t put(const T** q, const T* host, size_t n, cudaStream_t st) {
    T* d = nullptr;
    cudaError_t e = take(&d, n);
    *q = d;
    return (e != cudaSuccess || n == 0) ? e : cudaMemcpyAsync(d, host, n * sizeof(T), cudaMemcpyHostToDevice, st);
  }
  ~BlBufs() { for (void* q : p) cudaFree(q); }
};

// one g4r_bl_evaluate call after its argument checks: the counted events and the candidates on the host, their device copies, the
// outputs every kind's ranking fills (counts [2 x n_ev], lists [n_ev x k]) and the owner of the call's device buffers
struct BlCall {
  const int32_t* items; int64_t n_events; const int64_t* off; int64_t n_sessions; const int32_t* n_history;
  int mode, k; bool exclude;
  std::vector<int64_t> ev0;                             // counted events before each session [n_sessions + 1]
  int64_t n_ev;
  std::vector<int> mult, cdist;                         // candidates: multiplicities [n_items], distinct ascending (empty: every item)
  long long wtot;
  BlBufs bb;
  const int *d_items = nullptr, *d_nh = nullptr, *d_mult = nullptr, *d_cdist = nullptr;
  const int64_t *d_off = nullptr, *d_ev0 = nullptr;
  int *counts = nullptr, *out_items = nullptr;
  double* out_scores = nullptr;
  // the call's part of k_bl_rank's and k_sknn_rank's arguments
  BlEvalDev bl(int n_items) const {
    BlEvalDev d{};
    d.n_items = n_items; d.mode = mode; d.k = k; d.exclude = exclude; d.wtot = wtot;
    d.items = d_items; d.off = d_off; d.nh = d_nh; d.ev0 = d_ev0;
    d.mult = d_mult; d.cdist = d_cdist; d.n_cdist = (int)cdist.size();
    d.counts = counts; d.out_items = out_items; d.out_scores = out_scores;
    return d;
  }
};

// the counted events before each session, ev0 [n_sessions + 1]: a session counts its events after the first max(n_history, 1)
static int bl_counted(g4r_baselines* h, const char* fn, const int64_t* off, int64_t n_sessions, const int32_t* n_history, std::vector<int64_t>& ev0) {
  ev0.assign(n_sessions + 1, 0);
  for (int64_t s = 0; s < n_sessions; s++) {
    const int64_t len = off[s + 1] - off[s], hs = n_history ? n_history[s] : 0;
    if (hs < 0 || hs > len) FAIL(G4R_ERR_INVALID, std::string(fn) + ": n_history entry out of range");
    ev0[s + 1] = ev0[s] + std::max<int64_t>(0, len - std::max<int64_t>(hs, 1));
  }
  return G4R_OK;
}

static bool bl_offsets_ok(const int64_t* off, int64_t n_sessions, int64_t n_events) {
  if (off[0] != 0 || off[n_sessions] != n_events) return false;
  for (int64_t s = 0; s < n_sessions; s++) if (off[s + 1] < off[s]) return false;
  return true;
}

static cudaError_t bl_sort_rows(g4r_baselines* h) {
  k_knn_by_index<<<h->n_items, KF_THREADS, 0, h->stream>>>(h->dIdx, h->dSim, h->dLen, h->n_keep, h->dIdxI, h->dSimI);
  return cudaGetLastError();
}

// the row fits (ItemKNN here, SR and AR in g4r_rules.cuh): resident CTAs, each with a dense slice of n_items accumulators of
// acc_size bytes, touched columns and values, within KF_SCRATCH
static int bl_fit_grid(const g4r_baselines* h, size_t acc_size, size_t* scratch_bytes) {
  const size_t per_cta = (size_t)h->n_items * (acc_size + sizeof(int) + sizeof(double));
  const int grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)4 * h->n_sm, KF_SCRATCH / per_cta));
  if (scratch_bytes) *scratch_bytes = per_cta * grid;
  return grid;
}

// exclusive scan out[0 .. n] of in[0 .. n); tot holds (n + SCAN_B - 1) / SCAN_B block totals
static cudaError_t bl_scan(const long long* in, int64_t n, long long* out, long long* tot, cudaStream_t st) {
  const int64_t nb = (n + SCAN_B - 1) / SCAN_B;
  if (!nb) return cudaMemsetAsync(out, 0, sizeof(long long), st);
  k_scan_block<<<(unsigned)nb, SCAN_B, 0, st>>>(in, n, out, tot);
  k_scan_tot<<<1, 1, 0, st>>>(tot, nb);
  k_scan_add<<<(unsigned)nb, SCAN_B, 0, st>>>(out, n, tot);
  return cudaSuccess;
}

// the rows 0 .. n - 1 by decreasing pair work: the work buckets (bkt [65], zeroed) into order [n]
static void bl_row_order(const unsigned long long* work, int n, unsigned* bkt, int* order, cudaStream_t st) {
  const unsigned g = (unsigned)((n + 255) / 256);
  k_kp_bucket_count<<<g, 256, 0, st>>>(work, n, bkt);
  k_kp_bucket_start<<<1, 1, 0, st>>>(bkt);
  k_kp_bucket_place<<<g, 256, 0, st>>>(work, n, bkt, order);
}

// the end of a row fit, after its k_*_fit launch: the rows by index, the end event, the pair work and the device time since ev0
static int bl_fit_end(g4r_baselines* h, const unsigned long long* pairs, int64_t* pair_work, float* device_ms) {
  CK(bl_sort_rows(h));
  CK(cudaEventRecord(h->ev1, h->stream));
  unsigned long long hp = 0;
  CK(cudaMemcpyAsync(&hp, pairs, sizeof(hp), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (device_ms) CK(cudaEventElapsedTime(device_ms, h->ev0, h->ev1));
  if (pair_work) *pair_work = (int64_t)hp;
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_knn_fit(g4r_baselines* h, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_events,
                              const double* a, const double* b, int64_t* pair_work, size_t* scratch_bytes, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_ITEMKNN) FAIL(G4R_ERR_STATE, "g4r_bl_knn_fit: the handle is not an ItemKNN");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || !a || !b)
    FAIL(G4R_ERR_INVALID, "g4r_bl_knn_fit: null or negative argument");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_knn_fit: session offsets must rise from 0 to n_events");
  const int NI = h->n_items, K = h->n_keep;
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_knn_fit: item index out of range");
  for (int i = 0; i < NI; i++)
    if (!(a[i] >= 0.0 && a[i] < INFINITY && b[i] >= 0.0 && b[i] < INFINITY)) FAIL(G4R_ERR_INVALID, "g4r_bl_knn_fit: the norm factors must be finite and >= 0");
  if (n_sessions > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_knn_fit: more than 2^31 - 1 sessions");
  int64_t max_len = 0;
  for (int64_t s = 0; s < n_sessions; s++) max_len = std::max(max_len, session_offsets[s + 1] - session_offsets[s]);
  const int grid = bl_fit_grid(h, sizeof(unsigned), scratch_bytes);
  int cap = 1;                                         // long sessions: one padded session per CTA of k_kp_sort_long
  while (cap < max_len) cap <<= 1;
  const int grid_long = max_len > KP_SHORT ? (int)std::max<size_t>(1, std::min<size_t>((size_t)2 * h->n_sm, ((size_t)256 << 20) / ((size_t)cap * 4))) : 0;
  const int64_t S = n_sessions, E = n_events;
  const unsigned gs = (unsigned)((S + 7) / 8);
  const int64_t nbS = (S + SCAN_B - 1) / SCAN_B, nbI = (NI + SCAN_B - 1) / SCAN_B;
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  BlBufs bb;
  KnnFitDev d{};
  const int* dItems = nullptr; const int64_t* dOff = nullptr;
  int *srt, *long_list, *n_long, *scratch = nullptr, *s_item, *s_mult, *i_sess, *i_mult, *order, *next;
  long long *s_cnt, *s_off, *i_off, *tot;
  unsigned long long *i_cnt, *work, *pairs;
  unsigned *i_fill, *bkt;
  CK(bb.put(&dItems, items, E, st));
  CK(bb.put(&dOff, session_offsets, S + 1, st));
  CK(bb.put(&d.a, a, NI, st));
  CK(bb.put(&d.b, b, NI, st));
  CK(bb.take(&srt, E)); CK(bb.take(&long_list, S)); CK(bb.take(&n_long, 1));
  if (grid_long) CK(bb.take(&scratch, (size_t)cap * grid_long));
  CK(bb.take(&s_cnt, S)); CK(bb.take(&s_off, S + 1)); CK(bb.take(&tot, std::max(nbS, nbI)));
  CK(bb.take(&s_item, E)); CK(bb.take(&s_mult, E)); CK(bb.take(&i_sess, E)); CK(bb.take(&i_mult, E));
  CK(bb.take(&i_cnt, NI)); CK(bb.take(&work, NI)); CK(bb.take(&pairs, 1)); CK(bb.take(&i_off, NI + 1));
  CK(bb.take(&i_fill, NI)); CK(bb.take(&bkt, 65)); CK(bb.take(&order, NI)); CK(bb.take(&next, 1));
  CK(bb.take(&d.acc, (size_t)NI * grid));
  CK(bb.take(&d.touched, (size_t)NI * grid));
  CK(bb.take(&d.sims, (size_t)NI * grid));
  CK(cudaMemsetAsync(n_long, 0, sizeof(int), st));
  CK(cudaMemsetAsync(i_cnt, 0, NI * sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(work, 0, NI * sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(pairs, 0, sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(i_fill, 0, NI * sizeof(unsigned), st));
  CK(cudaMemsetAsync(bkt, 0, 65 * sizeof(unsigned), st));
  CK(cudaMemsetAsync(next, 0, sizeof(int), st));
  CK(cudaMemsetAsync(d.acc, 0, (size_t)NI * grid * sizeof(unsigned), st));
  h->ready = false;
  // everything from here to ev1 runs on the device without a host round trip: the derivation of the fit's inputs, the fit and
  // the rows by index
  CK(cudaEventRecord(h->ev0, st));
  if (S > 0) {
    k_kp_sort_short<<<gs, 256, 0, st>>>(dOff, S, dItems, srt, long_list, n_long);
    if (grid_long) k_kp_sort_long<<<grid_long, KF_THREADS, 0, st>>>(dOff, dItems, srt, long_list, n_long, scratch, cap);
    k_kp_count<<<gs, 256, 0, st>>>(dOff, S, srt, s_cnt);
  }
  CK(bl_scan(s_cnt, S, s_off, tot, st));
  if (S > 0) k_kp_emit<<<gs, 256, 0, st>>>(dOff, S, srt, (const int64_t*)s_off, s_item, s_mult, i_cnt, work, pairs);
  CK(bl_scan((const long long*)i_cnt, NI, i_off, tot, st));
  if (S > 0) k_kp_occ<<<gs, 256, 0, st>>>((const int64_t*)s_off, S, s_item, s_mult, (const int64_t*)i_off, i_fill, i_sess, i_mult);
  bl_row_order(work, NI, bkt, order, st);
  d.s_off = (const int64_t*)s_off; d.s_item = s_item; d.i_off = (const int64_t*)i_off; d.i_sess = i_sess; d.i_mult = i_mult;
  d.order = order; d.next = next; d.n_items = NI; d.n_keep = K;
  d.out_idx = h->dIdx; d.out_sim = h->dSim; d.out_len = h->dLen;
  k_knn_fit<<<grid, KF_THREADS, 0, st>>>(d);
  return bl_fit_end(h, pairs, pair_work, device_ms);
}

extern "C" int g4r_bl_set_pop(g4r_baselines* h, const double* scores, int64_t n) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_POP && h->kind != BL_SESSIONPOP) FAIL(G4R_ERR_STATE, "g4r_bl_set_pop: the handle is not a Pop / SessionPop");
  if (!scores || n != h->n_items) FAIL(G4R_ERR_INVALID, "g4r_bl_set_pop: need n_items scores");
  std::vector<int> top;
  for (int64_t i = 0; i < n; i++) {
    if (!(scores[i] >= 0.0 && scores[i] < INFINITY)) FAIL(G4R_ERR_INVALID, "g4r_bl_set_pop: scores must be finite and >= 0");
    if (scores[i] > 0.0) top.push_back((int)i);
  }
  if ((int64_t)top.size() > h->n_keep) FAIL(G4R_ERR_INVALID, "g4r_bl_set_pop: more positive scores than top_n");
  std::stable_sort(top.begin(), top.end(), [&](int x, int y) { return scores[x] > scores[y]; });
  std::vector<double> topS(top.size());
  for (size_t r = 0; r < top.size(); r++) topS[r] = scores[top[r]];
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(h->dPop, scores, n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  if (!top.empty()) {
    CK(cudaMemcpyAsync(h->dTop, top.data(), top.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->dTopS, topS.data(), top.size() * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  h->hTop = top;
  h->hPop.assign(scores, scores + n);
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_rows_export(g4r_baselines* h, int32_t* idx, double* sim, int32_t* len) {
  if (!h) return G4R_ERR_INVALID;
  if (!bl_has_rows(h->kind) || !h->ready) FAIL(G4R_ERR_STATE, "g4r_bl_rows_export: no fitted ItemKNN, SR or AR rows");
  if (!idx || !sim || !len) FAIL(G4R_ERR_INVALID, "g4r_bl_rows_export: null argument");
  const size_t rows = (size_t)h->n_items * h->n_keep;
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(idx, h->dIdx, rows * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(sim, h->dSim, rows * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(len, h->dLen, h->n_items * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

extern "C" int g4r_bl_rows_import(g4r_baselines* h, const int32_t* idx, const double* sim, const int32_t* len) {
  if (!h) return G4R_ERR_INVALID;
  if (!bl_has_rows(h->kind)) FAIL(G4R_ERR_STATE, "g4r_bl_rows_import: the handle is not an ItemKNN, SR or AR");
  if (!idx || !sim || !len) FAIL(G4R_ERR_INVALID, "g4r_bl_rows_import: null argument");
  const int NI = h->n_items, K = h->n_keep;
  std::vector<int> seen(NI, -1);                        // seen[j] == i: j is already in row i
  for (int i = 0; i < NI; i++) {
    if (len[i] < 0 || len[i] > K) FAIL(G4R_ERR_INVALID, "g4r_bl_rows_import: row length out of range");
    for (int q = 0; q < len[i]; q++) {
      const int j = idx[(size_t)i * K + q];
      const double v = sim[(size_t)i * K + q];
      if (j < 0 || j >= NI || j == i) FAIL(G4R_ERR_INDEX, "g4r_bl_rows_import: item index out of range");
      if (seen[j] == i) FAIL(G4R_ERR_INVALID, "g4r_bl_rows_import: an item occurs twice in a row");
      seen[j] = i;
      if (!(v > 0.0 && v < INFINITY)) FAIL(G4R_ERR_INVALID, "g4r_bl_rows_import: kept sims must be positive and finite");
      if (q > 0 && !(sim[(size_t)i * K + q - 1] > v || (sim[(size_t)i * K + q - 1] == v && idx[(size_t)i * K + q - 1] < j)))
        FAIL(G4R_ERR_INVALID, "g4r_bl_rows_import: a row must be in (sim desc, index asc) order");
    }
  }
  const size_t rows = (size_t)NI * K;
  cudaSetDevice(h->device);
  h->ready = false;
  CK(cudaMemcpyAsync(h->dIdx, idx, rows * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->dSim, sim, rows * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->dLen, len, NI * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CK(bl_sort_rows(h));
  CK(cudaStreamSynchronize(h->stream));
  h->ready = true;
  return G4R_OK;
}

// Pop, SessionPop, ItemKNN, SR and AR: k_bl_rank, warp per session (SR and AR rank as ItemKNN)
static int bl_rank_list(g4r_baselines* h, BlCall& c) {
  // competitor weights of the Pop list: prefix sums along (score desc, index asc)
  std::vector<long long> topW(h->hTop.size() + 1, 0);
  for (size_t r = 0; r < h->hTop.size(); r++) topW[r + 1] = topW[r] + (c.mult.empty() ? 1 : c.mult[h->hTop[r]]);
  cudaStream_t st = h->stream;
  BlEvalDev d = c.bl(h->n_items);
  d.K = h->n_keep; d.n_top = (int)h->hTop.size();
  CK(c.bb.take(&d.pl_item, c.n_events));
  CK(c.bb.take(&d.pl_cnt, c.n_events));
  CK(c.bb.put(&d.topW, topW.data(), topW.size(), st));
  d.rIdx = h->dIdx; d.rSim = h->dSim; d.rLen = h->dLen; d.rIdxI = h->dIdxI; d.rSimI = h->dSimI;
  d.pop = h->dPop; d.top = h->dTop; d.topS = h->dTopS;
  if (c.n_sessions > 0) {
    const unsigned grid = (unsigned)((c.n_sessions + 7) / 8);
    using Fn = void (*)(BlEvalDev, int64_t);
    static const Fn fns[3][2] = {{k_bl_rank<BL_POP, false>, k_bl_rank<BL_POP, true>},
                                 {k_bl_rank<BL_SESSIONPOP, false>, k_bl_rank<BL_SESSIONPOP, true>},
                                 {k_bl_rank<BL_ITEMKNN, false>, k_bl_rank<BL_ITEMKNN, true>}};
    fns[bl_has_rows(h->kind) ? BL_ITEMKNN : h->kind][c.k > 0]<<<grid, 256, 0, st>>>(d, c.n_sessions);
    CK(cudaGetLastError());
  }
  return G4R_OK;
}

extern "C" int g4r_bl_evaluate(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                               const int32_t* n_history, int32_t mode, const int32_t* cut_off, int32_t n_cut, const int32_t* cand,
                               int64_t n_cand, int32_t exclude_seen, int32_t k, double* recall_sum, double* mrr_sum, int64_t* n_counted,
                               int32_t* out_counts, int32_t* out_items, double* out_scores) {
  if (!h) return G4R_ERR_INVALID;
  if (!h->ready) FAIL(G4R_ERR_STATE, "g4r_bl_evaluate: the baseline is not fitted");
  if (h->kind == BL_VSTAN && !h->vs_set) FAIL(G4R_ERR_STATE, "g4r_bl_evaluate: the VSTAN settings are not set since the last fit (g4r_bl_vstan_set)");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || !cut_off || n_cut < 1 || n_cut > 64 ||
      !recall_sum || !mrr_sum || n_cand < 0 || n_cand > INT32_MAX || (n_cand > 0 && !cand))
    FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: null or out-of-range argument");
  if (mode < 0 || mode > 3) FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: mode must be 0 .. 3");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: session offsets must rise from 0 to n_events");
  const int NI = h->n_items;
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_evaluate: item index out of range");
  BlCall c{items, n_events, session_offsets, n_sessions, n_history, mode, k, exclude_seen != 0};
  c.wtot = NI;
  if (n_cand > 0) {
    c.mult.assign(NI, 0);
    for (int64_t q = 0; q < n_cand; q++) {
      if (cand[q] < 0 || cand[q] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_evaluate: candidate item index out of range");
      if (c.mult[cand[q]]++ == 0) c.cdist.push_back(cand[q]);
    }
    std::sort(c.cdist.begin(), c.cdist.end());
    c.wtot = n_cand;
  }
  const int n_distinct = n_cand > 0 ? (int)c.cdist.size() : NI;
  if (k < 0 || k > std::min(n_distinct, 1024) || (k > 0 && (!out_items || !out_scores)))
    FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: k must be in 0 .. min(distinct candidates, 1024), with output lists when k > 0");
  int rc = bl_counted(h, "g4r_bl_evaluate", session_offsets, n_sessions, n_history, c.ev0);
  if (rc) return rc;
  const int64_t n_ev = c.n_ev = c.ev0[n_sessions];
  if (n_ev > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: more than 2^31 - 1 counted events");
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  CK(c.bb.put(&c.d_items, items, n_events, st));
  CK(c.bb.put(&c.d_off, session_offsets, n_sessions + 1, st));
  if (n_history) CK(c.bb.put(&c.d_nh, n_history, n_sessions, st));
  CK(c.bb.put(&c.d_ev0, c.ev0.data(), n_sessions + 1, st));
  if (n_cand > 0) {
    CK(c.bb.put(&c.d_mult, c.mult.data(), c.mult.size(), st));
    CK(c.bb.put(&c.d_cdist, c.cdist.data(), c.cdist.size(), st));
  }
  CK(c.bb.take(&c.counts, (size_t)2 * n_ev));
  if (k) { CK(c.bb.take(&c.out_items, (size_t)n_ev * k)); CK(c.bb.take(&c.out_scores, (size_t)n_ev * k)); }
  rc = BL_KINDS[h->kind].rank(h, c);
  if (rc) return rc;
  // every kind: Recall / MRR from the counts, and the outputs
  const int* dCut = nullptr; double* dSums = nullptr;
  CK(c.bb.put(&dCut, cut_off, n_cut, st));
  CK(c.bb.take(&dSums, 128));
  k_bl_sums<<<1, 1024, 0, st>>>(c.counts, n_ev, dCut, n_cut, mode, dSums);
  CK(cudaGetLastError());
  std::vector<double> sums(2 * n_cut);
  CK(cudaMemcpyAsync(sums.data(), dSums, 2 * n_cut * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out_counts && n_ev) CK(cudaMemcpyAsync(out_counts, c.counts, (size_t)2 * n_ev * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (k && n_ev) {
    CK(cudaMemcpyAsync(out_items, c.out_items, (size_t)n_ev * k * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(out_scores, c.out_scores, (size_t)n_ev * k * sizeof(double), cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));
  for (int q = 0; q < n_cut; q++) { recall_sum[q] = sums[q]; mrr_sum[q] = sums[n_cut + q]; }
  if (n_counted) *n_counted = n_ev;
  return G4R_OK;
}
