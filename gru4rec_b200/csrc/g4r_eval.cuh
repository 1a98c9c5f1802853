// g4r_eval.cuh -- scoring path: evaluate_gpu's compiled function (evaluation.py:57-76) and predict
// (gru4rec.py:699-710).  Full-catalogue scores are never materialised for evaluation: each CTA scores a tile of
// consecutive items against all lanes and counts how many beat / tie the lane's target score.
// Included at the end of g4r_lib.cu (uses its handle type and helper macros).
#pragma once
#include "g4r_seen.cuh"
#include "g4r_eval_tc.cuh"

constexpr int EV_IT = 64;     // items per CTA tile
constexpr int EV_TB = 32;     // lanes per row tile
constexpr int EV_KT = 128;    // feature slab
constexpr int EV_LDS = EV_KT + 4;
constexpr int EV_THREADS = 256;

// mode 'tiebreaking' (evaluation.py:55,65): yhat += U(0,1) * 1e-10 before the standard ranking.  The reference draws the noise
// from Theano's MRG stream (not reproducible offline); here it is a counter hash of (evaluation step, lane, score column), so
// the target's own column carries the same noise in the target score and in the tile and never beats itself.
__device__ __forceinline__ float tie_noise(unsigned int seed, int s, int b, unsigned int col) {
  unsigned int k = mix32(seed ^ (0x9E3779B9U * (unsigned int)(s + 1)));
  k = mix32(k + (unsigned int)b * 0x85EBCA6BU);
  return (float)(mix32(k + col) >> 8) * (1.0f / 16777216.0f) * 1e-10f;
}

// fp32 score y_b . Wy[item] + By[item] of one (lane, item): the sequential k order of the tile loop (ev_tiles), so bitwise equal
// to the tile's score
__device__ __forceinline__ float ev_score_fp32(const ModelDev& md, int b, int item) {
  const float* yr = md.layer[md.n_layers - 1].y + (size_t)b * md.ldL;
  const float* wr = md.Wy + (size_t)item * md.ldL;
  float a = 0.f;
#pragma unroll 8
  for (int c4 = 0; c4 < md.ldL / 4; c4++) {          // loads batched by the unroll, the fma chain keeps its order
    const float4 y = ld4(yr + c4 * 4), w = ld4(wr + c4 * 4);
    a = fmaf(y.x, w.x, a); a = fmaf(y.y, w.y, a); a = fmaf(y.z, w.z, a); a = fmaf(y.w, w.w, a);
  }
  return a + md.By[item];
}

// item at position pos of a tile sweep over `subset` (nullptr: item pos)
__device__ __forceinline__ int ev_item(const int* __restrict__ subset, int pos) { return subset ? subset[pos] : pos; }

// fp32 FFMA tiles (k_eval_score, k_topk_fp32): the CTA scores positions i0 .. i0 + ni - 1 (item ev_item(subset, pos)) against
// every lane, in row blocks of EV_TB lanes.  Lane l of warp w accumulates lane b0 + l x position i0 + w + 8 q in acc[q], one
// sequential fma chain over k.  The Wy rows are staged once when ldL <= EV_KT, else per EV_KT-column slab together with Y.
// smem: [EV_TB][EV_LDS] Y, then [EV_IT][EV_LDS] Wy rows (EV_TILE_FLOATS).  epi(b0, acc): after every row block, on every thread.
constexpr int EV_TILE_FLOATS = (EV_TB + EV_IT) * EV_LDS;
template <class Epi>
__device__ __forceinline__ void ev_tiles(const ModelDev& md, float* smem, int M, int i0, int ni, const int* __restrict__ subset, Epi&& epi) {
  float* sY = smem;                        // [EV_TB][EV_LDS]
  float* sW = sY + EV_TB * EV_LDS;         // [EV_IT][EV_LDS]
  const int ldL = md.ldL;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* Y = md.layer[md.n_layers - 1].y;
  const bool hoist = ldL <= EV_KT;
  if (hoist) {
    const int kw = ldL / 4;
    for (int i = tid; i < EV_IT * kw; i += EV_THREADS) {
      const int rr = i / kw, c4 = i % kw;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rr < ni) v = ld4(md.Wy + (size_t)ev_item(subset, i0 + rr) * ldL + c4 * 4);
      st4(sW + rr * EV_LDS + c4 * 4, v);
    }
  }
  for (int b0 = 0; b0 < M; b0 += EV_TB) {
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; q++) acc[q] = 0.f;
    for (int k0 = 0; k0 < ldL; k0 += EV_KT) {
      const int kw = min(EV_KT, ldL - k0) / 4;
      __syncthreads();
      for (int i = tid; i < EV_TB * kw; i += EV_THREADS) {
        const int rr = i / kw, c4 = i % kw;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b0 + rr < M) v = ld4(Y + (size_t)(b0 + rr) * ldL + k0 + c4 * 4);
        st4(sY + rr * EV_LDS + c4 * 4, v);
      }
      if (!hoist) {
        for (int i = tid; i < EV_IT * kw; i += EV_THREADS) {
          const int rr = i / kw, c4 = i % kw;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (rr < ni) v = ld4(md.Wy + (size_t)ev_item(subset, i0 + rr) * ldL + k0 + c4 * 4);
          st4(sW + rr * EV_LDS + c4 * 4, v);
        }
      }
      __syncthreads();
      const float* yr = sY + lane * EV_LDS;
      for (int c4 = 0; c4 < kw; c4++) {
        const float4 y = ld4(yr + c4 * 4);
#pragma unroll
        for (int q = 0; q < 8; q++) {
          const float4 w = ld4(sW + (warp + 8 * q) * EV_LDS + c4 * 4);
          acc[q] = fmaf(y.x, w.x, acc[q]); acc[q] = fmaf(y.y, w.y, acc[q]); acc[q] = fmaf(y.z, w.z, acc[q]); acc[q] = fmaf(y.w, w.w, acc[q]);
        }
      }
    }
    epi(b0, acc);
  }
}

// target score of every lane, computed with the same sequential k order as the tile kernel (bitwise equal); SEEN: also adds the
// lane's input to its seen list (seen_insert) and flags the lanes whose target is in it (sd.miss).  KEY (ranking blocks of
// g4r_history.cuh): row b's tiebreaking noise is keyed by the (step, lane) pair key[2b], key[2b + 1] it was enqueued from
template <bool SEEN = false, bool KEY = false>
__global__ void __launch_bounds__(128) k_eval_tgt(int slot, int s, float* tgt, int* cnt, unsigned int tie, int subset_mode, int lohi_stride,
                                                  SeenDev sd = SeenDev{}, const int* __restrict__ key = nullptr) {
  const ModelDev& md = MD;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int M = md.wM[s];
  if (b >= M) return;
  const int item = md.wY[(size_t)s * md.B + b];
  float sc = ev_score_fp32(md, b, item);
  const float pre = sc;
  if (md.fact.kind <= G4R_ACT_SELU) sc = act_fwd(md.fact, sc);
  if (lohi_stride > 0) {      // tensor-core ranking: the two pre-activation thresholds of this lane (g4r_eval_tc.cuh)
    float lo, hi;
    tc_thresholds(md.fact, md.fact.kind <= G4R_ACT_SELU, sc, pre, lo, hi);
    tgt[lohi_stride + b] = lo; tgt[2 * lohi_stride + b] = hi;
  }
  if (tie) {
    const int ks = KEY ? key[2 * b] : s, kb = KEY ? key[2 * b + 1] : b;
    sc += tie_noise(tie, ks, kb, subset_mode ? 0x40000000U + (unsigned int)kb : (unsigned int)item);
  }
  tgt[b] = sc;
  cnt[b * 2 + 0] = 0; cnt[b * 2 + 1] = 0;
  if (SEEN) sd.miss[b] = seen_insert(md, sd, s, b, item) ? 1 : 0;
}

// Competitors: `subset` (evaluate_gpu(items=...), evaluation.py:52-56) lists the n_cand items that compete instead of the catalogue;
// without a subset, n_cand > 0 scores the leading items 0 .. n_cand - 1 and 0 the catalogue.  WRITE: out[b * n_comp + pos] = score.
// SEEN (counting only): an item on the lane's seen list is never compared -- a bit per held position, set from the list (a walk
// of the list's items inside the tile for the catalogue, a binary search per position for a subset, whose every occurrence of a
// seen item goes).  KEY: tiebreaking noise keyed per row as in k_eval_tgt<SEEN, true>
template <bool WRITE, bool SEEN = false, bool KEY = false>
__global__ void __launch_bounds__(EV_THREADS) k_eval_score(int slot, int s, const float* __restrict__ tgt, int* cnt, float* out,
                                                           const int* __restrict__ subset, int n_cand, unsigned int tie = 0u,
                                                           SeenDev sd = SeenDev{}, const int* __restrict__ key = nullptr) {
  const ModelDev& md = MD;
  extern __shared__ __align__(16) float smem[];
  int* sCnt = reinterpret_cast<int*>(smem + EV_TILE_FLOATS);   // [EV_TB][2]
  const int M = md.wM[s];
  const int I = n_cand > 0 ? n_cand : md.n_items;
  const int i0 = blockIdx.x * EV_IT;
  const int ni = min(EV_IT, I - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < EV_TB * 2) sCnt[tid] = 0;
  ev_tiles(md, smem, M, i0, ni, subset, [&](int b0, const float (&acc)[8]) {
    const int b = b0 + lane;
    if (b < M) {
      int gt = 0, eq = 0;
      const float t = WRITE ? 0.f : tgt[b];
      unsigned int xq = 0u;                      // SEEN: held positions i0 + warp + 8 q whose item is seen
      if (SEEN) {
        const int sl = md.wSlot[(size_t)s * md.B + b], n = sd.n[sl];
        const int* l = sd.list + (size_t)sl * sd.cap;
        if (subset) {
#pragma unroll
          for (int q = 0; q < 8; q++) if (warp + 8 * q < ni && sorted_has(l, n, subset[i0 + warp + 8 * q])) xq |= 1u << q;
        } else {
          for (int p = sorted_lb(l, n, i0); p < n && l[p] < i0 + ni; p++) {
            const int rel = l[p] - i0;
            if ((rel & 7) == warp) xq |= 1u << (rel >> 3);
          }
        }
      }
      float* orow = WRITE ? out + (size_t)b * I + i0 + warp : nullptr;   // one row pointer keeps the kernel free of spills
      const int ks = (KEY && tie) ? key[2 * b] : s, kb = (KEY && tie) ? key[2 * b + 1] : b;
#pragma unroll
      for (int q = 0; q < 8; q++) {
        const int it = i0 + warp + 8 * q;
        if (warp + 8 * q < ni && !((xq >> q) & 1u)) {
          float sc = acc[q] + md.By[ev_item(subset, it)];
          if (WRITE) orow[8 * q] = sc;
          else {
            if (md.fact.kind <= G4R_ACT_SELU) sc = act_fwd(md.fact, sc);
            if (tie) sc += tie_noise(tie, ks, kb, (unsigned int)it);
            gt += sc > t; eq += sc == t;
          }
        }
      }
      if (!WRITE) { if (gt) atomicAdd(&sCnt[lane * 2], gt); if (eq) atomicAdd(&sCnt[lane * 2 + 1], eq); }
    }
    __syncthreads();
    if (!WRITE && tid < EV_TB * 2) {             // flush and clear for the next row block (the tile loop syncs before its epilogue)
      const int bb = b0 + tid / 2;
      if (bb < M && sCnt[tid]) atomicAdd(&cnt[bb * 2 + (tid & 1)], sCnt[tid]);
      sCnt[tid] = 0;
    }
  });
}
static size_t eval_smem_bytes() { return (size_t)EV_TILE_FLOATS * sizeof(float) + EV_TB * 2 * sizeof(int) + 64; }

// ranks + per-cutoff sums (evaluation.py:60-75), accumulated in double on the device; SEEN: a lane flagged in miss (target
// already seen) is a miss, rank +inf, whatever its counts
template <bool SEEN = false>
__global__ void __launch_bounds__(256) k_eval_rank(int slot, int s, const int* cnt, const int* cut, int n_cut, int mode, double* sums,
                                                   const int* __restrict__ miss = nullptr) {
  const ModelDev& md = MD;
  if (blockIdx.x != 0) return;
  const int M = md.wM[s];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ double red[8][2];
  // one cut-off at a time: lanes strided over the threads, double sums reduced in a fixed order (deterministic)
  for (int j = 0; j < n_cut; j++) {
    double hit = 0.0, rr = 0.0;
    for (int b = tid; b < M; b += blockDim.x) {
      if (SEEN && miss[b]) continue;
      const int gt = cnt[b * 2], eq = cnt[b * 2 + 1];
      double rank;
      if (mode == 1) rank = (double)(gt + eq);
      else if (mode == 2) rank = (double)gt + 0.5 * (double)(eq - 1) + 1.0;
      else rank = (double)(gt + 1);
      if (rank <= (double)cut[j]) { hit += 1.0; rr += 1.0 / rank; }
    }
    for (int o = 16; o > 0; o >>= 1) { hit += __shfl_xor_sync(0xffffffffu, hit, o); rr += __shfl_xor_sync(0xffffffffu, rr, o); }
    __syncthreads();
    if (lane == 0) { red[warp][0] = hit; red[warp][1] = rr; }
    __syncthreads();
    if (tid == 0) {
      double h = 0.0, r = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); w++) { h += red[w][0]; r += red[w][1]; }
      sums[j] += h; sums[n_cut + j] += r;
    }
  }
}

// final activation of the predict path (gru4rec.py:499-505): elementwise, softmax, or softmax for softmax_logit
__global__ void __launch_bounds__(256) k_predict_act(int slot, float* out, int batch) {
  const ModelDev& md = MD;
  const int b = blockIdx.x;
  if (b >= batch) return;
  float* row = out + (size_t)b * md.n_items;
  const int I = md.n_items;
  __shared__ float red[32];
  if (md.fact.kind <= G4R_ACT_SELU) {
    for (int i = threadIdx.x; i < I; i += blockDim.x) row[i] = act_fwd(md.fact, row[i]);
    return;
  }
  float m = -INFINITY;
  for (int i = threadIdx.x; i < I; i += blockDim.x) m = fmaxf(m, row[i]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); w++) m = fmaxf(m, red[w]);
  __syncthreads();
  float z = 0.f;
  for (int i = threadIdx.x; i < I; i += blockDim.x) z += expf(row[i] - m);
  z = warp_sum(z);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = z;
  __syncthreads();
  z = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) z += red[w];
  for (int i = threadIdx.x; i < I; i += blockDim.x) row[i] = __fdiv_rn(expf(row[i] - m), z);
}

struct EvalCtx {
  ModelDev mde;
  int Be = 0;
  int *hX = nullptr, *hY = nullptr, *hSlot = nullptr, *hM = nullptr, *hSti = nullptr; uint8_t* hF = nullptr; uint32_t* hG = nullptr;
  int *dX = nullptr, *dY = nullptr, *dSlot = nullptr, *dM = nullptr, *dSti = nullptr; uint8_t* dF = nullptr; uint32_t* dG = nullptr;
  int* dCut = nullptr; double* dSums = nullptr; float* dOut = nullptr; size_t out_cap = 0;
  int cap = 0;
  int slot = -1;
  int* dCand = nullptr; int n_cand = 0; size_t cand_cap = 0;     // candidate subset of evaluate_gpu(items=...), item indices
  std::vector<int32_t> hCand;                                     // its host copy (the top-k filter of g4r_eval_events)
  // wgmma tiles (g4r_eval_tc.cuh): [hi | lo] TF32 operand blocks of the hidden states (per call) and of the item table, which
  // is kept between calls and tagged with the handle's wy_version it was made from
  unsigned char *dAsplit = nullptr, *dBsplit = nullptr;
  uint64_t split_version = ~0ull;
  void* topk = nullptr;                                           // TopkCtx* of g4r_predict_topk (g4r_topk.cuh)
  void* events = nullptr;                                         // EventsCtx* of g4r_eval_events (g4r_events.cuh)
  void* hist = nullptr;                                           // HistCtx* of history schedules (g4r_history.cuh)
  void* rest = nullptr;                                           // RestCtx* of g4r_eval_rest (g4r_rest.cuh)
  // exclude_seen (g4r_set_eval_exclude_seen, g4r_seen.cuh): per state slot the seen list, its length, the lanes' miss flags, and
  // the per-mini-batch CSR copy the top-k kernels of g4r_eval_events read as their exclusions
  bool seen_on = false;
  int* dSeen = nullptr; size_t seen_cap = 0;
  int *dSeenN = nullptr, *dMiss = nullptr;
  int* dSeenOff = nullptr; int* dSeenEx = nullptr; size_t seen_ex_cap = 0;
};
static void topk_release(EvalCtx& e);
static void events_release(EvalCtx& e);
static void hist_release(EvalCtx& e);
static void rest_release(EvalCtx& e);

// device buffer of at least n elements (contents not kept)
template <class T>
static cudaError_t dev_grow(T** p, size_t* cap, size_t n) {
  if (*cap >= n && *p) return cudaSuccess;
  if (*p) cudaFree(*p);
  *p = nullptr; *cap = 0;
  const cudaError_t r = cudaMalloc(p, n * sizeof(T));
  if (r == cudaSuccess) *cap = n;
  return r;
}

// Tile kind of a scoring call of `lanes` lanes against n_comp competing items: cfg.eval_tc 1 = fp32 FFMA tiles, 2 = wgmma
// 3xTF32 tiles, 0 = wgmma from 64 lanes and 2048 competitors on (the split item table is amortised over enough lanes; at one lane
// it is twice the bytes of Wy) and only when the competitors are at least a quarter of the catalogue (the wgmma tiles cover the
// whole catalogue)
static bool wgmma_tiles(const g4r_config& cfg, int lanes, int n_comp, int n_items) {
  return cfg.eval_tc == 2 || (cfg.eval_tc == 0 && lanes >= 64 && n_comp >= 2048 && 4 * (int64_t)n_comp >= n_items);
}

// operand buffers of the wgmma tiles, and the item-table split made again only if Wy / By may have changed since (wy_version)
static int tc_operands(g4r_handle* h, EvalCtx* e) {
  const int chunks = (h->md.L + 1 + TC_KC - 1) / TC_KC, tiles = (h->md.n_items + TC_N - 1) / TC_N;   // + the bias column
  if (!e->dAsplit) CK(cudaMalloc(&e->dAsplit, (size_t)((e->Be + TC_M - 1) / TC_M) * chunks * 2 * TC_A_BYTES));   // blocks of 128 lanes
  if (!e->dBsplit) CK(cudaMalloc(&e->dBsplit, (size_t)tiles * chunks * 2 * TC_B_BYTES));                         // blocks of 256 items
  if (e->split_version != h->wy_version) {
    k_tc_split<TC_N><<<dim3(tiles, chunks), 256, 0, h->stream>>>(h->md.Wy, h->md.n_items, h->md.ldL, h->md.L, e->dBsplit, chunks, h->md.By, 0.f);
    h->launches++;
    e->split_version = h->wy_version;
  }
  return G4R_OK;
}

static void eval_release(g4r_handle* h) {
  if (!h->eval_ctx) return;
  EvalCtx& e = *static_cast<EvalCtx*>(h->eval_ctx);
  topk_release(e);
  events_release(e);
  hist_release(e);
  rest_release(e);
  cudaFreeHost(e.hX); cudaFreeHost(e.hY); cudaFreeHost(e.hSlot); cudaFreeHost(e.hF); cudaFreeHost(e.hM); cudaFreeHost(e.hSti); cudaFreeHost(e.hG);
  cudaFree(e.dX); cudaFree(e.dY); cudaFree(e.dSlot); cudaFree(e.dF); cudaFree(e.dM); cudaFree(e.dSti); cudaFree(e.dG);
  cudaFree(e.dCut); cudaFree(e.dSums); if (e.dOut) cudaFree(e.dOut); if (e.dCand) cudaFree(e.dCand);
  if (e.dAsplit) cudaFree(e.dAsplit); if (e.dBsplit) cudaFree(e.dBsplit);
  for (void* p : {(void*)e.dSeen, (void*)e.dSeenN, (void*)e.dMiss, (void*)e.dSeenOff, (void*)e.dSeenEx}) if (p) cudaFree(p);
  slot_free(e.slot);
  delete static_cast<EvalCtx*>(h->eval_ctx);
  h->eval_ctx = nullptr;
}

static int eval_ctx(g4r_handle* h, EvalCtx** out) {
  if (h->eval_ctx) { *out = static_cast<EvalCtx*>(h->eval_ctx); return G4R_OK; }
  EvalCtx e;
  e.Be = h->cfg.eval_batch_size > 0 ? h->cfg.eval_batch_size : h->cfg.batch_size;
  e.cap = 512;
  const size_t nb = (size_t)e.cap * e.Be;
  CK(cudaMallocHost(&e.hX, nb * sizeof(int))); CK(cudaMallocHost(&e.hY, nb * sizeof(int))); CK(cudaMallocHost(&e.hSlot, nb * sizeof(int)));
  CK(cudaMallocHost(&e.hF, nb)); CK(cudaMallocHost(&e.hM, e.cap * sizeof(int))); CK(cudaMallocHost(&e.hSti, e.cap * sizeof(int))); CK(cudaMallocHost(&e.hG, e.cap * sizeof(uint32_t)));
  CK(cudaMalloc(&e.dX, nb * sizeof(int))); CK(cudaMalloc(&e.dY, nb * sizeof(int))); CK(cudaMalloc(&e.dSlot, nb * sizeof(int)));
  CK(cudaMalloc(&e.dF, nb)); CK(cudaMalloc(&e.dM, e.cap * sizeof(int))); CK(cudaMalloc(&e.dSti, e.cap * sizeof(int))); CK(cudaMalloc(&e.dG, e.cap * sizeof(uint32_t)));
  CK(cudaMalloc(&e.dCut, 64 * sizeof(int))); CK(cudaMalloc(&e.dSums, 128 * sizeof(double)));
  e.mde = h->md;
  e.mde.B = e.Be;
  e.mde.wX = e.dX; e.mde.wY = e.dY; e.mde.wSlot = e.dSlot; e.mde.wM = e.dM; e.mde.wSti = e.dSti; e.mde.wF = e.dF; e.mde.wG = e.dG;
  e.slot = slot_alloc();
  if (e.slot < 0) FAIL(G4R_ERR_STATE, "too many live g4r handles in this process");
  CK(slot_upload(e.slot, e.mde, h->stream));
  cudaFuncSetAttribute(k_eval_score<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eval_smem_bytes());
  cudaFuncSetAttribute(k_eval_score<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eval_smem_bytes());
  cudaFuncSetAttribute(k_eval_score<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eval_smem_bytes());
  cudaFuncSetAttribute(k_eval_score<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eval_smem_bytes());
  cudaFuncSetAttribute(k_eval_score<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eval_smem_bytes());
  if (cudaFuncSetAttribute(k_eval_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem)) != cudaSuccess) cudaGetLastError();
  if (cudaFuncSetAttribute(k_eval_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem)) != cudaSuccess) cudaGetLastError();
  h->eval_ctx = new EvalCtx(e);
  *out = static_cast<EvalCtx*>(h->eval_ctx);
  return G4R_OK;
}

// GRU forward of step s of the scoring window; Hst[li]: the hidden-state array of layer li that the staged slots address (the
// handle's lanes He, or a session table)
static int eval_forward(g4r_handle* h, EvalCtx* e, int s, float* const* Hst) {
  const ModelDev& md = e->mde;
  cudaStream_t st = h->stream;
  if (md.mode != 0) { k_gather_in<<<std::max(1, (e->Be + 7) / 8), 256, 0, st>>>(e->slot, nullptr, s, 0); h->launches++; }
  for (int li = 0; li < md.n_layers; li++) {
    const LayerDev& ly = md.layer[li];
    k_f1<<<tiles2(2 * ly.L, e->Be), GEMM_THREADS, 0, st>>>(e->slot, nullptr, s, li, Hst[li]);
    k_f2<<<tiles2(ly.L, e->Be), GEMM_THREADS, 0, st>>>(e->slot, nullptr, s, li, Hst[li], 0);
    h->launches += 2;
  }
  return G4R_OK;
}

// the staged window (w steps of e->hX .. hG, strided by the engine's scoring lanes) to the device, on the forward stream
static int eval_upload(g4r_handle* h, EvalCtx* e, int64_t w) {
  cudaStream_t st = h->stream;
  const size_t nb = (size_t)w * e->Be;
  CK(cudaMemcpyAsync(e->dX, e->hX, nb * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(e->dY, e->hY, nb * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(e->dSlot, e->hSlot, nb * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(e->dF, e->hF, nb, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(e->dM, e->hM, (size_t)w * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(e->dSti, e->hSti, (size_t)w * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(e->dG, e->hG, (size_t)w * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  return G4R_OK;
}

// What one ranking (eval_rank) ranks: the M rows of scoring descriptor `slot` at its step s -- a mini-batch of the staging window,
// or a ranking block of a history schedule (g4r_history.cuh)
struct RankUnit {
  int slot = -1, s = 0, M = 0;
  const float* y = nullptr;             // the rows' final-layer y, as the wgmma split reads them
  const int* key = nullptr;             // per-row tiebreaking keys, (step, lane) pairs (nullptr: keyed by (s, row))
  SeenDev sd;                           // exclude_seen: the lists ranked against and the rows' miss flags (list == nullptr: off)
  bool insert = false;                  // k_eval_tgt adds each row's input to sd (a mini-batch) or only reads it (a block's snapshot)
  int64_t step = 0;                     // schedule step of every row (steps == nullptr; row b is lane b) ...
  const int64_t* steps = nullptr; const int* lanes = nullptr;   // ... or of each row, and its lane (host arrays)
};

struct RestRun;

// the constants of one eval_run call, shared by every unit it ranks
struct RankConsts {
  unsigned int tie = 0u;
  bool tc_possible = false;             // the wgmma tiles are ready; a unit takes them if wgmma_tiles holds for its rows
  int n_cut = 0, mode = 0;
  bool seen = false; SeenDev sd;        // exclude_seen: the live lists of the scoring slots
  RestRun* rest = nullptr;              // g4r_eval_rest's per-unit work (g4r_rest.cuh); nullptr on the other entry points
};

// g4r_eval_events' per-event outputs (g4r_events.cuh); nullptr on g4r_eval_schedule's path
struct EventsRun;
static int events_begin(g4r_handle* h, EvalCtx* e, const g4r_schedule* s, EventsRun* ev, const SeenDev* sd);
static bool events_lists(const EventsRun* ev);      // k > 0
static int events_stage(g4r_handle* h, EvalCtx* e, EventsRun* ev, const RankUnit& u, cudaStream_t rk);
static int events_step(g4r_handle* h, EvalCtx* e, EventsRun* ev, const RankUnit& u, cudaStream_t rk);
static int events_flush(g4r_handle* h, EvalCtx* e, EventsRun* ev, cudaStream_t rk);

// history schedules (g4r_history.cuh): only the lanes flagged 4 are ranked, in blocks
struct HistCtx;
static int hist_begin(g4r_handle* h, EvalCtx* e, const g4r_schedule* s, const SeenDev* sd, HistCtx** out);
static int hist_window(g4r_handle* h, EvalCtx* e, HistCtx* c, const g4r_schedule* s, int64_t w, int64_t done, const RankConsts& cs, EventsRun* ev);

// g4r_eval_rest (g4r_rest.cuh): relevant lists and thresholds before the tiles, the multi-threshold passes after k_eval_rank
static int rest_begin(g4r_handle* h, EvalCtx* e, const g4r_schedule* s, RestRun* rr, int n_cut, bool tc);
static int rest_stage(g4r_handle* h, EvalCtx* e, RestRun* rr, const RankUnit& u, const RankConsts& cs, cudaStream_t rk);
static int rest_step(g4r_handle* h, EvalCtx* e, RestRun* rr, const RankUnit& u, const RankConsts& cs, cudaStream_t rk);
static int rest_flush(g4r_handle* h, RestRun* rr, cudaStream_t rk);

// One ranking of unit u on the ranking stream rk: the target scores (with exclude_seen, a mini-batch's seen insert, and the CSR
// exclusions of g4r_eval_events' lists), the fp32 or wgmma tiles, the per-cutoff sums, then g4r_eval_events' per-event work
// (ev != nullptr).  released (nullptr: none) is recorded once the rows' y has been read, and the forward stream waits on it.
// Everything the ranking kernels share (target scores, counters, operand blocks, metric sums) is ordered by rk itself, so the
// sums accumulate in unit order.
static int eval_rank(g4r_handle* h, EvalCtx* e, const RankUnit& u, const RankConsts& cs, EventsRun* ev, cudaStream_t rk, cudaEvent_t released) {
  const int Be = e->Be, I = h->md.n_items, M = u.M;
  const bool seen = u.sd.list != nullptr;
  const int subset_mode = e->n_cand > 0 ? 1 : 0, lohi = cs.tc_possible ? Be : 0;
  if (seen && u.insert) k_eval_tgt<true><<<(Be + 31) / 32, 32, 0, rk>>>(u.slot, u.s, h->dTgt, h->dRankCnt, cs.tie, subset_mode, lohi, u.sd);
  else if (u.key) k_eval_tgt<false, true><<<(Be + 31) / 32, 32, 0, rk>>>(u.slot, u.s, h->dTgt, h->dRankCnt, cs.tie, subset_mode, lohi, SeenDev{}, u.key);
  else k_eval_tgt<<<(Be + 31) / 32, 32, 0, rk>>>(u.slot, u.s, h->dTgt, h->dRankCnt, cs.tie, subset_mode, lohi);
  h->launches++;
  if (cs.rest) {
    int rc = rest_stage(h, e, cs.rest, u, cs, rk);     // reads the rows' y before the forward may move on
    if (rc) return rc;
  }
  if (ev) {
    if (seen && events_lists(ev)) {
      k_seen_csr<<<1, SEEN_CSR_THREADS, 0, rk>>>(u.slot, u.s, u.sd, e->dSeenOff, e->dSeenEx);
      h->launches++;
    }
    int rc = events_stage(h, e, ev, u, rk);     // saves the rows' y before the forward may move on
    if (rc) return rc;
  }
  if (cs.tc_possible && wgmma_tiles(h->cfg, M, I, I)) {
    const int tc_chunks = (h->md.L + 1 + TC_KC - 1) / TC_KC, tc_tiles = (I + TC_N - 1) / TC_N;   // + the bias column
    k_tc_split<TC_M><<<dim3((M + TC_M - 1) / TC_M, tc_chunks), 256, 0, rk>>>(u.y, M, h->md.ldL, h->md.L, e->dAsplit, tc_chunks, nullptr, 1.0f);
    if (released) CK(cudaEventRecord(released, rk));
    (seen ? k_eval_tc<true> : k_eval_tc<false>)<<<std::min(tc_tiles, h->n_sm), TC_THREADS, sizeof(TcSmem), rk>>>(u.slot, u.s, h->dTgt, Be, h->dRankCnt,
                                                                                                                 e->dAsplit, e->dBsplit, u.sd);
    h->launches += 2;
  } else {
    const int n_comp = e->n_cand > 0 ? e->n_cand : I;
    auto kern = u.key ? (seen ? k_eval_score<false, true, true> : k_eval_score<false, false, true>) : (seen ? k_eval_score<false, true> : k_eval_score<false>);
    kern<<<(n_comp + EV_IT - 1) / EV_IT, EV_THREADS, eval_smem_bytes(), rk>>>(u.slot, u.s, h->dTgt, h->dRankCnt, nullptr, e->n_cand > 0 ? e->dCand : nullptr,
                                                                              e->n_cand, cs.tie, u.sd, u.key);
    if (released) CK(cudaEventRecord(released, rk));
    h->launches++;
  }
  if (released) CK(cudaStreamWaitEvent(h->stream, released, 0));
  (seen ? k_eval_rank<true> : k_eval_rank<false>)<<<1, 256, 0, rk>>>(u.slot, u.s, h->dRankCnt, e->dCut, cs.n_cut, cs.mode, e->dSums, u.sd.miss);
  h->launches++;
  if (cs.rest) {
    int rc = rest_step(h, e, cs.rest, u, cs, rk);
    if (rc) return rc;
  }
  return ev ? events_step(h, e, ev, u, rk) : G4R_OK;
}

// the w staged mini-batches of a plain schedule (first schedule step `done`).  Two streams: the GRU forward of mini-batch i+1
// (forward stream) overlaps the ranking of mini-batch i (ranking stream), which reads the hidden output only in its first kernels
// (target scores, operand split -- or the fp32 tile kernel itself), after which the forward stream may overwrite it
static int eval_window(g4r_handle* h, EvalCtx* e, int64_t w, int64_t done, const RankConsts& cs, EventsRun* ev) {
  cudaStream_t st = h->stream, rk = h->side;
  for (int64_t i = 0; i < w; i++) {
    eval_forward(h, e, (int)i, h->He);
    CK(cudaEventRecord(h->ts_ev[0], st)); CK(cudaStreamWaitEvent(rk, h->ts_ev[0], 0));
    RankUnit u;
    u.slot = e->slot; u.s = (int)i; u.M = e->hM[i]; u.y = h->md.layer[h->md.n_layers - 1].y;
    u.sd = cs.sd; u.insert = true;     // inserts this mini-batch's inputs on the ranking stream: after i-1's ranking has read the
                                       // lists, while i+1's forward runs
    u.step = done + i;
    int rc = eval_rank(h, e, u, cs, ev, rk, h->ts_ev[1]);
    if (rc) return rc;
  }
  return G4R_OK;
}

// exclude_seen: lists of capacity cap = the schedule's longest session - 1 for every scoring slot (eval_run empties them);
// refused before any device work when B x cap x 4 bytes (B: the schedule's lanes) exceed SEEN_BYTES, the 256 MiB budget of g4r_eval_events' window
// buffers (G4R_SEEN_BUDGET in the environment lowers it, for tests)
constexpr size_t SEEN_BYTES = (size_t)256 << 20;
static int seen_begin(g4r_handle* h, EvalCtx* e, const g4r_schedule* s, bool csr, SeenDev* sd) {
  const int64_t cap = std::max<int64_t>(1, s->max_len - 1);
  size_t budget = SEEN_BYTES;
  if (const char* b = getenv("G4R_SEEN_BUDGET")) budget = std::min<size_t>(budget, (size_t)std::max(0LL, atoll(b)));
  if ((size_t)s->B * (size_t)cap * sizeof(int) > budget) {
    char msg[256];
    snprintf(msg, sizeof msg, "exclude_seen: the longest session (%lld events) needs seen lists of %d lanes x %lld items, over the %zu-byte budget",
             (long long)s->max_len, s->B, (long long)cap, budget);
    FAIL(G4R_ERR_INVALID, msg);
  }
  const size_t n = (size_t)s->B * (size_t)cap;             // state slots of the schedule: 0 .. B - 1
  CK(dev_grow(&e->dSeen, &e->seen_cap, n));
  if (!e->dSeenN) CK(cudaMalloc(&e->dSeenN, (size_t)e->Be * sizeof(int)));
  if (!e->dMiss) CK(cudaMalloc(&e->dMiss, (size_t)e->Be * sizeof(int)));
  if (csr) {
    if (!e->dSeenOff) CK(cudaMalloc(&e->dSeenOff, (size_t)(e->Be + 1) * sizeof(int)));
    CK(dev_grow(&e->dSeenEx, &e->seen_ex_cap, n));
  }
  sd->list = e->dSeen; sd->n = e->dSeenN; sd->cap = (int)cap; sd->miss = e->dMiss;
  return G4R_OK;
}

// The evaluation schedule in staging windows of e->cap mini-batches (g4r_eval_schedule); ev != nullptr adds g4r_eval_events'
// per-event work on the ranking stream, after the kernels of g4r_eval_schedule, which stay as they are and see the same step
// indices (the tiebreaking noise hashes them) whatever the per-event window
static int eval_run(g4r_handle* h, const g4r_schedule* s, const int32_t* cut_off, int32_t n_cut, int32_t mode,
                    double* recall_sum, double* mrr_sum, int64_t* n_events, EventsRun* ev, RestRun* rest = nullptr) {
  if (mode < 0 || mode > 3) FAIL(G4R_ERR_INVALID, "eval mode must be 0 (standard), 1 (conservative), 2 (median) or 3 (tiebreaking)");
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  int rc = eval_ctx(h, &e);
  if (rc) return rc;
  if (s->B > e->Be) FAIL(G4R_ERR_INVALID, "schedule batch size exceeds eval_batch_size");
  RankConsts cs;
  cs.tie = mode == 3 ? 0x5bd1e995u : 0u; cs.n_cut = n_cut; cs.mode = mode; cs.seen = e->seen_on;
  const SeenDev* sd = cs.seen ? &cs.sd : nullptr;
  if (sd) {
    rc = seen_begin(h, e, s, ev && events_lists(ev), &cs.sd);
    if (rc) return rc;
  }
  if (ev) {
    rc = events_begin(h, e, s, ev, sd);
    if (rc) return rc;
  }
  const int Be = e->Be, Bs = s->B, I = h->md.n_items;
  cudaStream_t st = h->stream;
  for (int i = 0; i < h->md.n_layers; i++) CK(cudaMemsetAsync(h->He[i], 0, (size_t)Be * h->md.layer[i].ldL * sizeof(float), st));   // gru4rec.py:731-733
  CK(cudaMemcpyAsync(e->dCut, cut_off, n_cut * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(e->dSums, 0, 128 * sizeof(double), st));
  if (sd) CK(cudaMemsetAsync(sd->n, 0, (size_t)Be * sizeof(int), st));   // every lane starts a session with the schedule
  // wgmma tiles (full-catalogue ranking of a wide batch; candidate subsets and tiebreaking take the fp32 tiles): decided once
  // with the schedule's batch, then per unit with its rows
  cs.tc_possible = e->n_cand == 0 && mode != 3 && wgmma_tiles(h->cfg, Bs, I, I);
  if (cs.tc_possible) {
    rc = tc_operands(h, e);
    if (rc) return rc;
  }
  if (rest) {
    rc = rest_begin(h, e, s, rest, n_cut, cs.tc_possible);   // its passes take the wgmma tiles where the next-item ranking would
    if (rc) return rc;
    cs.rest = rest;
  }
  HistCtx* hc = nullptr;
  if (s->hist) {
    rc = hist_begin(h, e, s, sd, &hc);
    if (rc) return rc;
  }
  int64_t done = 0;
  while (done < s->n_steps) {
    const int64_t w = std::min<int64_t>(e->cap, s->n_steps - done);
    CK(cudaStreamSynchronize(st));   // staging buffers are reused
    for (int64_t i = 0; i < w; i++) {   // the window arrays are strided by the engine's scoring lanes
      memcpy(e->hX + i * Be, s->X.data() + (done + i) * Bs, (size_t)Bs * sizeof(int));
      memcpy(e->hY + i * Be, s->Y.data() + (done + i) * Bs, (size_t)Bs * sizeof(int));
      memcpy(e->hSlot + i * Be, s->slots.data() + (done + i) * Bs, (size_t)Bs * sizeof(int));
      memcpy(e->hF + i * Be, s->F.data() + (done + i) * Bs, (size_t)Bs);
    }
    memcpy(e->hM, s->M.data() + done, (size_t)w * sizeof(int));
    for (int64_t i = 0; i < w; i++) {
      e->hSti[i] = -1; e->hG[i] = 0;
      const int M = e->hM[i];
      for (int b = 0; b < M; b++) {
        const int x = e->hX[i * Be + b], y = e->hY[i * Be + b];
        if (x < 0 || x >= I || y < 0 || y >= I) FAIL(G4R_ERR_INDEX, "Index out of bounds");
      }
    }
    rc = eval_upload(h, e, w);
    if (rc) return rc;
    rc = hc ? hist_window(h, e, hc, s, w, done, cs, ev) : eval_window(h, e, w, done, cs, ev);
    if (rc) return rc;
    if (ev) {
      rc = events_flush(h, e, ev, h->side);    // the rest of the per-event window before the staging is reused
      if (rc) return rc;
    }
    if (rest) {
      rc = rest_flush(h, rest, h->side);
      if (rc) return rc;
    }
    CK(cudaEventRecord(h->ts_ev[2], h->side)); CK(cudaStreamWaitEvent(st, h->ts_ev[2], 0));   // window complete before its staging is reused
    CK(cudaGetLastError());
    done += w;
  }
  std::vector<double> sums(128);
  CK(cudaMemcpyAsync(sums.data(), e->dSums, 128 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int j = 0; j < n_cut; j++) { recall_sum[j] = sums[j]; mrr_sum[j] = sums[n_cut + j]; }
  if (n_events) *n_events = s->n_events;
  return G4R_OK;
}

extern "C" int g4r_eval_schedule(g4r_handle* h, const g4r_schedule* s, const int32_t* cut_off, int32_t n_cut, int32_t mode,
                                 double* recall_sum, double* mrr_sum, int64_t* n_events) {
  if (!h || !s || !cut_off || n_cut <= 0 || n_cut > 64 || !recall_sum || !mrr_sum) return G4R_ERR_INVALID;
  return eval_run(h, s, cut_off, n_cut, mode, recall_sum, mrr_sum, n_events, nullptr);
}

extern "C" int g4r_eval_counts(g4r_handle* h, int32_t* out, int64_t n_lanes) {
  if (!h || !out || n_lanes < 0) return G4R_ERR_INVALID;
  const int Be = h->cfg.eval_batch_size > 0 ? h->cfg.eval_batch_size : h->cfg.batch_size;
  if (n_lanes > Be) FAIL(G4R_ERR_INVALID, "n_lanes exceeds eval_batch_size");
  cudaSetDevice(h->cfg.device);
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(out, h->dRankCnt, (size_t)n_lanes * 2 * sizeof(int), cudaMemcpyDeviceToHost));
  return G4R_OK;
}

// evaluate_gpu(exclude_seen=True): later g4r_eval_schedule / g4r_eval_events calls rank each target without the items its session
// has input so far (the current input included); a target among them is a miss (g4r_seen.cuh, DESIGN §3g)
extern "C" int g4r_set_eval_exclude_seen(g4r_handle* h, int32_t on) {
  if (!h) return G4R_ERR_INVALID;
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  int rc = eval_ctx(h, &e);
  if (rc) return rc;
  e->seen_on = on != 0;
  return G4R_OK;
}

// evaluate_gpu(items=...) (evaluation.py:52-56,84-100): the targets are ranked against this candidate list (item indices,
// duplicates allowed as in the reference) instead of the whole catalogue; n = 0 restores the full-catalogue ranking.
extern "C" int g4r_set_eval_items(g4r_handle* h, const int64_t* items, int64_t n) {
  if (!h || n < 0 || (n > 0 && !items)) return G4R_ERR_INVALID;
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  int rc = eval_ctx(h, &e);
  if (rc) return rc;
  if (n == 0) { e->n_cand = 0; return G4R_OK; }
  if (n > (int64_t)1 << 30) FAIL(G4R_ERR_INVALID, "too many candidate items");
  std::vector<int> tmp((size_t)n);
  for (int64_t i = 0; i < n; i++) {
    if (items[i] < 0 || items[i] >= h->md.n_items) FAIL(G4R_ERR_INDEX, "Index out of bounds");
    tmp[(size_t)i] = (int)items[i];
  }
  CK(dev_grow(&e->dCand, &e->cand_cap, (size_t)n));
  CK(cudaMemcpyAsync(e->dCand, tmp.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  e->n_cand = (int)n;
  e->hCand = std::move(tmp);
  return G4R_OK;
}

// the single mini-batch of a predict call (lanes 0 .. batch-1, reset_mask zeroes lanes first) staged on the scoring path; nothing
// reaches the device unless every input index is valid
static int predict_stage(g4r_handle* h, EvalCtx* e, const int32_t* X, int32_t batch, const uint8_t* reset_mask) {
  const int Be = e->Be, I = h->md.n_items;
  if (batch <= 0 || batch > Be) FAIL(G4R_ERR_INVALID, "predict batch exceeds eval_batch_size");
  for (int b = 0; b < Be; b++) {
    e->hX[b] = b < batch ? X[b] : -1; e->hY[b] = 0; e->hSlot[b] = b;
    e->hF[b] = (b < batch && reset_mask && reset_mask[b]) ? 2 : 0;
    if (b < batch && (X[b] < 0 || X[b] >= I)) FAIL(G4R_ERR_INDEX, "Index out of bounds");
  }
  e->hM[0] = batch; e->hSti[0] = -1; e->hG[0] = 0;
  return eval_upload(h, e, 1);
}

extern "C" int g4r_predict(g4r_handle* h, const int32_t* X, int32_t batch, const uint8_t* reset_mask, float* out) {
  if (!h || !X || !out) return G4R_ERR_INVALID;
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  int rc = eval_ctx(h, &e);
  if (rc) return rc;
  rc = predict_stage(h, e, X, batch, reset_mask);
  if (rc) return rc;
  const int I = h->md.n_items;
  cudaStream_t st = h->stream;
  const size_t need = (size_t)batch * I;
  CK(dev_grow(&e->dOut, &e->out_cap, need));
  eval_forward(h, e, 0, h->He);
  k_eval_score<true><<<(I + EV_IT - 1) / EV_IT, EV_THREADS, eval_smem_bytes(), st>>>(e->slot, 0, nullptr, nullptr, e->dOut, nullptr, 0);
  k_predict_act<<<batch, 256, 0, st>>>(e->slot, e->dOut, batch);
  h->launches += 2;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, e->dOut, need * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return G4R_OK;
}

// hidden state of the scoring path (predict_next_batch zeroes it when the batch size changes, gru4rec.py:696-697)
extern "C" int g4r_reset_eval_hidden(g4r_handle* h) {
  if (!h) return G4R_ERR_INVALID;
  cudaSetDevice(h->cfg.device);
  const int Be = h->cfg.eval_batch_size > 0 ? h->cfg.eval_batch_size : h->cfg.batch_size;
  for (int i = 0; i < h->md.n_layers; i++) CK(cudaMemsetAsync(h->He[i], 0, (size_t)Be * h->md.layer[i].ldL * sizeof(float), h->stream));
  return G4R_OK;
}

#include "g4r_topk.cuh"
#include "g4r_sessions.cuh"
#include "g4r_events.cuh"
#include "g4r_history.cuh"
#include "g4r_rest.cuh"
