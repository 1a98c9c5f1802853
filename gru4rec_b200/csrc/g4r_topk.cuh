// g4r_topk.cuh -- predict_next_batch reduced on the device to the k best items of every lane (g4r_predict_topk, DESIGN §3d).
// Included at the end of g4r_eval.cuh (uses EvalCtx, eval_forward, k_eval_score and the k_eval_tc pipeline pieces).
//
// Ranking key of item i in lane b: act(x) for the elementwise final activations, the pre-activation x = y_b . Wy[i] + By[i] for
// softmax / softmax_logit; equal keys put the smaller index first.  Both are folded into one 64-bit key
//   (ordered fp32 bits of the key) << 32 | ~i
// so the order is total and the list unique.  The [lanes x items] score matrix is never written:
//   1. tau       exact fp32 scores of a catalogue prefix (k_eval_score, the predict kernel) and, per lane, their k-th key tau_b:
//                the k-th key of any subset bounds the k-th key of the catalogue from below
//   2. filter    the catalogue in tiles -- fp32 FFMA tiles (the very fma chain of k_eval_score, so exact) or wgmma 3xTF32 tiles
//                (within delta_b of fp32) -- keeps an item only if its key can still reach tau_b and appends its index to the lane's
//                survivor list; the softmax normaliser (max, sum of exp) is accumulated per tile on the way
//   3. select    one CTA per lane rescores its survivors with the fp32 chain of k_eval_tgt, radix-selects the k-th key and sorts
//                the k winners; a lane whose survivors overflowed its list scores its whole row in fp32 instead (bounded, exact)
#pragma once

constexpr int TOPK_THREADS = 512;          // select / tau kernels: one CTA per lane
constexpr int TOPK_PREFIX_MIN = 2048;      // items scored exactly for tau: max(k, 2048, n_items / 16), at most n_items
constexpr int TOPK_SURV_BASE = 4096;       // survivor list of a lane: min(n_items, 16 k + 4096) item indices

struct TopkCtx {
  unsigned char *dAsplit = nullptr, *dBsplit = nullptr;   // hidden-state / item-table [hi | lo] TF32 blocks (k_tc_split)
  uint64_t split_version = ~0ull;                         // handle's wy_version the item-table split was made from
  unsigned int* dAbsMax = nullptr;                        // max |Wy|, max |By| as fp32 bits (with the split)
  int* dIota = nullptr; int iota_n = 0;                   // 0, 1, 2, ...: the prefix as a k_eval_score item list
  float* dPre = nullptr; size_t pre_cap = 0;              // [batch x P] prefix pre-activations
  float* dTau = nullptr;                                  // [Be x 4] lo, hi, delta, tau item (int bits)
  int* dCnt = nullptr;                                    // [Be] survivors appended (may exceed the list)
  int* dSurv = nullptr; size_t surv_cap = 0;              // [batch x C] survivor items
  float* dSurvPre = nullptr; size_t surv_pre_cap = 0;     // [batch x C] their fp32 pre-activations
  float2* dPart = nullptr; size_t part_cap = 0;           // [batch x n_part] softmax partials (max, sum exp(x - max))
  int *dOvList = nullptr, *dOvRow = nullptr;              // overflowed lanes / row of each lane in the fallback buffer (-1: none)
  int* dItems = nullptr; size_t items_cap = 0;            // [batch x k] results
  float* dScores = nullptr; size_t scores_cap = 0;
};

static void topk_release(EvalCtx& e) {
  if (!e.topk) return;
  TopkCtx& t = *static_cast<TopkCtx*>(e.topk);
  for (void* p : {(void*)t.dAsplit, (void*)t.dBsplit, (void*)t.dAbsMax, (void*)t.dIota, (void*)t.dPre, (void*)t.dTau, (void*)t.dCnt, (void*)t.dSurv,
                  (void*)t.dSurvPre, (void*)t.dPart, (void*)t.dOvList, (void*)t.dOvRow, (void*)t.dItems, (void*)t.dScores})
    if (p) cudaFree(p);
  delete static_cast<TopkCtx*>(e.topk);
  e.topk = nullptr;
}

template <class T>
static cudaError_t topk_grow(T** p, size_t* cap, size_t n) {
  if (*cap >= n && *p) return cudaSuccess;
  if (*p) cudaFree(*p);
  *p = nullptr; *cap = 0;
  const cudaError_t r = cudaMalloc(p, n * sizeof(T));
  if (r == cudaSuccess) *cap = n;
  return r;
}

// -0 and +0 are the same key (the index decides between them)
__device__ __forceinline__ uint64_t topk_key(float kf, int item) {
  if (kf == 0.f) kf = 0.f;
  return ((uint64_t)tc_fkey(kf) << 32) | (uint64_t)(~(uint32_t)item);
}
__device__ __forceinline__ float topk_keyval(const ActSpec a, float pre) { return a.kind <= G4R_ACT_SELU ? act_fwd(a, pre) : pre; }

// fp32 score of (lane b, item): the sequential fma chain of k_eval_tgt / k_eval_score (bitwise equal to g4r_predict's value)
__device__ __forceinline__ float topk_score_fp32(const ModelDev& md, int b, int item) {
  const float* yr = md.layer[md.n_layers - 1].y + (size_t)b * md.ldL;
  const float* wr = md.Wy + (size_t)item * md.ldL;
  float a = 0.f;
#pragma unroll 8
  for (int c4 = 0; c4 < md.ldL / 4; c4++) {
    const float4 y = ld4(yr + c4 * 4), w = ld4(wr + c4 * 4);
    a = fmaf(y.x, w.x, a); a = fmaf(y.y, w.y, a); a = fmaf(y.z, w.z, a); a = fmaf(y.w, w.w, a);
  }
  return a + md.By[item];
}

// candidates of one lane: position j is item idx[j] (idx == nullptr: item j) with fp32 pre-activation pre[j]
struct TopkSrc { const int* idx; const float* pre; int n; };
__device__ __forceinline__ uint64_t topk_src_key(const ActSpec a, const TopkSrc& s, int j) {
  return topk_key(topk_keyval(a, s.pre[j]), s.idx ? s.idx[j] : j);
}

// The k-th largest key among the candidates (keys are distinct, so exactly k candidates are >= it): MSB-first radix select,
// eight passes of 8 bits with a shared histogram.  With fewer than k candidates (only non-finite weights get there) the result is
// some key below all of them.  Every thread of the block returns the same value.
__device__ uint64_t topk_kth(const ActSpec a, const TopkSrc& s, int k, unsigned int* hist, unsigned int* bc) {
  uint64_t prefix = 0, mask = 0;
  unsigned int kk = (unsigned int)k;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
    for (int j = threadIdx.x; j < s.n; j += blockDim.x) {
      const uint64_t key = topk_src_key(a, s, j);
      if ((key & mask) == prefix) atomicAdd(&hist[(unsigned int)(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int c = 0; int d = 255;
      for (; d > 0; d--) { if (c + hist[d] >= kk) break; c += hist[d]; }
      bc[0] = (unsigned int)d; bc[1] = kk - c;
    }
    __syncthreads();
    prefix |= (uint64_t)bc[0] << shift; mask |= 255ull << shift; kk = bc[1];
  }
  return prefix;
}

// pass 1: tau_b = the k-th key of the exact prefix scores, as the two pre-activation thresholds of k_eval_tc (act(x) > key <=>
// x > hi, act(x) == key <=> lo <= x <= hi) plus its item; delta_b bounds |3xTF32 - fp32| of every score of the lane (absmax !=
// nullptr, the wgmma tiles): (||y_b||_1 max|Wy| + max|By|) * dscale
__global__ void __launch_bounds__(TOPK_THREADS) k_topk_tau(int slot, const float* __restrict__ pre, int P, int k, float* tau,
                                                          const unsigned int* __restrict__ absmax, float dscale) {
  const ModelDev& md = MD;
  const int b = blockIdx.x;
  __shared__ unsigned int hist[256], bc[2];
  __shared__ float red[TOPK_THREADS / 32];
  const TopkSrc s{nullptr, pre + (size_t)b * P, P};
  const uint64_t T = topk_kth(md.fact, s, k, hist, bc);
  float delta = 0.f;
  if (absmax) {
    const float* yr = md.layer[md.n_layers - 1].y + (size_t)b * md.ldL;
    float n1 = 0.f;
    for (int c = threadIdx.x; c < md.ldL; c += blockDim.x) n1 += fabsf(yr[c]);
    n1 = warp_sum(n1);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = n1;
    __syncthreads();
    n1 = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) n1 += red[w];
    delta = (n1 * __uint_as_float(absmax[0]) + __uint_as_float(absmax[1])) * dscale;
  }
  if (threadIdx.x == 0) {
    const int ti = (int)~(uint32_t)T;
    const float t = tc_fkey_inv((uint32_t)(T >> 32)), xt = (ti >= 0 && ti < P) ? s.pre[ti] : t;
    float lo, hi;
    tc_thresholds(md.fact, md.fact.kind <= G4R_ACT_SELU, t, xt, lo, hi);
    tau[b * 4 + 0] = lo; tau[b * 4 + 1] = hi; tau[b * 4 + 2] = delta; tau[b * 4 + 3] = __int_as_float(ti);
  }
}

// x = the item's score as the tile computed it; keeps it if x_fp32 <= x + delta can still be >= tau (key, then index)
__device__ __forceinline__ bool topk_keep(float x, float delta, float lo, float hi, int item, int ti) {
  const float xd = x + delta;
  return xd > hi || (xd >= lo && item <= ti);
}
__device__ __forceinline__ void topk_append(int* cnt, int* surv, int C, int b, int item) {
  const int pos = atomicAdd(&cnt[b], 1);
  if (pos < C) surv[(size_t)b * C + pos] = item;
}
// (max, sum exp(x - max)) of two disjoint parts
__device__ __forceinline__ float2 topk_smx_merge(float2 p, float2 q) {
  const float m = fmaxf(p.x, q.x);
  if (m == -INFINITY) return make_float2(m, 0.f);
  return make_float2(m, (p.x == -INFINITY ? 0.f : p.y * expf(p.x - m)) + (q.x == -INFINITY ? 0.f : q.y * expf(q.x - m)));
}

// pass 2, fp32 FFMA tiles: k_eval_score's tiles and fma order (scores bitwise equal to the fp32 chain, so delta = 0); partial
// softmax normaliser per (lane, 64-item tile)
__global__ void __launch_bounds__(EV_THREADS) k_topk_fp32(int slot, const float* __restrict__ tau, int* cnt, int* surv, int C, float2* part, int n_part) {
  const ModelDev& md = MD;
  extern __shared__ __align__(16) float smem[];
  float* sY = smem;                        // [EV_TB][EV_LDS]
  float* sW = sY + EV_TB * EV_LDS;         // [EV_IT][EV_LDS]
  float2* sP = reinterpret_cast<float2*>(sW + EV_IT * EV_LDS);   // [8 warps][EV_TB]
  const int M = md.wM[0], I = md.n_items, ldL = md.ldL;
  const int i0 = blockIdx.x * EV_IT;
  const int ni = min(EV_IT, I - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool soft = md.fact.kind > G4R_ACT_SELU;
  const float* Y = md.layer[md.n_layers - 1].y;
  const bool hoist = ldL <= EV_KT;
  if (hoist) {
    const int kw = ldL / 4;
    for (int i = tid; i < EV_IT * kw; i += EV_THREADS) {
      const int rr = i / kw, c4 = i % kw;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rr < ni) v = ld4(md.Wy + (size_t)(i0 + rr) * ldL + c4 * 4);
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
          if (rr < ni) v = ld4(md.Wy + (size_t)(i0 + rr) * ldL + k0 + c4 * 4);
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
    const int b = b0 + lane;
    float2 sm = make_float2(-INFINITY, 0.f);
    if (b < M) {
      const float lo = tau[b * 4 + 0], hi = tau[b * 4 + 1];
      const int ti = __float_as_int(tau[b * 4 + 3]);
#pragma unroll
      for (int q = 0; q < 8; q++) {
        const int it = i0 + warp + 8 * q;
        if (warp + 8 * q < ni) {
          acc[q] += md.By[it];
          if (topk_keep(acc[q], 0.f, lo, hi, it, ti)) topk_append(cnt, surv, C, b, it);
          sm.x = fmaxf(sm.x, acc[q]);
        }
      }
      if (soft && sm.x != -INFINITY) {
#pragma unroll
        for (int q = 0; q < 8; q++) if (warp + 8 * q < ni) sm.y += expf(acc[q] - sm.x);
      }
    }
    if (soft) {
      sP[warp * EV_TB + lane] = sm;
      __syncthreads();
      if (warp == 0 && b < M) {
        float2 r = sP[lane];
        for (int w = 1; w < EV_THREADS / 32; w++) r = topk_smx_merge(r, sP[w * EV_TB + lane]);
        part[(size_t)b * n_part + blockIdx.x] = r;
      }
    }
  }
}
static size_t topk_fp32_smem_bytes() { return (size_t)(EV_TB * EV_LDS + EV_IT * EV_LDS) * sizeof(float) + (EV_THREADS / 32) * EV_TB * sizeof(float2) + 64; }

// pass 2, wgmma 3xTF32 tiles: k_eval_tc's pipeline (persistent CTAs, [A hi | A lo | B hi | B lo] stages fed by bulk copies,
// four warpgroups of 64 lanes x 128 items) with a filtering epilogue: a thread holds two lanes x 32 items of the tile and keeps
// those whose score x satisfies x + delta_b >= tau_b (topk_keep); partial softmax normaliser per (lane, tile, column half)
__global__ void __launch_bounds__(TC_THREADS, 1) k_topk_tc(int slot, const float* __restrict__ tau, int* cnt, int* surv, int C, float2* part, int n_part,
                                                           const unsigned char* __restrict__ Asplit, const unsigned char* __restrict__ Bsplit) {
  extern __shared__ __align__(1024) unsigned char tc_raw[];
  TcSmem& sm = *reinterpret_cast<TcSmem*>(tc_raw);
  const ModelDev& md = MD;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int M = md.wM[0], I = md.n_items, K = md.L + 1;       // + the bias column
  const bool soft = md.fact.kind > G4R_ACT_SELU;
  const int n_tiles = (I + TC_N - 1) / TC_N;
  const int n_lb = (M + TC_M - 1) / TC_M;
  const int n_chunk = (K + TC_KC - 1) / TC_KC;
  const int my_tiles = blockIdx.x < n_tiles ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const unsigned int total = (unsigned int)(n_lb * my_tiles * n_chunk);
  if (tid == 0) {
    for (int i = 0; i < TC_STAGES; i++) { tc_mbar_init(&sm.stage_free[i], 4); tc_mbar_init(&sm.stage_full[i], 1); }
    sm.err = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](unsigned int it) {
    const int c = (int)(it % n_chunk), q = (int)(it / n_chunk), t = blockIdx.x + (q % my_tiles) * gridDim.x, lb = q / my_tiles;
    const uint32_t st = it % TC_STAGES;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(tc_smem_u32(&sm.stage_full[st])), "r"(TC_STAGE_BYTES) : "memory");
    tc_bulk_copy(sm.stage[st], Asplit + ((size_t)lb * n_chunk + c) * 2 * TC_A_BYTES, 2 * TC_A_BYTES, &sm.stage_full[st]);
    tc_bulk_copy(sm.stage[st] + 2 * TC_A_BYTES, Bsplit + ((size_t)t * n_chunk + c) * 2 * TC_B_BYTES, 2 * TC_B_BYTES, &sm.stage_full[st]);
  };
  if (tid == 0) for (unsigned int it = 0; it < total && it < (unsigned)TC_STAGES; it++) issue(it);
  __syncwarp();
  const int wr = (wg & 1) * 64, wc = (wg >> 1) * 128;
  const int rq = (warp & 3) * 16 + (lane >> 2);
  unsigned int it = 0;
  for (int lb = 0; lb < n_lb; lb++) {
    int bb[2], ti[2]; bool vrow[2]; float lo[2], hi[2], dl[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      bb[h] = lb * TC_M + wr + rq + 8 * h;
      vrow[h] = bb[h] < M;
      lo[h] = vrow[h] ? tau[bb[h] * 4 + 0] : INFINITY; hi[h] = vrow[h] ? tau[bb[h] * 4 + 1] : INFINITY;
      dl[h] = vrow[h] ? tau[bb[h] * 4 + 2] : 0.f; ti[h] = vrow[h] ? __float_as_int(tau[bb[h] * 4 + 3]) : -1;
    }
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; i++) d[i] = 0.f;
      for (int c = 0; c < n_chunk; c++, it++) {
        const uint32_t st = it % TC_STAGES, use = it / TC_STAGES;
        tc_mbar_wait(&sm.stage_full[st], use & 1u, &sm.err);
        const uint32_t a_hi = tc_smem_u32(sm.stage[st]) + wr * 128, a_lo = a_hi + TC_A_BYTES;
        const uint32_t b_hi = tc_smem_u32(sm.stage[st]) + 2 * TC_A_BYTES + wc * 128, b_lo = b_hi + TC_B_BYTES;
        wg_chunk_3xtf32(d, a_hi, a_lo, b_hi, b_lo);
        if ((tid & 127) == 0) tc_mbar_arrive(&sm.stage_free[st]);
        if (tid == 0 && it + TC_STAGES < total) { tc_mbar_wait(&sm.stage_free[st], use & 1u, &sm.err); issue(it + TC_STAGES); }
        __syncwarp();
      }
      // columns past the catalogue (last tile) are neither kept nor summed
      const int c0 = t * TC_N + wc + 2 * (lane & 3);                // item of d[0]; d[i] holds item c0 + 8 * (i / 4) + i % 2
      const int n_live = I - c0;
      float2 smx[2] = {make_float2(-INFINITY, 0.f), make_float2(-INFINITY, 0.f)};
#pragma unroll
      for (int i = 0; i < 64; i++) {
        const int h = (i >> 1) & 1, col = (i >> 2) * 8 + (i & 1);
        if (col < n_live) {
          if (vrow[h] && topk_keep(d[i], dl[h], lo[h], hi[h], c0 + col, ti[h])) topk_append(cnt, surv, C, bb[h], c0 + col);
          smx[h].x = fmaxf(smx[h].x, d[i]);
        }
      }
      if (soft) {
#pragma unroll
        for (int i = 0; i < 64; i++) {
          const int h = (i >> 1) & 1, col = (i >> 2) * 8 + (i & 1);
          if (col < n_live && smx[h].x != -INFINITY) smx[h].y += expf(d[i] - smx[h].x);
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {                                  // the four threads of a quad share the two lanes
          float2 r = smx[h];
          r = topk_smx_merge(r, make_float2(__shfl_xor_sync(0xffffffffu, r.x, 1), __shfl_xor_sync(0xffffffffu, r.y, 1)));
          r = topk_smx_merge(r, make_float2(__shfl_xor_sync(0xffffffffu, r.x, 2), __shfl_xor_sync(0xffffffffu, r.y, 2)));
          if ((lane & 3) == 0 && vrow[h]) part[(size_t)bb[h] * n_part + 2 * t + (wg >> 1)] = r;
        }
      }
    }
  }
}

// overflow fallback: the fp32 row of every overflowed lane (blockIdx.y-th entry of ov_list) into rows[y * n_items ...]
__global__ void __launch_bounds__(128) k_topk_rows(int slot, const int* __restrict__ ov_list, float* rows) {
  const ModelDev& md = MD;
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= md.n_items) return;
  rows[(size_t)blockIdx.y * md.n_items + item] = topk_score_fp32(md, ov_list[blockIdx.y], item);
}

// pass 3: per lane (one CTA) the exact fp32 pre-activations of the candidates -- the survivors, rescored with the fp32 chain, or
// the lane's whole fallback row -- then the k-th key, the k winners sorted best first, and their scores: the activated score for
// the elementwise activations, exp(x - m) / z with the catalogue's normaliser merged from the tile partials for softmax
__global__ void __launch_bounds__(TOPK_THREADS) k_topk_final(int slot, int k, const int* __restrict__ cnt, const int* __restrict__ surv, float* surv_pre, int C,
                                                            const int* __restrict__ ov_row, const float* __restrict__ rows, const float2* __restrict__ part, int n_part,
                                                            int* out_items, float* out_scores) {
  const ModelDev& md = MD;
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ unsigned int hist[256], bc[2], n_got;
  __shared__ unsigned long long keys[G4R_TOPK_MAX];
  __shared__ float redf[TOPK_THREADS / 32];
  __shared__ double redd[TOPK_THREADS / 32];
  TopkSrc s;
  if (ov_row && ov_row[b] >= 0) s = TopkSrc{nullptr, rows + (size_t)ov_row[b] * md.n_items, md.n_items};
  else {
    s = TopkSrc{surv + (size_t)b * C, surv_pre + (size_t)b * C, min(cnt[b], C)};
    for (int j = tid; j < s.n; j += blockDim.x) surv_pre[(size_t)b * C + j] = topk_score_fp32(md, b, s.idx[j]);
    __syncthreads();
  }
  const uint64_t T = topk_kth(md.fact, s, k, hist, bc);
  int kp = 1;
  while (kp < k) kp <<= 1;
  if (tid == 0) n_got = 0u;
  __syncthreads();
  for (int j = tid; j < s.n; j += blockDim.x) {
    const uint64_t key = topk_src_key(md.fact, s, j);
    if (key >= T) { const unsigned int p = atomicAdd(&n_got, 1u); if (p < (unsigned)k) keys[p] = key; }
  }
  __syncthreads();
  for (int i = min(n_got, (unsigned)k) + tid; i < kp; i += blockDim.x) keys[i] = 0ull;   // (fewer than k only with non-finite weights)
  // bitonic sort, descending
  for (int size = 2; size <= kp; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = tid; i < kp; i += blockDim.x) {
        const int j = i ^ stride;
        if (j > i) {
          const unsigned long long a = keys[i], c = keys[j];
          if (((i & size) == 0) == (a < c)) { keys[i] = c; keys[j] = a; }
        }
      }
    }
  }
  __syncthreads();
  float m = -INFINITY, z = 0.f;
  if (md.fact.kind > G4R_ACT_SELU) {
    const float2* pr = part + (size_t)b * n_part;
    for (int j = tid; j < n_part; j += blockDim.x) m = fmaxf(m, pr[j].x);
    m = warp_max(m);
    if ((tid & 31) == 0) redf[tid >> 5] = m;
    __syncthreads();
    m = redf[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) m = fmaxf(m, redf[w]);
    double zz = 0.0;
    for (int j = tid; j < n_part; j += blockDim.x) if (pr[j].x != -INFINITY) zz += (double)pr[j].y * exp((double)pr[j].x - (double)m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) zz += __shfl_xor_sync(0xffffffffu, zz, o);
    if ((tid & 31) == 0) redd[tid >> 5] = zz;
    __syncthreads();
    zz = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) zz += redd[w];
    z = (float)zz;
  }
  for (int i = tid; i < k; i += blockDim.x) {
    const unsigned long long key = keys[i];
    const float kf = tc_fkey_inv((uint32_t)(key >> 32));
    out_items[(size_t)b * k + i] = (int)~(uint32_t)key;
    out_scores[(size_t)b * k + i] = md.fact.kind > G4R_ACT_SELU ? __fdiv_rn(expf(kf - m), z) : kf;
  }
}

// max |Wy| (the L live columns) and max |By| as fp32 bits; out zeroed by the caller
__global__ void __launch_bounds__(256) k_topk_absmax(const float* __restrict__ Wy, const float* __restrict__ By, int I, int ld, int L, unsigned int* out) {
  unsigned int mw = 0u, mb = 0u;
  const size_t n = (size_t)I * L, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) mw = max(mw, __float_as_uint(fabsf(Wy[(i / L) * ld + i % L])));
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)I; i += stride) mb = max(mb, __float_as_uint(fabsf(By[i])));
  mw = __reduce_max_sync(0xffffffffu, mw); mb = __reduce_max_sync(0xffffffffu, mb);
  if ((threadIdx.x & 31) == 0) { atomicMax(&out[0], mw); atomicMax(&out[1], mb); }
}
__global__ void k_topk_iota(int* p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}

static int topk_ctx(g4r_handle* h, EvalCtx* e, TopkCtx** out) {
  if (!e->topk) {
    TopkCtx t;
    CK(cudaMalloc(&t.dAbsMax, 2 * sizeof(unsigned int)));
    CK(cudaMalloc(&t.dTau, (size_t)e->Be * 4 * sizeof(float)));
    CK(cudaMalloc(&t.dCnt, (size_t)e->Be * sizeof(int)));
    CK(cudaMalloc(&t.dOvList, (size_t)e->Be * sizeof(int)));
    CK(cudaMalloc(&t.dOvRow, (size_t)e->Be * sizeof(int)));
    CK(cudaFuncSetAttribute(k_topk_fp32, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)topk_fp32_smem_bytes()));
    if (cudaFuncSetAttribute(k_topk_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem)) != cudaSuccess) cudaGetLastError();
    e->topk = new TopkCtx(t);
  }
  *out = static_cast<TopkCtx*>(e->topk);
  return G4R_OK;
}

extern "C" int g4r_predict_topk(g4r_handle* h, const int32_t* X, int32_t batch, const uint8_t* reset_mask, int32_t k,
                                int32_t* out_items, float* out_scores) {
  if (!h || !X || !out_items || !out_scores) return G4R_ERR_INVALID;
  const int I = h->md.n_items;
  if (k < 1 || k > I || k > G4R_TOPK_MAX) FAIL(G4R_ERR_INVALID, "k must be in 1 .. min(n_items, G4R_TOPK_MAX)");
  if (h->shard) FAIL(G4R_ERR_STATE, "g4r_predict_topk: not available on a row-sharded multi-GPU handle");
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  int rc = eval_ctx(h, &e);
  if (rc) return rc;
  rc = predict_stage(h, e, X, batch, reset_mask);
  if (rc) return rc;
  TopkCtx* t = nullptr;
  rc = topk_ctx(h, e, &t);
  if (rc) return rc;
  cudaStream_t st = h->stream;
  const int Be = e->Be, L = h->md.L;
  const int P = std::min(I, std::max(k, std::max(TOPK_PREFIX_MIN, (I / 16 + 63) & ~63)));
  const int C = std::min(I, 16 * k + TOPK_SURV_BASE);
  // tile kind: the rule of g4r_eval_schedule (cfg.eval_tc 1 = fp32 FFMA tiles, 2 = wgmma tiles, 0 = wgmma for >= 64 lanes and
  // >= 2048 items, where the split table is amortised over enough lanes)
  const bool tc = h->cfg.eval_tc == 2 || (h->cfg.eval_tc == 0 && batch >= 64 && I >= 2048);
  const int tc_chunks = (L + 1 + TC_KC - 1) / TC_KC, tc_tiles = (I + TC_N - 1) / TC_N;
  const int n_part = tc ? 2 * tc_tiles : (I + EV_IT - 1) / EV_IT;
  if (t->iota_n < P) {
    if (t->dIota) cudaFree(t->dIota);
    t->dIota = nullptr; t->iota_n = 0;
    CK(cudaMalloc(&t->dIota, (size_t)P * sizeof(int)));
    k_topk_iota<<<(P + 255) / 256, 256, 0, st>>>(t->dIota, P);
    t->iota_n = P;
  }
  CK(topk_grow(&t->dPre, &t->pre_cap, (size_t)batch * P));
  CK(topk_grow(&t->dSurv, &t->surv_cap, (size_t)batch * C));
  CK(topk_grow(&t->dSurvPre, &t->surv_pre_cap, (size_t)batch * C));
  CK(topk_grow(&t->dPart, &t->part_cap, (size_t)batch * n_part));
  CK(topk_grow(&t->dItems, &t->items_cap, (size_t)batch * k));
  CK(topk_grow(&t->dScores, &t->scores_cap, (size_t)batch * k));
  if (tc && (!t->dBsplit || t->split_version != h->wy_version)) {        // the cached item-table split is stale
    if (!t->dBsplit) CK(cudaMalloc(&t->dBsplit, (size_t)tc_tiles * tc_chunks * 2 * TC_B_BYTES));
    k_tc_split<TC_N><<<dim3(tc_tiles, tc_chunks), 256, 0, st>>>(h->md.Wy, I, h->md.ldL, L, t->dBsplit, tc_chunks, h->md.By, 0.f);
    CK(cudaMemsetAsync(t->dAbsMax, 0, 2 * sizeof(unsigned int), st));
    k_topk_absmax<<<2 * h->n_sm, 256, 0, st>>>(h->md.Wy, h->md.By, I, h->md.ldL, L, t->dAbsMax);
    h->launches += 2;
    t->split_version = h->wy_version;
  }
  eval_forward(h, e, 0);
  // 1. exact fp32 scores of the prefix [0, P) (the predict kernel over the item list 0 .. P-1) and tau_b
  k_eval_score<true><<<(P + EV_IT - 1) / EV_IT, EV_THREADS, eval_smem_bytes(), st>>>(e->slot, 0, nullptr, nullptr, t->dPre, t->dIota, P);
  // delta_b = (||y_b||_1 max|Wy| + max|By|) (L + 3) 2^-18: four times the worst case of |3xTF32 - fp32| (DESIGN §3d)
  k_topk_tau<<<batch, TOPK_THREADS, 0, st>>>(e->slot, t->dPre, P, k, t->dTau, tc ? t->dAbsMax : nullptr, ldexpf((float)(L + 3), -18));
  CK(cudaMemsetAsync(t->dCnt, 0, (size_t)batch * sizeof(int), st));
  // 2. the catalogue in tiles: survivors and softmax partials
  if (tc) {
    if (!t->dAsplit) CK(cudaMalloc(&t->dAsplit, (size_t)((Be + TC_M - 1) / TC_M) * tc_chunks * 2 * TC_A_BYTES));
    k_tc_split<TC_M><<<dim3((batch + TC_M - 1) / TC_M, tc_chunks), 256, 0, st>>>(h->md.layer[h->md.n_layers - 1].y, batch, h->md.ldL, L, t->dAsplit, tc_chunks, nullptr, 1.0f);
    k_topk_tc<<<std::min(tc_tiles, h->n_sm), TC_THREADS, sizeof(TcSmem), st>>>(e->slot, t->dTau, t->dCnt, t->dSurv, C, t->dPart, n_part, t->dAsplit, t->dBsplit);
    h->launches += 2;
  } else {
    k_topk_fp32<<<(I + EV_IT - 1) / EV_IT, EV_THREADS, topk_fp32_smem_bytes(), st>>>(e->slot, t->dTau, t->dCnt, t->dSurv, C, t->dPart, n_part);
    h->launches++;
  }
  h->launches += 2;
  CK(cudaGetLastError());
  // 3. overflowed lanes (more survivors than their list holds) take their whole fp32 row, in g4r_predict's score buffer
  std::vector<int> cnt((size_t)batch), ov_row((size_t)batch, -1), ov_list;
  CK(cudaMemcpyAsync(cnt.data(), t->dCnt, (size_t)batch * sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int b = 0; b < batch; b++) if (cnt[(size_t)b] > C) { ov_row[(size_t)b] = (int)ov_list.size(); ov_list.push_back(b); }
  const int n_ov = (int)ov_list.size();
  if (n_ov > 0) {
    const size_t need = (size_t)n_ov * I;
    if (e->out_cap < need) { if (e->dOut) cudaFree(e->dOut); e->dOut = nullptr; e->out_cap = 0; CK(cudaMalloc(&e->dOut, need * sizeof(float))); e->out_cap = need; }
    CK(cudaMemcpyAsync(t->dOvList, ov_list.data(), (size_t)n_ov * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(t->dOvRow, ov_row.data(), (size_t)batch * sizeof(int), cudaMemcpyHostToDevice, st));
    k_topk_rows<<<dim3((I + 127) / 128, n_ov), 128, 0, st>>>(e->slot, t->dOvList, e->dOut);
    h->launches++;
  }
  k_topk_final<<<batch, TOPK_THREADS, 0, st>>>(e->slot, k, t->dCnt, t->dSurv, t->dSurvPre, C, n_ov > 0 ? t->dOvRow : nullptr, e->dOut, t->dPart, n_part,
                                               t->dItems, t->dScores);
  h->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out_items, t->dItems, (size_t)batch * k * sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_scores, t->dScores, (size_t)batch * k * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return G4R_OK;
}
