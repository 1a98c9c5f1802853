// g4r_topk.cuh -- predict_next_batch reduced on the device to the k best items of every lane (g4r_predict_topk, DESIGN §3d).
// Included at the end of g4r_eval.cuh (uses EvalCtx and its operand split, eval_forward, k_eval_score, the tile loops ev_tiles /
// tc_sweep and the score chain ev_score_fp32).
//
// Ranking key of item i in lane b: act(x) for the elementwise final activations, the pre-activation x = y_b . Wy[i] + By[i] for
// softmax / softmax_logit; equal keys put the smaller index first.  Both are folded into one 64-bit key
//   (ordered fp32 bits of the key) << 32 | ~i
// so the order is total and the list unique.  The [lanes x items] score matrix is never written:
//   1. tau       exact fp32 scores of a catalogue prefix (k_eval_score, the predict kernel) and, per lane, their k-th key tau_b:
//                the k-th key of any subset bounds the k-th key of the catalogue from below
//   2. filter    the catalogue in tiles -- fp32 FFMA tiles (k_eval_score's tile loop, so exact) or wgmma 3xTF32 tiles
//                (within delta_b of fp32) -- keeps an item only if its key can still reach tau_b and appends its index to the lane's
//                survivor list; the softmax normaliser (max, sum of exp) is accumulated per tile on the way
//   3. select    one CTA per lane rescores its survivors with the fp32 chain of k_eval_tgt, radix-selects the k-th key and sorts
//                the k winners; a lane whose survivors overflowed its list scores its whole row in fp32 instead (bounded, exact)
// Filters (g4r_predict_topk_filtered): a candidate set (an n_items-bit mask plus the ascending list of its items, cached between
// calls by content) and per-lane exclusion lists (sorted CSR, uploaded per call).  The prefix of step 1 is the first P candidates
// with each lane's exclusions left out of its tau; the fp32 tiles run over the candidate list, the wgmma tiles over the catalogue
// with the mask; excluded items are never appended; step 3 applies both filters to a fallback row.  When every candidate is in
// the prefix, the prefix itself is the survivor set and no tile kernel runs.
#pragma once

constexpr int TOPK_THREADS = 512;          // select / tau kernels: one CTA per lane
constexpr int TOPK_PREFIX_MIN = 2048;      // items scored exactly for tau: max(k + exclusions, 2048, n_items / 16), at most n_cand
constexpr int TOPK_SURV_BASE = 4096;       // survivor list of a lane: min(n_items, 16 k + 4096) item indices

struct TopkCtx {
  unsigned int* dAbsMax = nullptr;                        // max |Wy|, max |By| as fp32 bits
  uint64_t absmax_version = ~0ull;                        // handle's wy_version they were taken from (as EvalCtx::split_version)
  float* dPre = nullptr; size_t pre_cap = 0;              // [batch x P] prefix pre-activations
  float* dTau = nullptr;                                  // [Be x 4] lo, hi, delta, tau item (int bits)
  int* dCnt = nullptr;                                    // [Be] survivors appended (may exceed the list)
  int* dSurv = nullptr; size_t surv_cap = 0;              // [batch x C] survivor items
  float* dSurvPre = nullptr; size_t surv_pre_cap = 0;     // [batch x C] their fp32 pre-activations
  float2* dPart = nullptr; size_t part_cap = 0;           // [batch x n_part] softmax partials (max, sum exp(x - max))
  int *dOvList = nullptr, *dOvRow = nullptr;              // overflowed lanes / row of each lane in the fallback buffer (-1: none)
  int* dItems = nullptr; size_t items_cap = 0;            // [batch x k] results
  float* dScores = nullptr; size_t scores_cap = 0;
  std::vector<uint32_t> hMask;                            // candidate bitmap last uploaded (the cache key; empty: none)
  unsigned int* dMask = nullptr; size_t mask_cap = 0;     // its device copy
  int* dCand = nullptr; size_t cand_cap = 0;              // its items, ascending
  int* dExOff = nullptr; size_t ex_off_cap = 0;           // [batch + 1] exclusion offsets of this call
  int* dEx = nullptr; size_t ex_cap = 0;                  // exclusions, sorted and distinct per lane
};

static void topk_release(EvalCtx& e) {
  if (!e.topk) return;
  TopkCtx& t = *static_cast<TopkCtx*>(e.topk);
  for (void* p : {(void*)t.dAbsMax, (void*)t.dPre, (void*)t.dTau, (void*)t.dCnt, (void*)t.dSurv,
                  (void*)t.dSurvPre, (void*)t.dPart, (void*)t.dOvList, (void*)t.dOvRow, (void*)t.dItems, (void*)t.dScores,
                  (void*)t.dMask, (void*)t.dCand, (void*)t.dExOff, (void*)t.dEx})
    if (p) cudaFree(p);
  delete static_cast<TopkCtx*>(e.topk);
  e.topk = nullptr;
}

// -0 and +0 are the same key (the index decides between them)
__device__ __forceinline__ uint64_t topk_key(float kf, int item) {
  if (kf == 0.f) kf = 0.f;
  return ((uint64_t)tc_fkey(kf) << 32) | (uint64_t)(~(uint32_t)item);
}
__device__ __forceinline__ float topk_keyval(const ActSpec a, float pre) { return a.kind <= G4R_ACT_SELU ? act_fwd(a, pre) : pre; }

// item in the candidate bitmap (nullptr: every item)
__device__ __forceinline__ bool topk_is_cand(const unsigned int* __restrict__ mask, int item) {
  return !mask || ((mask[item >> 5] >> (item & 31)) & 1u);
}
// item on lane b's exclusion list (ex_off == nullptr: no exclusions)
__device__ __forceinline__ bool topk_excluded(const int* __restrict__ ex_off, const int* __restrict__ ex, int b, int item) {
  if (!ex_off) return false;
  const int e0 = ex_off[b];
  return sorted_has(ex + e0, ex_off[b + 1] - e0, item);
}

// candidates of one lane: position j is item idx[j] (idx == nullptr: item j) with fp32 pre-activation pre[j]; an item outside
// `cand` (nullptr: none is) or on the sorted list ex[0 .. n_ex) does not compete
struct TopkSrc { const int* idx; const float* pre; int n; const unsigned int* cand = nullptr; const int* ex = nullptr; int n_ex = 0; };
__device__ __forceinline__ uint64_t topk_src_key(const ActSpec a, const TopkSrc& s, int j) {
  return topk_key(topk_keyval(a, s.pre[j]), s.idx ? s.idx[j] : j);
}
__device__ __forceinline__ bool topk_src_live(const TopkSrc& s, int j) {
  if (!s.cand && s.n_ex == 0) return true;
  const int item = s.idx ? s.idx[j] : j;
  return topk_is_cand(s.cand, item) && !sorted_has(s.ex, s.n_ex, item);
}
__device__ __forceinline__ void topk_set_excl(TopkSrc& s, const int* ex_off, const int* ex, int b) {
  if (ex_off) { s.ex = ex + ex_off[b]; s.n_ex = ex_off[b + 1] - ex_off[b]; }
}

// The k-th largest key among the live candidates (keys are distinct, so exactly k of them are >= it): MSB-first radix select,
// eight passes of 8 bits with a shared histogram.  With fewer than k live candidates (non-finite weights, or a filtered lane with
// fewer than k eligible items) the result is 0, below every key.  Every thread of the block returns the same value.
__device__ uint64_t topk_kth(const ActSpec a, const TopkSrc& s, int k, unsigned int* hist, unsigned int* bc) {
  uint64_t prefix = 0, mask = 0;
  unsigned int kk = (unsigned int)k;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
    for (int j = threadIdx.x; j < s.n; j += blockDim.x) {
      const uint64_t key = topk_src_key(a, s, j);
      if ((key & mask) == prefix && topk_src_live(s, j)) atomicAdd(&hist[(unsigned int)(key >> shift) & 255u], 1u);
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
// nullptr, the wgmma tiles): (||y_b||_1 max|Wy| + max|By|) * dscale.  Prefix position j is item pidx[j] (nullptr: item j); the
// lane's exclusions are left out of the select, so tau_b is the k-th key of its eligible prefix items
// (FILT = false: pidx / ex_off ignored, the unfiltered instantiation)
template <bool FILT>
__global__ void __launch_bounds__(TOPK_THREADS) k_topk_tau(int slot, const float* __restrict__ pre, int P, int k, float* tau,
                                                          const unsigned int* __restrict__ absmax, float dscale, const int* __restrict__ pidx_,
                                                          const int* __restrict__ ex_off_, const int* __restrict__ ex) {
  const ModelDev& md = MD;
  const int* pidx = FILT ? pidx_ : nullptr;
  const int* ex_off = FILT ? ex_off_ : nullptr;
  const int b = blockIdx.x;
  __shared__ unsigned int hist[256], bc[2];
  __shared__ float red[TOPK_THREADS / 32];
  __shared__ int tpos;
  TopkSrc s{pidx, pre + (size_t)b * P, P};
  topk_set_excl(s, ex_off, ex, b);
  if (threadIdx.x == 0) tpos = -1;
  const uint64_t T = topk_kth(md.fact, s, k, hist, bc);
  if (pidx) {                     // the prefix position of tau's item
    const int ti = (int)~(uint32_t)T;
    for (int j = threadIdx.x; j < P; j += blockDim.x) if (pidx[j] == ti) tpos = j;
    __syncthreads();
  }
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
    const int tj = pidx ? tpos : ti;
    const float t = tc_fkey_inv((uint32_t)(T >> 32)), xt = (tj >= 0 && tj < P) ? s.pre[tj] : t;
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
// softmax normaliser per (lane, 64-item tile).  subset != nullptr: the tiles run over the n_comp items subset[0 .. n_comp) instead
// of the catalogue; items on the lane's exclusion list are not appended (but are summed: exclusions never change a score)
// FILT = false: the unfiltered instantiation (subset / ex_off ignored), so g4r_predict_topk runs the code it ran before filters
template <bool FILT>
__global__ void __launch_bounds__(EV_THREADS) k_topk_fp32(int slot, const float* __restrict__ tau, int* cnt, int* surv, int C, float2* part, int n_part,
                                                          const int* __restrict__ subset_, int n_comp, const int* __restrict__ ex_off_, const int* __restrict__ ex) {
  const ModelDev& md = MD;
  const int* subset = FILT ? subset_ : nullptr;
  const int* ex_off = FILT ? ex_off_ : nullptr;
  extern __shared__ __align__(16) float smem[];
  float2* sP = reinterpret_cast<float2*>(smem + EV_TILE_FLOATS);   // [8 warps][EV_TB]
  const int M = md.wM[0], I = subset ? n_comp : md.n_items;
  const int i0 = blockIdx.x * EV_IT;
  const int ni = min(EV_IT, I - i0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool soft = md.fact.kind > G4R_ACT_SELU;
  ev_tiles(md, smem, M, i0, ni, subset, [&](int b0, float (&acc)[8]) {
    const int b = b0 + lane;
    float2 sm = make_float2(-INFINITY, 0.f);
    if (b < M) {
      const float lo = tau[b * 4 + 0], hi = tau[b * 4 + 1];
      const int ti = __float_as_int(tau[b * 4 + 3]);
      unsigned int keep = 0u;               // FILT: kept q, tested against the exclusions outside the unrolled loop
#pragma unroll
      for (int q = 0; q < 8; q++) {
        if (warp + 8 * q < ni) {
          const int it = ev_item(subset, i0 + warp + 8 * q);
          acc[q] += md.By[it];
          if (topk_keep(acc[q], 0.f, lo, hi, it, ti)) { if (FILT) keep |= 1u << q; else topk_append(cnt, surv, C, b, it); }
          sm.x = fmaxf(sm.x, acc[q]);
        }
      }
      while (FILT && keep) {
        const int q = __ffs(keep) - 1, it = ev_item(subset, i0 + warp + 8 * q);
        keep &= keep - 1u;
        if (!topk_excluded(ex_off, ex, b, it)) topk_append(cnt, surv, C, b, it);
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
  });
}
static size_t topk_fp32_smem_bytes() { return (size_t)EV_TILE_FLOATS * sizeof(float) + (EV_THREADS / 32) * EV_TB * sizeof(float2) + 64; }

// pass 2, wgmma 3xTF32 tiles: the sweep of k_eval_tc (tc_sweep) with a filtering epilogue: a thread keeps those of its two lanes
// x 32 items of the tile whose score x satisfies x + delta_b >= tau_b (topk_keep); partial softmax normaliser per (lane, tile,
// column half).  Items outside the candidate bitmap `cand` (nullptr: none) are neither kept nor summed; excluded items are summed,
// not kept.  FILT = false: the unfiltered instantiation (cand / ex_off ignored)
template <bool FILT>
__global__ void __launch_bounds__(TC_THREADS, 1) k_topk_tc(int slot, const float* __restrict__ tau, int* cnt, int* surv, int C, float2* part, int n_part,
                                                           const unsigned char* __restrict__ Asplit, const unsigned char* __restrict__ Bsplit,
                                                           const unsigned int* __restrict__ cand_, const int* __restrict__ ex_off_, const int* __restrict__ ex) {
  const unsigned int* cand = FILT ? cand_ : nullptr;
  const int* ex_off = FILT ? ex_off_ : nullptr;
  const ModelDev& md = MD;
  const int M = md.wM[0], I = md.n_items, lane = threadIdx.x & 31;
  const bool soft = md.fact.kind > G4R_ACT_SELU;
  int bb[2], ti[2]; bool vrow[2]; float lo[2], hi[2], dl[2];
  auto lane_block = [&](int b) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      bb[h] = b + 8 * h;
      vrow[h] = bb[h] < M;
      lo[h] = vrow[h] ? tau[bb[h] * 4 + 0] : INFINITY; hi[h] = vrow[h] ? tau[bb[h] * 4 + 1] : INFINITY;
      dl[h] = vrow[h] ? tau[bb[h] * 4 + 2] : 0.f; ti[h] = vrow[h] ? __float_as_int(tau[bb[h] * 4 + 3]) : -1;
    }
  };
  auto tile = [&](const float (&d)[64], int c0, bool) {
    // columns past the catalogue (last tile) and non-candidates are neither kept nor summed
    const int n_live = I - c0;
    float2 smx[2] = {make_float2(-INFINITY, 0.f), make_float2(-INFINITY, 0.f)};
#pragma unroll
    for (int i = 0; i < 64; i++) {
      const int h = (i >> 1) & 1, col = (i >> 2) * 8 + (i & 1);
      if (col < n_live && topk_is_cand(cand, c0 + col)) {
        if (vrow[h] && topk_keep(d[i], dl[h], lo[h], hi[h], c0 + col, ti[h]) && !topk_excluded(ex_off, ex, bb[h], c0 + col))
          topk_append(cnt, surv, C, bb[h], c0 + col);
        smx[h].x = fmaxf(smx[h].x, d[i]);
      }
    }
    if (soft) {
#pragma unroll
      for (int i = 0; i < 64; i++) {
        const int h = (i >> 1) & 1, col = (i >> 2) * 8 + (i & 1);
        if (col < n_live && topk_is_cand(cand, c0 + col) && smx[h].x != -INFINITY) smx[h].y += expf(d[i] - smx[h].x);
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {                                  // the four threads of a quad share the two lanes
        float2 r = smx[h];
        r = topk_smx_merge(r, make_float2(__shfl_xor_sync(0xffffffffu, r.x, 1), __shfl_xor_sync(0xffffffffu, r.y, 1)));
        r = topk_smx_merge(r, make_float2(__shfl_xor_sync(0xffffffffu, r.x, 2), __shfl_xor_sync(0xffffffffu, r.y, 2)));
        if ((lane & 3) == 0 && vrow[h]) part[(size_t)bb[h] * n_part + c0 / 128] = r;   // c0 / 128 = 2 * tile + column half
      }
    }
  };
  tc_sweep(M, I, md.L + 1, Asplit, Bsplit, lane_block, tile);
}

// overflow fallback: the fp32 row of every overflowed lane (blockIdx.y-th entry of ov_list) into rows[y * n_items ...]
__global__ void __launch_bounds__(128) k_topk_rows(int slot, const int* __restrict__ ov_list, float* rows) {
  const ModelDev& md = MD;
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= md.n_items) return;
  rows[(size_t)blockIdx.y * md.n_items + item] = ev_score_fp32(md, ov_list[blockIdx.y], item);
}

// pass 3: per lane (one CTA) the exact fp32 pre-activations of the candidates -- the survivors, rescored with the fp32 chain, or
// the lane's whole fallback row -- then the k-th key, the k winners sorted best first, and their scores: the activated score for
// the elementwise activations, exp(x - m) / z with the catalogue's normaliser merged from the tile partials for softmax.
// cnt == nullptr (every candidate is in the prefix, no tile ran): the candidates are the prefix pidx[0 .. P) (nullptr: items
// 0 .. P-1) with pre-activations ppre, and the softmax normaliser is summed over them here (part unused).  The lane's exclusions
// never win; a fallback row is also restricted to the candidate bitmap `cand`.  Slots past the lane's eligible items: key 0,
// i.e. item -1 and a NaN score.
// (FILT = false: cnt != nullptr, and cand / ex_off ignored, the unfiltered instantiation)
template <bool FILT>
__global__ void __launch_bounds__(TOPK_THREADS) k_topk_final(int slot, int k, const int* __restrict__ cnt, const int* __restrict__ surv, float* surv_pre, int C,
                                                            const int* __restrict__ ov_row, const float* __restrict__ rows, const float2* __restrict__ part, int n_part,
                                                            int* out_items, float* out_scores, const int* __restrict__ pidx, const float* __restrict__ ppre, int P,
                                                            const unsigned int* __restrict__ cand_, const int* __restrict__ ex_off_, const int* __restrict__ ex) {
  const ModelDev& md = MD;
  const unsigned int* cand = FILT ? cand_ : nullptr;
  const int* ex_off = FILT ? ex_off_ : nullptr;
  const bool from_prefix = FILT && !cnt;
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ unsigned int hist[256], bc[2], n_got;
  __shared__ unsigned long long keys[G4R_TOPK_MAX];
  __shared__ float redf[TOPK_THREADS / 32];
  __shared__ double redd[TOPK_THREADS / 32];
  TopkSrc s;
  if (from_prefix) s = TopkSrc{pidx, ppre + (size_t)b * P, P};
  else if (ov_row && ov_row[b] >= 0) s = TopkSrc{nullptr, rows + (size_t)ov_row[b] * md.n_items, md.n_items, cand};
  else {
    s = TopkSrc{surv + (size_t)b * C, surv_pre + (size_t)b * C, min(cnt[b], C)};
    for (int j = tid; j < s.n; j += blockDim.x) surv_pre[(size_t)b * C + j] = ev_score_fp32(md, b, s.idx[j]);
    __syncthreads();
  }
  topk_set_excl(s, ex_off, ex, b);
  const uint64_t T = topk_kth(md.fact, s, k, hist, bc);
  int kp = 1;
  while (kp < k) kp <<= 1;
  if (tid == 0) n_got = 0u;
  __syncthreads();
  for (int j = tid; j < s.n; j += blockDim.x) {
    const uint64_t key = topk_src_key(md.fact, s, j);
    if (key >= T && topk_src_live(s, j)) { const unsigned int p = atomicAdd(&n_got, 1u); if (p < (unsigned)k) keys[p] = key; }
  }
  __syncthreads();
  for (int i = min(n_got, (unsigned)k) + tid; i < kp; i += blockDim.x) keys[i] = 0ull;   // fewer than k eligible (or non-finite weights)
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
    // the partials (max, sum exp(x - max)) of the tiles, or one (x, 1) per prefix candidate
    const float2* pr = from_prefix ? nullptr : part + (size_t)b * n_part;
    const int n_pr = from_prefix ? s.n : n_part;
    auto part_at = [&](int j) -> float2 { return pr ? pr[j] : make_float2(s.pre[j], 1.f); };
    for (int j = tid; j < n_pr; j += blockDim.x) m = fmaxf(m, part_at(j).x);
    m = warp_max(m);
    if ((tid & 31) == 0) redf[tid >> 5] = m;
    __syncthreads();
    m = redf[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) m = fmaxf(m, redf[w]);
    double zz = 0.0;
    for (int j = tid; j < n_pr; j += blockDim.x) {
      const float2 p = part_at(j);
      if (p.x != -INFINITY) zz += (double)p.y * exp((double)p.x - (double)m);
    }
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

static int topk_ctx(g4r_handle* h, EvalCtx* e, TopkCtx** out) {
  if (!e->topk) {
    TopkCtx t;
    CK(cudaMalloc(&t.dAbsMax, 2 * sizeof(unsigned int)));
    CK(cudaMalloc(&t.dTau, (size_t)e->Be * 4 * sizeof(float)));
    CK(cudaMalloc(&t.dCnt, (size_t)e->Be * sizeof(int)));
    CK(cudaMalloc(&t.dOvList, (size_t)e->Be * sizeof(int)));
    CK(cudaMalloc(&t.dOvRow, (size_t)e->Be * sizeof(int)));
    CK(cudaFuncSetAttribute(k_topk_fp32<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)topk_fp32_smem_bytes()));
    CK(cudaFuncSetAttribute(k_topk_fp32<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)topk_fp32_smem_bytes()));
    if (cudaFuncSetAttribute(k_topk_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem)) != cudaSuccess) cudaGetLastError();
    if (cudaFuncSetAttribute(k_topk_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem)) != cudaSuccess) cudaGetLastError();
    e->topk = new TopkCtx(t);
  }
  *out = static_cast<TopkCtx*>(e->topk);
  return G4R_OK;
}

// The candidate filter of a top-k call, validated with k: a bitmap of the distinct candidate items (the cache key of the device
// copy; empty: the whole catalogue)
struct TopkFilter {
  std::vector<uint32_t> cmask;
  int n_distinct = 0;
  bool use_cand = false;                                  // false when every item is a candidate: the unfiltered catalogue
  bool is_cand(int v) const { return !use_cand || ((cmask[(size_t)v >> 5] >> (v & 31)) & 1u); }
};

static int topk_filter(g4r_handle* h, int32_t k, const int32_t* cand, int64_t n_cand, TopkFilter* f) {
  const int I = h->md.n_items;
  f->n_distinct = I;
  if (cand) {
    if (n_cand < 0) FAIL(G4R_ERR_INVALID, "n_cand must be >= 0");
    f->cmask.assign((size_t)(I + 31) / 32, 0u);
    for (int64_t i = 0; i < n_cand; i++) {
      const int32_t c = cand[i];
      if (c < 0 || c >= I) FAIL(G4R_ERR_INDEX, "candidate item out of bounds");
      f->cmask[(size_t)c >> 5] |= 1u << (c & 31);
    }
    f->n_distinct = 0;
    for (const uint32_t w : f->cmask) f->n_distinct += __builtin_popcount(w);
  }
  if (k < 1 || k > f->n_distinct || k > G4R_TOPK_MAX)
    FAIL(G4R_ERR_INVALID, cand ? "k must be in 1 .. min(distinct candidates, G4R_TOPK_MAX)" : "k must be in 1 .. min(n_items, G4R_TOPK_MAX)");
  if (h->shard) FAIL(G4R_ERR_STATE, "g4r_predict_topk: not available on a row-sharded multi-GPU handle");
  f->use_cand = cand && f->n_distinct < I;
  if (!f->use_cand) f->cmask.clear();
  return G4R_OK;
}

// excl_off[0 .. n] of a call with n lanes: non-decreasing from 0, items in range
static int topk_check_excl(g4r_handle* h, int64_t n, const int64_t* excl_off, const int32_t* excl_items) {
  if (excl_off[0] != 0) FAIL(G4R_ERR_INVALID, "excl_off[0] must be 0");
  for (int64_t b = 0; b < n; b++) if (excl_off[b + 1] < excl_off[b]) FAIL(G4R_ERR_INVALID, "excl_off must be non-decreasing");
  if (excl_off[n] > 0 && !excl_items) FAIL(G4R_ERR_INVALID, "excl_items is NULL");
  for (int64_t j = 0; j < excl_off[n]; j++)
    if (excl_items[j] < 0 || excl_items[j] >= h->md.n_items) FAIL(G4R_ERR_INDEX, "excluded item out of bounds");
  return G4R_OK;
}

// exclusions of one lane: the (validated) items v[0 .. n) that are candidates (no other item can win anyway) appended to ex
static void topk_add_excl(const TopkFilter& f, const int32_t* v, int64_t n, std::vector<int>& ex) {
  for (int64_t j = 0; j < n; j++) if (f.is_cand(v[j])) ex.push_back(v[j]);
}
// ends the lane whose exclusions start at ex[e0]: sorted and distinct, its end offset appended to ex_off
static int topk_close_lane(g4r_handle* h, std::vector<int>& ex_off, std::vector<int>& ex, size_t e0) {
  std::sort(ex.begin() + e0, ex.end());
  ex.erase(std::unique(ex.begin() + e0, ex.end()), ex.end());
  if (ex.size() > (size_t)INT32_MAX) FAIL(G4R_ERR_INVALID, "too many exclusions");
  ex_off.push_back((int)ex.size());
  return G4R_OK;
}

static int topk_rank(g4r_handle* h, EvalCtx* e, float* const* Hst, int batch, int32_t k, const TopkFilter& f,
                     const std::vector<int>& ex_off, const std::vector<int>& ex, int32_t* out_items, float* out_scores);

// operands of the wgmma filter tiles: tc_operands' split item table and max |Wy|, max |By| (both remade only after Wy / By changed)
static int topk_tc_operands(g4r_handle* h, EvalCtx* e, TopkCtx* t) {
  int rc = tc_operands(h, e);
  if (rc) return rc;
  if (t->absmax_version != h->wy_version) {
    CK(cudaMemsetAsync(t->dAbsMax, 0, 2 * sizeof(unsigned int), h->stream));
    k_topk_absmax<<<2 * h->n_sm, 256, 0, h->stream>>>(h->md.Wy, h->md.By, h->md.n_items, h->md.ldL, h->md.L, t->dAbsMax);
    h->launches++;
    t->absmax_version = h->wy_version;
  }
  return G4R_OK;
}

// the device copy of f's candidate set (bitmap and ascending item list), uploaded only when it differs from the cached one
static int topk_upload_cand(g4r_handle* h, TopkCtx* t, const TopkFilter& f) {
  if (!f.use_cand || t->hMask == f.cmask) return G4R_OK;
  cudaStream_t st = h->stream;
  t->hMask.clear();
  std::vector<int> list;
  list.reserve((size_t)f.n_distinct);
  for (int i = 0; i < h->md.n_items; i++) if (f.is_cand(i)) list.push_back(i);
  CK(dev_grow(&t->dMask, &t->mask_cap, f.cmask.size()));
  CK(dev_grow(&t->dCand, &t->cand_cap, list.size()));
  CK(cudaMemcpyAsync(t->dMask, f.cmask.data(), f.cmask.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(t->dCand, list.data(), list.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  t->hMask = f.cmask;
  return G4R_OK;
}

// The constants of a top-k ranking of units of at most `lanes` lanes under the filter f, with at most max_ex exclusions per lane
struct TopkPlan {
  TopkCtx* t = nullptr;
  int k = 0, n_comp = 0, P = 0, C = 0;
  int n_part_fp32 = 0, n_part_tc = 0;                     // softmax partials per lane of each tile kind
  bool no_tile = false;                                   // every candidate is in the prefix: no filter tiles, no overflow
  bool filt = false;                                      // the filtering instances: candidates and / or exclusions
  bool tc_any = false;                                    // some unit may take the wgmma tiles (their operands are ready)
  const unsigned int* dmask = nullptr; const int* dcand = nullptr;   // the candidate set (nullptr: the catalogue)
};

// the plan, the top-k buffers sized for `lanes` lanes, and the candidate set and wgmma operands on the device.  The prefix is the
// first P candidates; P covers k eligible items of every lane, or every candidate (then it is the survivor set and no tile runs)
static int topk_plan(g4r_handle* h, EvalCtx* e, const TopkFilter& f, int k, int max_ex, int lanes, TopkPlan* p) {
  const int I = h->md.n_items;
  int rc = topk_ctx(h, e, &p->t);
  if (rc) return rc;
  TopkCtx* t = p->t;
  rc = topk_upload_cand(h, t, f);
  if (rc) return rc;
  p->k = k;
  p->filt = f.use_cand || max_ex > 0;
  p->n_comp = f.use_cand ? f.n_distinct : I;
  p->P = std::min(p->n_comp, std::max(k + max_ex, std::max(TOPK_PREFIX_MIN, (I / 16 + 63) & ~63)));
  p->no_tile = p->filt && p->P == p->n_comp;
  p->C = std::min(p->n_comp, 16 * k + TOPK_SURV_BASE);
  p->n_part_fp32 = (p->n_comp + EV_IT - 1) / EV_IT;
  p->n_part_tc = 2 * ((I + TC_N - 1) / TC_N);
  p->tc_any = !p->no_tile && wgmma_tiles(h->cfg, lanes, p->n_comp, I);
  p->dmask = f.use_cand ? t->dMask : nullptr;
  p->dcand = f.use_cand ? t->dCand : nullptr;
  CK(dev_grow(&t->dPre, &t->pre_cap, (size_t)lanes * p->P));
  if (!p->no_tile) {
    CK(dev_grow(&t->dSurv, &t->surv_cap, (size_t)lanes * p->C));
    CK(dev_grow(&t->dSurvPre, &t->surv_pre_cap, (size_t)lanes * p->C));
    CK(dev_grow(&t->dPart, &t->part_cap, (size_t)lanes * std::max(p->n_part_fp32, p->n_part_tc)));
  }
  if (p->tc_any) {
    rc = topk_tc_operands(h, e, t);
    if (rc) return rc;
  }
  return G4R_OK;
}

// Steps 1 and 2 for the M lanes of scoring descriptor `slot` (their final-layer y at y) on stream st, under the exclusions
// ex_off / ex (nullptr: none): the exact prefix scores and tau_b, then, unless no_tile, the filter tiles, which append to the
// survivor counters cnt (zeroed by the caller) and write the softmax partials.  Returns the partials per lane (0: no tile ran)
static int topk_tiles(g4r_handle* h, EvalCtx* e, const TopkPlan& p, int slot, const float* y, int M, int* cnt, const int* ex_off, const int* ex,
                      cudaStream_t st) {
  TopkCtx* t = p.t;
  const int I = h->md.n_items, L = h->md.L;
  k_eval_score<true><<<(p.P + EV_IT - 1) / EV_IT, EV_THREADS, eval_smem_bytes(), st>>>(slot, 0, nullptr, nullptr, t->dPre, p.dcand, p.P);
  h->launches++;
  if (p.no_tile) return 0;
  const bool tc = p.tc_any && wgmma_tiles(h->cfg, M, p.n_comp, I);
  // delta_b = (||y_b||_1 max|Wy| + max|By|) (L + 3) 2^-18: four times the worst case of |3xTF32 - fp32| (DESIGN §3d)
  (p.filt ? k_topk_tau<true> : k_topk_tau<false>)<<<M, TOPK_THREADS, 0, st>>>(slot, t->dPre, p.P, p.k, t->dTau, tc ? t->dAbsMax : nullptr,
                                                                              ldexpf((float)(L + 3), -18), p.dcand, ex_off, ex);
  if (tc) {
    const int tc_chunks = (L + 1 + TC_KC - 1) / TC_KC, tc_tiles = (I + TC_N - 1) / TC_N;
    k_tc_split<TC_M><<<dim3((M + TC_M - 1) / TC_M, tc_chunks), 256, 0, st>>>(y, M, h->md.ldL, L, e->dAsplit, tc_chunks, nullptr, 1.0f);
    (p.filt ? k_topk_tc<true> : k_topk_tc<false>)<<<std::min(tc_tiles, h->n_sm), TC_THREADS, sizeof(TcSmem), st>>>(
        slot, t->dTau, cnt, t->dSurv, p.C, t->dPart, p.n_part_tc, e->dAsplit, e->dBsplit, p.dmask, ex_off, ex);
    h->launches += 3;
    return p.n_part_tc;
  }
  (p.filt ? k_topk_fp32<true> : k_topk_fp32<false>)<<<p.n_part_fp32, EV_THREADS, topk_fp32_smem_bytes(), st>>>(
      slot, t->dTau, cnt, t->dSurv, p.C, t->dPart, p.n_part_fp32, p.dcand, p.n_comp, ex_off, ex);
  h->launches += 2;
  return p.n_part_fp32;
}

// Step 3 for the M lanes of descriptor `slot`: each lane selects from its survivors (cnt; nullptr: from the prefix) or from its
// fallback row rows[ov_row[b]] (ov_row nullptr: none), with the softmax partials part [M x n_part], into items / scores [M x k]
static void topk_select(g4r_handle* h, const TopkPlan& p, int slot, int M, const int* cnt, const int* ov_row, const float* rows, const float2* part,
                        int n_part, int* items, float* scores, const int* ex_off, const int* ex, cudaStream_t st) {
  TopkCtx* t = p.t;
  (p.filt ? k_topk_final<true> : k_topk_final<false>)<<<M, TOPK_THREADS, 0, st>>>(slot, p.k, cnt, t->dSurv, t->dSurvPre, p.C, ov_row, rows, part, n_part,
                                                                                  items, scores, p.dcand, t->dPre, p.P, p.dmask, ex_off, ex);
  h->launches++;
}

extern "C" int g4r_predict_topk_filtered(g4r_handle* h, const int32_t* X, int32_t batch, const uint8_t* reset_mask, int32_t k,
                                         const int32_t* cand, int64_t n_cand, const int64_t* excl_off, const int32_t* excl_items,
                                         int32_t* out_items, float* out_scores) {
  if (!h || !X || !out_items || !out_scores) return G4R_ERR_INVALID;
  TopkFilter f;
  int rc = topk_filter(h, k, cand, n_cand, &f);
  if (rc) return rc;
  // exclusions: per lane sorted and distinct, restricted to the candidates
  std::vector<int> ex_off, ex;
  if (excl_off) {
    if (batch <= 0) FAIL(G4R_ERR_INVALID, "predict batch exceeds eval_batch_size");
    rc = topk_check_excl(h, batch, excl_off, excl_items);
    if (rc) return rc;
    ex_off.push_back(0);
    for (int b = 0; b < batch; b++) {
      const size_t e0 = ex.size();
      topk_add_excl(f, excl_items + excl_off[b], excl_off[b + 1] - excl_off[b], ex);
      rc = topk_close_lane(h, ex_off, ex, e0);
      if (rc) return rc;
    }
  }
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  rc = eval_ctx(h, &e);
  if (rc) return rc;
  rc = predict_stage(h, e, X, batch, reset_mask);
  if (rc) return rc;
  return topk_rank(h, e, h->He, batch, k, f, ex_off, ex, out_items, out_scores);
}

// The shared ranking of g4r_predict_topk_filtered and g4r_sessions_topk: the GRU forward of the lanes staged at step 0 of the
// scoring window, reading and writing hidden states in Hst (one array per layer, addressed by the staged slots), then the k best
// items of every lane under the filter f and the per-lane exclusions ex_off / ex (empty: none; built by topk_add_excl /
// topk_close_lane) into out_items / out_scores [batch x k] (host)
static int topk_rank(g4r_handle* h, EvalCtx* e, float* const* Hst, int batch, int32_t k, const TopkFilter& f,
                     const std::vector<int>& ex_off, const std::vector<int>& ex, int32_t* out_items, float* out_scores) {
  const int I = h->md.n_items;
  const bool use_ex = !ex.empty();
  int max_ex = 0;
  for (size_t b = 1; b < ex_off.size(); b++) max_ex = std::max(max_ex, ex_off[b] - ex_off[b - 1]);
  TopkPlan p;
  int rc = topk_plan(h, e, f, k, max_ex, batch, &p);
  if (rc) return rc;
  TopkCtx* t = p.t;
  cudaStream_t st = h->stream;
  if (use_ex) {
    CK(dev_grow(&t->dExOff, &t->ex_off_cap, ex_off.size()));
    CK(dev_grow(&t->dEx, &t->ex_cap, ex.size()));
    CK(cudaMemcpyAsync(t->dExOff, ex_off.data(), ex_off.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(t->dEx, ex.data(), ex.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  }
  const int* dexoff = use_ex ? t->dExOff : nullptr;
  const int* dex = use_ex ? t->dEx : nullptr;
  CK(dev_grow(&t->dItems, &t->items_cap, (size_t)batch * k));
  CK(dev_grow(&t->dScores, &t->scores_cap, (size_t)batch * k));
  eval_forward(h, e, 0, Hst);
  if (!p.no_tile) CK(cudaMemsetAsync(t->dCnt, 0, (size_t)batch * sizeof(int), st));
  const int n_part = topk_tiles(h, e, p, e->slot, h->md.layer[h->md.n_layers - 1].y, batch, t->dCnt, dexoff, dex, st);
  int n_ov = 0;
  if (!p.no_tile) {
    CK(cudaGetLastError());
    // overflowed lanes (more survivors than their list holds) take their whole fp32 row, in g4r_predict's score buffer
    std::vector<int> cnt((size_t)batch), ov_row((size_t)batch, -1), ov_list;
    CK(cudaMemcpyAsync(cnt.data(), t->dCnt, (size_t)batch * sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int b = 0; b < batch; b++) if (cnt[(size_t)b] > p.C) { ov_row[(size_t)b] = (int)ov_list.size(); ov_list.push_back(b); }
    n_ov = (int)ov_list.size();
    if (n_ov > 0) {
      const size_t need = (size_t)n_ov * I;
      CK(dev_grow(&e->dOut, &e->out_cap, need));
      CK(cudaMemcpyAsync(t->dOvList, ov_list.data(), (size_t)n_ov * sizeof(int), cudaMemcpyHostToDevice, st));
      CK(cudaMemcpyAsync(t->dOvRow, ov_row.data(), (size_t)batch * sizeof(int), cudaMemcpyHostToDevice, st));
      k_topk_rows<<<dim3((I + 127) / 128, n_ov), 128, 0, st>>>(e->slot, t->dOvList, e->dOut);
      h->launches++;
    }
  }
  topk_select(h, p, e->slot, batch, p.no_tile ? nullptr : t->dCnt, n_ov > 0 ? t->dOvRow : nullptr, e->dOut, t->dPart, n_part, t->dItems, t->dScores,
              dexoff, dex, st);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out_items, t->dItems, (size_t)batch * k * sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(out_scores, t->dScores, (size_t)batch * k * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return G4R_OK;
}

extern "C" int g4r_predict_topk(g4r_handle* h, const int32_t* X, int32_t batch, const uint8_t* reset_mask, int32_t k,
                                int32_t* out_items, float* out_scores) {
  return g4r_predict_topk_filtered(h, X, batch, reset_mask, k, nullptr, 0, nullptr, nullptr, out_items, out_scores);
}
