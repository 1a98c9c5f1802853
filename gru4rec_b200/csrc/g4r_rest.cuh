// g4r_rest.cuh -- g4r_eval_rest (DESIGN §3m): rest-of-session evaluation.  Every counted event of the evaluation schedule is
// ranked against each DISTINCT item of the rest of its session (rows p+1 .. end for the input at row p, first occurrence first),
// each as if it were the event's target, from ONE scoring of the catalogue per event.  Included at the end of g4r_eval.cuh.
//
// The unit of work is the RankUnit of eval_rank (a mini-batch, or a ranking block of a history schedule), on the ranking stream:
//   stage  right after k_eval_tgt (before the rows' y may be overwritten): the host builds the unit's relevant lists -- per row
//          its (item, column) pairs, from the schedule's positions -- and uploads them; k_rest_thr computes every pair's
//          threshold, the relevant item's score in the sequential k order of the fp32 tile (bitwise the tile's score), with the
//          activation and the noise of its own column, and flags misses (seen, or not among the candidate items); k_rest_stage
//          keeps the rows' y, noise keys and seen-list index
//   step   after k_eval_rank: k_rest_sort orders each row's thresholds descending (misses last); each pass k of RS_P thresholds
//          per row is one sweep of the fp32 tiles (ev_tiles) over the rows that hold more than k RS_P pairs (k_rest_gather +
//          k_rest_score; on the wgmma tiles k_tc_split + k_rest_tc, where the next-item ranking takes them, with the pre-activation
//          thresholds of tc_thresholds): a competitor's score is placed among its row's thresholds by binary search and bumps a (greater,
//          equal) histogram bin in shared memory, flushed per row block; k_rest_counts prefix-sums the bins into per-pair
//          (#greater, #equal) and k_rest_sums adds the six metrics per cut-off in double, in a fixed order
// The pair counts go through a window buffer to the host (flushed when full and at the end of each staging window).
#pragma once

constexpr int RS_P = 32;                                  // thresholds per row and pass
constexpr size_t REST_WINDOW_PAIRS = (size_t)1 << 22;     // pair counts buffered on the device before a copy to the host
constexpr int REST_METRICS = 6;                           // hitrate, precision, recall, mrr, ndcg, map

struct RestCtx {
  int slot = -1;                                          // scoring descriptor of the passes: layer[last].y = dYp, wM = dMp
  float* dYa = nullptr;                                   // [Be x ldL] the unit's y rows
  float* dYp = nullptr;                                   // [Be x ldL] the rows of one pass
  int* dMp = nullptr;                                     // rows of the pass
  int* dRowKey = nullptr;                                 // [Be x 2] tiebreaking key (step, lane) of every row
  int* dRowSlot = nullptr;                                // [Be] seen-list index of every row
  int* dNv = nullptr;                                     // [Be] ranked (non-miss) pairs of every row
  int* dU = nullptr; size_t u_cap = 0;                    // uploaded unit lists: [Be + 1] offsets | [3 x pairs] pairs | pass rows
  float* dThr = nullptr; float* dSThr = nullptr; int* dPMiss = nullptr; int* dSIdx = nullptr; int* dBin = nullptr; int2* dSCnt = nullptr;
  size_t pair_cap = 0;
  // wgmma passes: pre-activation thresholds (lo, hi) per pair, unsorted and sorted; the items in sorted order; the per-pair
  // correction of the relevant item's own column
  float *dLo = nullptr, *dHi = nullptr, *dSLo = nullptr, *dSHi = nullptr; int* dSItem = nullptr; int2* dCorr = nullptr;
  size_t tc_cap = 0;
  int2* dWCnt = nullptr; size_t wcnt_cap = 0;             // window buffer of pair counts (unit pairs in schedule order)
  double* dSums = nullptr;                                // [REST_METRICS x 64]
  int* hU[2] = {nullptr, nullptr}; size_t hu_cap = 0;     // pinned host lists, alternating between units
  cudaEvent_t hu_free[2] = {nullptr, nullptr};            // the upload from hU[i] has completed
  int skip = 1;                                           // a score below the row's lowest threshold skips the search
                                                          // (G4R_REST_SEARCH_ALL=1 at creation: it is searched, for measurement)
};

// one g4r_eval_rest call
struct RestRun {
  RestCtx* x = nullptr;
  const g4r_schedule* sched = nullptr;
  int32_t* out_counts = nullptr; int64_t* out_offsets = nullptr;
  std::vector<int32_t> item;                              // item of every data row the schedule walks (-1: not walked)
  std::vector<uint8_t> has_next;                          // row p is an input (row p + 1 belongs to its session)
  std::vector<int64_t> stamp;                             // per item: last event that listed it (dedup)
  std::vector<int> first_pos;                             // candidate items: first position of each item in the list (-1: not listed)
  size_t unit_cap = 0;                                    // pairs of one unit at most (rest_walk's bound)
  int half = 0;                                           // pinned list buffer of the next unit
  int64_t ev = 0, pairs = 0;                              // events / pairs so far
  int64_t flushed = 0;                                    // pairs copied to the host so far
  size_t wused = 0;                                       // pairs in the window buffer
  int n_pass = 0, n_prow = 0;                             // current unit: passes and pass rows
  std::vector<int> pass_off;                              // [n_pass + 1] offsets of the passes' rows
  int unit_pairs = 0;
  bool tc = false;                                        // the wgmma tiles are ready (RankConsts::tc_possible): thresholds (lo, hi) kept
};

static void rest_release(EvalCtx& e) {
  if (!e.rest) return;
  RestCtx& x = *static_cast<RestCtx*>(e.rest);
  for (void* p : {(void*)x.dYa, (void*)x.dYp, (void*)x.dMp, (void*)x.dRowKey, (void*)x.dRowSlot, (void*)x.dNv, (void*)x.dU, (void*)x.dThr,
                  (void*)x.dSThr, (void*)x.dPMiss, (void*)x.dSIdx, (void*)x.dBin, (void*)x.dSCnt, (void*)x.dWCnt, (void*)x.dSums,
                  (void*)x.dLo, (void*)x.dHi, (void*)x.dSLo, (void*)x.dSHi, (void*)x.dSItem, (void*)x.dCorr})
    if (p) cudaFree(p);
  for (int i = 0; i < 2; i++) {
    if (x.hU[i]) cudaFreeHost(x.hU[i]);
    if (x.hu_free[i]) cudaEventDestroy(x.hu_free[i]);
  }
  slot_free(x.slot);
  delete static_cast<RestCtx*>(e.rest);
  e.rest = nullptr;
}

// the number of counted events and of (event, relevant item) pairs of schedule s (host only); also fills the row arrays of rr
// unit_max: the most pairs any B consecutive counted events hold (a unit -- a mini-batch or a history ranking block -- is such a run)
static int rest_walk(const g4r_schedule* s, int64_t* n_events, int64_t* n_pairs, RestRun* rr, int32_t* max_item = nullptr, int64_t* unit_max = nullptr) {
  const int B = s->B;
  int64_t rows = 0;
  for (int64_t t = 0; t < s->n_steps; t++)
    for (int b = 0; b < s->M[(size_t)t]; b++) rows = std::max<int64_t>(rows, s->P[(size_t)(t * B + b)] + 2);
  std::vector<int32_t> item((size_t)rows, -1);
  std::vector<uint8_t> nx((size_t)rows, 0);
  int32_t n_items = 0;
  for (int64_t t = 0; t < s->n_steps; t++)
    for (int b = 0; b < s->M[(size_t)t]; b++) {
      const size_t o = (size_t)(t * B + b);
      const int64_t p = s->P[o];
      item[(size_t)p] = s->X[o]; item[(size_t)p + 1] = s->Y[o]; nx[(size_t)p] = 1;
      n_items = std::max(n_items, std::max(s->X[o], s->Y[o]) + 1);
    }
  std::vector<int64_t> stamp((size_t)n_items, -1);
  int64_t ne = 0, np = 0, run = 0, best = 0;
  std::vector<int32_t> per;                       // pairs of every counted event (unit_max only)
  for (int64_t t = 0; t < s->n_steps; t++)
    for (int b = 0; b < s->M[(size_t)t]; b++) {
      const size_t o = (size_t)(t * B + b);
      if (s->hist && !(s->F[o] & 4)) continue;
      const int64_t np0 = np;
      for (int64_t q = s->P[o] + 1;; q++) {
        if (stamp[(size_t)item[(size_t)q]] != ne) { stamp[(size_t)item[(size_t)q]] = ne; np++; }
        if (!nx[(size_t)q]) break;
      }
      if (unit_max) {
        per.push_back((int32_t)(np - np0));
        run += np - np0;
        if ((int64_t)per.size() > B) run -= per[per.size() - 1 - (size_t)B];
        best = std::max(best, run);
      }
      ne++;
    }
  *n_events = ne; *n_pairs = np;
  if (unit_max) *unit_max = best;
  if (max_item) *max_item = n_items - 1;
  if (rr) { rr->item.swap(item); rr->has_next.swap(nx); }
  return G4R_OK;
}

// y rows b < M of step s into ya, the rows' noise keys and seen-list index
template <bool KEY>
__global__ void __launch_bounds__(256) k_rest_stage(int slot, int s, float* __restrict__ ya, int* __restrict__ rkey, int* __restrict__ rslot,
                                                    const int* __restrict__ key) {
  const ModelDev& md = MD;
  const int M = md.wM[s];
  const float* y = md.layer[md.n_layers - 1].y;
  const int n4 = M * md.ldL / 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) st4(ya + 4 * i, ld4(y + 4 * i));
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < M; b += gridDim.x * blockDim.x) {
    rkey[2 * b] = KEY ? key[2 * b] : s; rkey[2 * b + 1] = KEY ? key[2 * b + 1] : b;
    rslot[b] = md.wSlot[(size_t)s * md.B + b];
  }
}

// threshold of every pair p = (item, column, row): the item's score for the row as the fp32 tile computes it (ev_score_fp32),
// activation, and in tiebreaking the noise of the item's own column; miss if the column is -1 (not a candidate) or, SEEN, the
// item is on the row's seen list
// lo != nullptr (the unit's passes may take the wgmma tiles): also the pair's two pre-activation thresholds (tc_thresholds)
template <bool SEEN, bool KEY>
__global__ void __launch_bounds__(128) k_rest_thr(int slot, int s, int n_pairs, const int* __restrict__ pair, float* __restrict__ thr, int* __restrict__ pmiss,
                                                  unsigned int tie, SeenDev sd, const int* __restrict__ key, float* __restrict__ lo, float* __restrict__ hi) {
  const ModelDev& md = MD;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pairs) return;
  const int j = pair[3 * p], col = pair[3 * p + 1], b = pair[3 * p + 2];
  bool miss = col < 0;
  if (SEEN && !miss) {
    const int sl = md.wSlot[(size_t)s * md.B + b];
    miss = sorted_has(sd.list + (size_t)sl * sd.cap, sd.n[sl], j);
  }
  float sc = ev_score_fp32(md, b, j);
  const float pre = sc;
  if (md.fact.kind <= G4R_ACT_SELU) sc = act_fwd(md.fact, sc);
  if (lo) {
    float l, u;
    tc_thresholds(md.fact, md.fact.kind <= G4R_ACT_SELU, sc, pre, l, u);
    lo[p] = l; hi[p] = u;
  }
  if (tie && !miss) sc += tie_noise(tie, KEY ? key[2 * b] : s, KEY ? key[2 * b + 1] : b, (unsigned int)col);
  thr[p] = sc; pmiss[p] = miss ? 1 : 0;
}

// a total order of the thresholds (descending by value; the bit-pattern key also orders NaN)
__device__ __forceinline__ uint32_t rest_key(float f) { return tc_fkey(f); }

// row b of the unit (one CTA): its pairs off[b] .. off[b+1] in the order (threshold desc, pair asc), misses after them in pair
// order; nv[b] = ranked pairs; the pairs' histogram bins cleared.  lo != nullptr (wgmma passes): the (lo, hi) pairs and the items
// in the same order, and the corrections cleared.  Each pair's place is
// counted over the row's pairs (O(n^2 / 128) per row; a row holds at most longest session - 1 pairs)
__global__ void __launch_bounds__(128) k_rest_sort(const int* __restrict__ off, const float* __restrict__ thr, const int* __restrict__ pmiss,
                                                   float* __restrict__ sthr, int* __restrict__ sidx, int* __restrict__ nv, int* __restrict__ bins,
                                                   const int* __restrict__ pair, const float* __restrict__ lo, const float* __restrict__ hi,
                                                   float* __restrict__ slo, float* __restrict__ shi, int* __restrict__ sitem, int2* __restrict__ corr) {
  const int b = blockIdx.x, o = off[b], n = off[b + 1] - o, tid = threadIdx.x;
  __shared__ int red[4];
  int c = 0;
  for (int p = tid; p < n; p += blockDim.x) c += pmiss[o + p] ? 0 : 1;
  for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
  if ((tid & 31) == 0) red[tid >> 5] = c;
  __syncthreads();
  const int nvb = red[0] + red[1] + red[2] + red[3];
  for (int p = tid; p < n; p += blockDim.x) {
    const bool mp = pmiss[o + p] != 0;
    const uint32_t kp = rest_key(thr[o + p]);
    int r = 0;
    if (!mp) {
      for (int q = 0; q < n; q++) {
        if (pmiss[o + q]) continue;
        const uint32_t kq = rest_key(thr[o + q]);
        r += (kq > kp || (kq == kp && q < p)) ? 1 : 0;
      }
    } else {
      r = nvb;
      for (int q = 0; q < p; q++) r += pmiss[o + q] ? 1 : 0;
    }
    sthr[o + r] = thr[o + p]; sidx[o + r] = p;
    bins[2 * (o + p)] = 0; bins[2 * (o + p) + 1] = 0;
    if (lo) {
      slo[o + r] = lo[o + p]; shi[o + r] = hi[o + p];
      sitem[o + r] = pair[3 * (o + p)];
      corr[o + p] = make_int2(0, 0);
    }
  }
  if (tid == 0) nv[b] = nvb;
}

// the n rows prow[0 .. n) of ya into yp (*mp = n)
__global__ void __launch_bounds__(256) k_rest_gather(const float* __restrict__ ya, const int* __restrict__ prow, int n, int ldL, float* __restrict__ yp, int* mp) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *mp = n;
  const int kw = ldL / 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * kw; i += gridDim.x * blockDim.x) {
    const int r = i / kw, c4 = i % kw;
    st4(yp + (size_t)r * ldL + 4 * c4, ld4(ya + (size_t)prow[r] * ldL + 4 * c4));
  }
}

// Pass `pass` over the competitors (the catalogue, or the n_cand positions of `subset`) for the pass rows (row g of the
// descriptor is unit row prow[g]): the fp32 tiles of k_eval_score, and an epilogue that places every competitor's score among
// the row's thresholds pass * RS_P .. + RS_P - 1 (descending, in shared memory).  With a = #thresholds >= x and e = #thresholds
// > x, the score is greater than thresholds a .. and equal to e .. a - 1: bin a of the greater histogram and the difference
// bins e (+1) / a (-1) of the equal histogram.  A score below the row's lowest threshold (or NaN) counts nowhere and skips the
// search.  The bins are flushed to the pairs' global bins once per row block.  SEEN: the row's seen items are not compared (the
// bits of k_eval_score).  Tiebreaking noise keyed by the row's (step, lane) pair, as in the tile that ranks the next item.
constexpr int RS_BINS = RS_P + 1;
constexpr int RS_LDT = RS_P + 1;
template <bool SEEN>
__global__ void __launch_bounds__(EV_THREADS) k_rest_score(int slot, int pass, const int* __restrict__ prow, const int* __restrict__ off,
                                                           const int* __restrict__ nv, const float* __restrict__ sthr, int* bins,
                                                           const int* __restrict__ subset, int n_cand, unsigned int tie, SeenDev sd,
                                                           const int* __restrict__ rslot, const int* __restrict__ rkey, int skip) {
  const ModelDev& md = MD;
  extern __shared__ __align__(16) float smem[];
  float* sT = smem + EV_TILE_FLOATS;                                  // [EV_TB][RS_LDT] thresholds (odd stride: lanes on distinct banks)
  int* sG = reinterpret_cast<int*>(sT + EV_TB * RS_LDT);              // [EV_TB][RS_BINS] greater bins
  int* sE = sG + EV_TB * RS_BINS;                                     // [EV_TB][RS_BINS] equal difference bins
  int* sN = sE + EV_TB * RS_BINS;                                     // [EV_TB] thresholds of the row in this pass
  const int M = md.wM[0];
  const int I = n_cand > 0 ? n_cand : md.n_items;
  const int i0 = blockIdx.x * EV_IT;
  const int ni = min(EV_IT, I - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 2 * EV_TB * RS_BINS; i += EV_THREADS) sG[i] = 0;
  ev_tiles(md, smem, M, i0, ni, subset, [&](int b0, const float (&acc)[8]) {
    for (int i = tid; i < EV_TB * RS_P; i += EV_THREADS) {
      const int r = i / RS_P, k = i % RS_P, g = b0 + r;
      float v = 0.f;
      if (g < M) {
        const int ob = prow[g];
        if (k < nv[ob] - pass * RS_P) v = sthr[off[ob] + pass * RS_P + k];
      }
      sT[r * RS_LDT + k] = v;
    }
    if (tid < EV_TB) {
      const int g = b0 + tid;
      sN[tid] = g < M ? max(0, min(RS_P, nv[prow[g]] - pass * RS_P)) : 0;
    }
    __syncthreads();
    const int g = b0 + lane, n = sN[lane];
    if (g < M && n > 0) {
      const int ob = prow[g];
      const float* T = sT + lane * RS_LDT;
      const float tlow = T[n - 1];
      unsigned int xq = 0u;
      if (SEEN) {
        const int sl = rslot[ob], ns = sd.n[sl];
        const int* l = sd.list + (size_t)sl * sd.cap;
        if (subset) {
#pragma unroll
          for (int q = 0; q < 8; q++) if (warp + 8 * q < ni && sorted_has(l, ns, subset[i0 + warp + 8 * q])) xq |= 1u << q;
        } else {
          for (int p = sorted_lb(l, ns, i0); p < ns && l[p] < i0 + ni; p++) {
            const int rel = l[p] - i0;
            if ((rel & 7) == warp) xq |= 1u << (rel >> 3);
          }
        }
      }
      const int ks = rkey[2 * ob], kb = rkey[2 * ob + 1];
      int* G = sG + lane * RS_BINS;
      int* E = sE + lane * RS_BINS;
#pragma unroll
      for (int q = 0; q < 8; q++) {
        const int it = i0 + warp + 8 * q;
        if (warp + 8 * q < ni && !((xq >> q) & 1u)) {
          float sc = acc[q] + md.By[ev_item(subset, it)];
          if (md.fact.kind <= G4R_ACT_SELU) sc = act_fwd(md.fact, sc);
          if (tie) sc += tie_noise(tie, ks, kb, (unsigned int)it);
          if (sc != sc || (skip && sc < tlow)) continue;         // NaN counts nowhere; below every threshold neither
          int lo = 0, hi = n;
          while (lo < hi) { const int m = (lo + hi) >> 1; if (T[m] >= sc) lo = m + 1; else hi = m; }
          const int a = lo;
          lo = 0;
          while (lo < hi) { const int m = (lo + hi) >> 1; if (T[m] > sc) lo = m + 1; else hi = m; }
          if (a < n) atomicAdd(&G[a], 1);
          if (lo < a) { atomicAdd(&E[lo], 1); atomicAdd(&E[a], -1); }
        }
      }
    }
    __syncthreads();
    for (int i = tid; i < 2 * EV_TB * RS_BINS; i += EV_THREADS) {   // flush and clear for the next row block
      const int kind = i / (EV_TB * RS_BINS), r = (i % (EV_TB * RS_BINS)) / RS_BINS, k = i % RS_BINS;
      const int v = sG[i];
      if (v && k < sN[r]) atomicAdd(&bins[2 * (off[prow[b0 + r]] + pass * RS_P + k) + kind], v);
      sG[i] = 0;
    }
  });
}
static size_t rest_smem_bytes() { return (size_t)EV_TILE_FLOATS * sizeof(float) + EV_TB * RS_LDT * sizeof(float) + (2 * EV_TB * RS_BINS + EV_TB) * sizeof(int) + 64; }

// Pass `pass` on the wgmma tiles (tc_sweep over the pass rows' split y and the item table's split, full catalogue, no noise):
// the epilogue of k_eval_tc with many thresholds per row.  A pre-activation score x is greater than pair k's item iff x > hi_k
// and equal iff lo_k <= x <= hi_k (tc_thresholds); both are non-increasing along the sorted pairs, so a = #{k: hi_k >= x} and
// e = #{k: lo_k > x} place x exactly as the fp32 epilogue places act(x): the same bins, in shared memory after the stages,
// flushed once per lane block (the CTA's last tile of it).  The thresholds are read from global memory (L1).  A relevant item's
// own column is compared with its own thresholds by its 3xTF32 value; as in k_eval_tc it must count as exactly one tie, so the
// thread that holds it (it checks the chunk's items, at most RS_P, against its columns per tile) books the difference in the
// pair's correction.  SEEN: the
// seen columns are not placed (a seen relevant item is a miss and has no pair to correct).
template <bool SEEN>
__global__ void __launch_bounds__(TC_THREADS, 1) k_rest_tc(int slot, int pass, const int* __restrict__ prow, const int* __restrict__ off,
                                                           const int* __restrict__ nv, const float* __restrict__ slo, const float* __restrict__ shi,
                                                           const int* __restrict__ sitem, int* bins, int2* corr,
                                                           const unsigned char* __restrict__ Asplit, const unsigned char* __restrict__ Bsplit,
                                                           SeenDev sd, const int* __restrict__ rslot, int skip) {
  const ModelDev& md = MD;
  extern __shared__ __align__(1024) unsigned char tc_raw[];
  int* sG = reinterpret_cast<int*>(tc_raw + sizeof(TcSmem));          // [TC_M][RS_BINS] greater bins
  int* sE = sG + TC_M * RS_BINS;                                       // [TC_M][RS_BINS] equal difference bins
  const int M = md.wM[0], I = md.n_items, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 2 * TC_M * RS_BINS; i += TC_THREADS) sG[i] = 0;   // before tc_sweep's first barrier
  int lb0 = 0, bb[2], nb[2], base[2]; float lolast[2];
  const int* sl_l[2]; int sl_n[2], sl_p[2], sl_nx[2];                 // SEEN: as k_eval_tc
  auto lane_block = [&](int b) {
    lb0 = b - ((warp >> 2) & 1) * 64 - ((warp & 3) * 16 + (lane >> 2));
#pragma unroll
    for (int h = 0; h < 2; h++) {
      bb[h] = b + 8 * h;
      const bool v = bb[h] < M;
      const int ob = v ? prow[bb[h]] : 0;
      nb[h] = v ? max(0, min(RS_P, nv[ob] - pass * RS_P)) : 0;
      base[h] = off[ob] + pass * RS_P;
      lolast[h] = nb[h] > 0 ? slo[base[h] + nb[h] - 1] : INFINITY;
      if (SEEN) {
        const int sl = v ? rslot[ob] : 0;
        sl_l[h] = sd.list + (size_t)sl * sd.cap; sl_n[h] = v ? sd.n[sl] : 0;
        sl_p[h] = 0; sl_nx[h] = sl_n[h] > 0 ? sl_l[h][0] : INT_MAX;
      }
    }
  };
  auto tile = [&](const float (&d)[64], int c0, bool last) {
    const int n_live = I - c0;
    unsigned int xm[2] = {0u, 0u};                                     // SEEN: bit 2 (i / 4) + i % 2 of a seen column
    if (SEEN) {
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (sl_nx[h] < c0) {
          sl_p[h] += sorted_lb(sl_l[h] + sl_p[h], sl_n[h] - sl_p[h], c0);
          sl_nx[h] = sl_p[h] < sl_n[h] ? sl_l[h][sl_p[h]] : INT_MAX;
        }
        while (sl_nx[h] < c0 + 128) {
          const int rel = sl_nx[h] - c0;
          if ((rel & 7) < 2) xm[h] |= 1u << ((rel >> 3) * 2 + (rel & 1));
          sl_p[h]++;
          sl_nx[h] = sl_p[h] < sl_n[h] ? sl_l[h][sl_p[h]] : INT_MAX;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 64; i++) {
      const int h = (i >> 1) & 1;
      const float x = d[i];
      if ((i >> 2) * 8 + (i & 1) >= n_live || (SEEN && ((xm[h] >> ((i >> 2) * 2 + (i & 1))) & 1u)) || x != x || (skip && x < lolast[h])) continue;
      const float* H = shi + base[h];
      const float* L = slo + base[h];
      int lo = 0, hi = nb[h];
      while (lo < hi) { const int m = (lo + hi) >> 1; if (H[m] >= x) lo = m + 1; else hi = m; }
      const int a = lo;
      lo = 0;
      while (lo < hi) { const int m = (lo + hi) >> 1; if (L[m] > x) lo = m + 1; else hi = m; }
      const int r = bb[h] - lb0;
      if (a < nb[h]) atomicAdd(&sG[r * RS_BINS + a], 1);
      if (lo < a) { atomicAdd(&sE[r * RS_BINS + lo], 1); atomicAdd(&sE[r * RS_BINS + a], -1); }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {                                      // the rows' relevant items among the held columns
      for (int k = 0; k < nb[h]; k++) {
        const int rel = sitem[base[h] + k] - c0;
        if (rel >= 0 && rel < 128 && (rel & 7) < 2) {
          float xs = 0.f;
#pragma unroll
          for (int i = 0; i < 64; i++) if (((i >> 1) & 1) == h && (i >> 2) * 8 + (i & 1) == rel) xs = d[i];
          const float l = slo[base[h] + k], u = shi[base[h] + k];
          const int g = xs > u ? 1 : 0, e = (xs >= l && xs <= u) ? 1 : 0;
          if (g || !e) atomicAdd(&corr[base[h] + k].x, -g), atomicAdd(&corr[base[h] + k].y, 1 - e);
        }
      }
    }
    if (!last) return;
    __syncthreads();
    for (int i = tid; i < 2 * TC_M * RS_BINS; i += TC_THREADS) {      // flush and clear for the next lane block
      const int kind = i / (TC_M * RS_BINS), r = (i % (TC_M * RS_BINS)) / RS_BINS, k = i % RS_BINS, g = lb0 + r;
      const int v = sG[i];
      if (v && g < M) {
        const int ob = prow[g];
        if (k < min(RS_P, nv[ob] - pass * RS_P)) atomicAdd(&bins[2 * (off[ob] + pass * RS_P + k) + kind], v);   // bin RS_P: past the chunk
      }
      sG[i] = 0;
    }
    __syncthreads();
  };
  tc_sweep(M, I, md.L + 1, Asplit, Bsplit, lane_block, tile);
}
static size_t rest_tc_smem_bytes() { return sizeof(TcSmem) + 2 * TC_M * RS_BINS * sizeof(int); }

// every row (one CTA): the bins of each pass chunk prefix-summed into the (#greater, #equal) of the sorted pairs (scnt), and into
// the window buffer in pair order (wcnt); a miss gets (-1, -1)
// (corr != nullptr: the wgmma passes' per-pair corrections added)
__global__ void __launch_bounds__(32) k_rest_counts(const int* __restrict__ off, const int* __restrict__ nv, const int* __restrict__ sidx,
                                                    const int* __restrict__ bins, int2* __restrict__ scnt, int2* __restrict__ wcnt,
                                                    const int2* __restrict__ corr) {
  const int b = blockIdx.x, o = off[b], n = off[b + 1] - o, nvb = nv[b];
  for (int c = threadIdx.x; c * RS_P < n; c += blockDim.x) {
    int gt = 0, eq = 0;
    for (int k = c * RS_P; k < min(n, (c + 1) * RS_P); k++) {
      int2 v = make_int2(-1, -1);
      if (k < nvb) {
        gt += bins[2 * (o + k)]; eq += bins[2 * (o + k) + 1]; v = make_int2(gt, eq);
        if (corr) { v.x += corr[o + k].x; v.y += corr[o + k].y; }
      }
      scnt[o + k] = v;
      wcnt[o + sidx[o + k]] = v;
    }
  }
}

// the six metrics of the unit's M rows per cut-off, added to sums[m * n_cut + j] in double (fixed order: rows strided over the
// threads, a shuffle tree, then the warps in order).  A row's ranked pairs are in rank order (the thresholds are descending, and
// every mode's rank is non-decreasing along them), so the first gives the MRR and the count of ranks <= r_j is the end of r_j's run
__global__ void __launch_bounds__(256) k_rest_sums(int M, const int* __restrict__ off, const int* __restrict__ nv, const int2* __restrict__ scnt,
                                                   const int* __restrict__ cut, int n_cut, int mode, double* sums) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ double red[8][REST_METRICS];
  auto rank_of = [&](int2 c) -> double {
    if (mode == 1) return (double)(c.x + c.y);
    if (mode == 2) return (double)c.x + 0.5 * (double)(c.y - 1) + 1.0;
    return (double)(c.x + 1);
  };
  for (int j = 0; j < n_cut; j++) {
    const double N = (double)cut[j];
    double a[REST_METRICS] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int b = tid; b < M; b += blockDim.x) {
      const int o = off[b], n = off[b + 1] - o, nvb = nv[b];
      double hits = 0.0, dcg = 0.0, ap = 0.0, mrr = 0.0;
      for (int k = 0; k < nvb; k++) {
        const double r = rank_of(scnt[o + k]);
        if (!(r <= N)) break;
        if (k == 0) mrr = 1.0 / r;
        int e = k + 1;
        while (e < nvb && rank_of(scnt[o + e]) == r) e++;
        hits += 1.0;
        dcg += 1.0 / log2(r + 1.0);
        ap += (double)e / r;
      }
      double idcg = 0.0;
      const int m = (int)min((double)n, N);
      for (int i = 1; i <= m; i++) idcg += 1.0 / log2((double)i + 1.0);
      a[0] += hits > 0.0 ? 1.0 : 0.0;
      a[1] += hits / N;
      a[2] += hits / (double)n;
      a[3] += mrr;
      a[4] += m > 0 ? dcg / idcg : 0.0;
      a[5] += m > 0 ? ap / (double)m : 0.0;
    }
#pragma unroll
    for (int i = 0; i < REST_METRICS; i++)
      for (int d = 16; d > 0; d >>= 1) a[i] += __shfl_xor_sync(0xffffffffu, a[i], d);
    __syncthreads();
    if (lane == 0) for (int i = 0; i < REST_METRICS; i++) red[warp][i] = a[i];
    __syncthreads();
    if (tid == 0)
      for (int i = 0; i < REST_METRICS; i++) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += red[w][i];
        sums[i * n_cut + j] += t;
      }
  }
}

static int rest_ctx(g4r_handle* h, EvalCtx* e, RestCtx** out) {
  if (!e->rest) {
    const int slot = slot_alloc();
    if (slot < 0) FAIL(G4R_ERR_STATE, "too many live g4r handles in this process");
    e->rest = new RestCtx();
    RestCtx& x = *static_cast<RestCtx*>(e->rest);
    x.slot = slot;
    if (const char* v = getenv("G4R_REST_SEARCH_ALL")) x.skip = atoi(v) ? 0 : 1;
    const int Be = e->Be;
    const size_t rows = (size_t)Be * h->md.ldL;
    CK(cudaMalloc(&x.dYa, rows * sizeof(float)));
    CK(cudaMalloc(&x.dYp, rows * sizeof(float)));
    CK(cudaMalloc(&x.dMp, sizeof(int)));
    CK(cudaMalloc(&x.dRowKey, (size_t)Be * 2 * sizeof(int)));
    CK(cudaMalloc(&x.dRowSlot, (size_t)Be * sizeof(int)));
    CK(cudaMalloc(&x.dNv, (size_t)Be * sizeof(int)));
    CK(cudaMalloc(&x.dSums, (size_t)REST_METRICS * 64 * sizeof(double)));
    for (int i = 0; i < 2; i++) CK(cudaEventCreateWithFlags(&x.hu_free[i], cudaEventDisableTiming));
    ModelDev md = e->mde;
    md.layer[md.n_layers - 1].y = x.dYp;
    md.wM = x.dMp;
    CK(slot_upload(x.slot, md, h->stream));
    CK(cudaFuncSetAttribute(k_rest_score<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rest_smem_bytes()));
    CK(cudaFuncSetAttribute(k_rest_score<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rest_smem_bytes()));
    CK(cudaFuncSetAttribute(k_rest_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rest_tc_smem_bytes()));
    CK(cudaFuncSetAttribute(k_rest_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rest_tc_smem_bytes()));
  }
  *out = static_cast<RestCtx*>(e->rest);
  return G4R_OK;
}

// lists of (lanes x (longest session - 1)) int32 over the seen-list budget are refused before any device work
static int rest_budget(g4r_handle* h, const g4r_schedule* s) {
  const int64_t cap = std::max<int64_t>(1, s->max_len - 1);
  size_t budget = SEEN_BYTES;
  if (const char* b = getenv("G4R_SEEN_BUDGET")) budget = std::min<size_t>(budget, (size_t)std::max(0LL, atoll(b)));
  if ((size_t)s->B * (size_t)cap * sizeof(int) > budget) {
    char msg[256];
    snprintf(msg, sizeof msg, "eval_rest: the longest session (%lld events) needs relevant lists of %d lanes x %lld items, over the %zu-byte budget",
             (long long)s->max_len, s->B, (long long)cap, budget);
    FAIL(G4R_ERR_INVALID, msg);
  }
  return G4R_OK;
}

// the call's buffers: unit lists of up to lanes x (longest session - 1) pairs, the window buffer, the cleared sums
static int rest_begin(g4r_handle* h, EvalCtx* e, const g4r_schedule* s, RestRun* rr, int n_cut, bool tc) {
  rr->tc = tc;
  int rc = rest_ctx(h, e, &rr->x);
  if (rc) return rc;
  RestCtx* x = rr->x;
  const int Be = e->Be;
  rr->sched = s;
  int64_t ne = 0, np = 0, umax = 0;
  rc = rest_walk(s, &ne, &np, rr, nullptr, &umax);
  if (rc) return rc;
  rr->unit_cap = (size_t)std::max<int64_t>(1, umax);     // <= lanes x (longest session - 1), the budgeted bound
  const size_t up = rr->unit_cap;
  const size_t u_ints = (size_t)(Be + 1) + 3 * up + (size_t)Be + up / RS_P + 1;
  if (x->hu_cap < u_ints) {
    for (int i = 0; i < 2; i++) {
      if (x->hU[i]) { CK(cudaEventSynchronize(x->hu_free[i])); cudaFreeHost(x->hU[i]); x->hU[i] = nullptr; }
      CK(cudaMallocHost(&x->hU[i], u_ints * sizeof(int)));
    }
    x->hu_cap = u_ints;
  }
  CK(dev_grow(&x->dU, &x->u_cap, u_ints));
  if (x->pair_cap < up) {
    for (void* p : {(void*)x->dThr, (void*)x->dSThr, (void*)x->dPMiss, (void*)x->dSIdx, (void*)x->dBin, (void*)x->dSCnt}) if (p) cudaFree(p);
    x->dThr = x->dSThr = nullptr; x->dPMiss = x->dSIdx = x->dBin = nullptr; x->dSCnt = nullptr; x->pair_cap = 0;
    CK(cudaMalloc(&x->dThr, up * sizeof(float))); CK(cudaMalloc(&x->dSThr, up * sizeof(float)));
    CK(cudaMalloc(&x->dPMiss, up * sizeof(int))); CK(cudaMalloc(&x->dSIdx, up * sizeof(int)));
    CK(cudaMalloc(&x->dBin, 2 * up * sizeof(int))); CK(cudaMalloc(&x->dSCnt, up * sizeof(int2)));
    x->pair_cap = up;
  }
  if (rr->tc && x->tc_cap < up) {
    for (void* p : {(void*)x->dLo, (void*)x->dHi, (void*)x->dSLo, (void*)x->dSHi, (void*)x->dSItem, (void*)x->dCorr}) if (p) cudaFree(p);
    x->dLo = x->dHi = x->dSLo = x->dSHi = nullptr; x->dSItem = nullptr; x->dCorr = nullptr; x->tc_cap = 0;
    CK(cudaMalloc(&x->dLo, up * sizeof(float))); CK(cudaMalloc(&x->dHi, up * sizeof(float)));
    CK(cudaMalloc(&x->dSLo, up * sizeof(float))); CK(cudaMalloc(&x->dSHi, up * sizeof(float)));
    CK(cudaMalloc(&x->dSItem, up * sizeof(int))); CK(cudaMalloc(&x->dCorr, up * sizeof(int2)));
    x->tc_cap = up;
  }
  CK(dev_grow(&x->dWCnt, &x->wcnt_cap, std::max(up, std::min<size_t>((size_t)np, REST_WINDOW_PAIRS))));
  CK(cudaMemsetAsync(x->dSums, 0, (size_t)REST_METRICS * 64 * sizeof(double), h->stream));
  rr->stamp.assign((size_t)h->md.n_items, -1);
  if (e->n_cand > 0) {
    rr->first_pos.assign((size_t)h->md.n_items, -1);
    for (int i = e->n_cand - 1; i >= 0; i--) rr->first_pos[(size_t)e->hCand[(size_t)i]] = i;
  } else {
    rr->first_pos.clear();
  }
  if (rr->out_offsets) rr->out_offsets[0] = 0;
  return G4R_OK;
}

// the window buffer's pair counts to the host (the call's output), on the ranking stream
static int rest_flush(g4r_handle* h, RestRun* rr, cudaStream_t rk) {
  if (rr->wused == 0) return G4R_OK;
  if (rr->out_counts)
    CK(cudaMemcpyAsync(rr->out_counts + 2 * rr->flushed, rr->x->dWCnt, rr->wused * sizeof(int2), cudaMemcpyDeviceToHost, rk));
  CK(cudaStreamSynchronize(rk));
  rr->flushed += (int64_t)rr->wused;
  rr->wused = 0;
  return G4R_OK;
}

// unit u right after its target scores: its relevant lists built on the host and uploaded, the pair thresholds, the rows saved
static int rest_stage(g4r_handle* h, EvalCtx* e, RestRun* rr, const RankUnit& u, const RankConsts& cs, cudaStream_t rk) {
  RestCtx* x = rr->x;
  const g4r_schedule* s = rr->sched;
  const int Be = e->Be, M = u.M, B = s->B;
  const size_t up = rr->unit_cap;
  const int hf = rr->half;
  rr->half ^= 1;
  CK(cudaEventSynchronize(x->hu_free[hf]));                 // the previous upload from this buffer has completed
  int* hoff = x->hU[hf];
  int* hpair = hoff + (Be + 1);
  int* hprow = hpair + 3 * up;
  int np = 0, longest = 0;
  hoff[0] = 0;
  for (int b = 0; b < M; b++) {
    const int64_t step = u.steps ? u.steps[b] : u.step;
    const int lane = u.lanes ? u.lanes[b] : b;
    const int64_t ev = rr->ev++;
    const int np0 = np;
    for (int64_t q = s->P[(size_t)(step * B + lane)] + 1;; q++) {
      const int j = rr->item[(size_t)q];
      if (rr->stamp[(size_t)j] != ev) {
        rr->stamp[(size_t)j] = ev;
        if ((size_t)np >= up) FAIL(G4R_ERR_STATE, "eval_rest: a unit's relevant lists exceed their bound");
        hpair[3 * np] = j;
        hpair[3 * np + 1] = rr->first_pos.empty() ? j : rr->first_pos[(size_t)j];
        hpair[3 * np + 2] = b;
        np++;
      }
      if (!rr->has_next[(size_t)q]) break;
    }
    hoff[b + 1] = np;
    longest = std::max(longest, np - np0);
    if (rr->out_offsets) rr->out_offsets[ev + 1] = rr->out_offsets[ev] + (np - np0);
  }
  rr->pairs += np;
  rr->unit_pairs = np;
  // pass k ranks thresholds k RS_P .. of the rows that hold more than k RS_P pairs (pass 0: every row)
  rr->n_pass = (longest + RS_P - 1) / RS_P;
  rr->pass_off.assign((size_t)rr->n_pass + 1, 0);
  int n_prow = 0;
  for (int k = 0; k < rr->n_pass; k++) {
    for (int b = 0; b < M; b++) if (hoff[b + 1] - hoff[b] > k * RS_P) hprow[n_prow++] = b;
    rr->pass_off[(size_t)k + 1] = n_prow;
  }
  rr->n_prow = n_prow;
  int* dOff = x->dU;
  int* dPair = dOff + (Be + 1);
  int* dProw = dPair + 3 * up;
  CK(cudaMemcpyAsync(dOff, hoff, (size_t)(M + 1) * sizeof(int), cudaMemcpyHostToDevice, rk));
  if (np) CK(cudaMemcpyAsync(dPair, hpair, (size_t)np * 3 * sizeof(int), cudaMemcpyHostToDevice, rk));
  if (n_prow) CK(cudaMemcpyAsync(dProw, hprow, (size_t)n_prow * sizeof(int), cudaMemcpyHostToDevice, rk));
  CK(cudaEventRecord(x->hu_free[hf], rk));
  const bool seen = u.sd.list != nullptr, key = u.key != nullptr;
  const unsigned int tie = cs.tie;
  if (np) {
    auto thr = seen ? (key ? k_rest_thr<true, true> : k_rest_thr<true, false>) : (key ? k_rest_thr<false, true> : k_rest_thr<false, false>);
    thr<<<(np + 127) / 128, 128, 0, rk>>>(u.slot, u.s, np, dPair, x->dThr, x->dPMiss, tie, u.sd, u.key, rr->tc ? x->dLo : nullptr, x->dHi);
    h->launches++;
  }
  const size_t rows = (size_t)M * h->md.ldL;
  (key ? k_rest_stage<true> : k_rest_stage<false>)<<<std::max(1, std::min<int>((int)((rows / 4 + 255) / 256), 2 * h->n_sm)), 256, 0, rk>>>(
      u.slot, u.s, x->dYa, x->dRowKey, x->dRowSlot, u.key);
  h->launches++;
  return G4R_OK;
}

// unit u after k_eval_rank: sort, the passes over the competitors, the pair counts and the metric sums
static int rest_step(g4r_handle* h, EvalCtx* e, RestRun* rr, const RankUnit& u, const RankConsts& cs, cudaStream_t rk) {
  RestCtx* x = rr->x;
  const int Be = e->Be, M = u.M, np = rr->unit_pairs;
  const size_t up = rr->unit_cap;
  if (M == 0) return G4R_OK;
  if (rr->wused + (size_t)np > x->wcnt_cap) {
    int rc = rest_flush(h, rr, rk);
    if (rc) return rc;
  }
  int* dOff = x->dU;
  int* dProw = dOff + (Be + 1) + 3 * up;
  const bool seen = u.sd.list != nullptr;
  int* dPair = dOff + (Be + 1);
  k_rest_sort<<<M, 128, 0, rk>>>(dOff, x->dThr, x->dPMiss, x->dSThr, x->dSIdx, x->dNv, x->dBin, dPair, rr->tc ? x->dLo : nullptr, x->dHi,
                                 x->dSLo, x->dSHi, x->dSItem, x->dCorr);
  h->launches++;
  const int I = h->md.n_items, n_comp = e->n_cand > 0 ? e->n_cand : I;
  for (int k = 0; k < rr->n_pass; k++) {
    const int n = rr->pass_off[(size_t)k + 1] - rr->pass_off[(size_t)k];
    const int* prow = dProw + rr->pass_off[(size_t)k];
    k_rest_gather<<<std::max(1, std::min(2 * h->n_sm, (n * h->md.ldL / 4 + 255) / 256)), 256, 0, rk>>>(x->dYa, prow, n, h->md.ldL, x->dYp, x->dMp);
    if (rr->tc && wgmma_tiles(h->cfg, n, I, I)) {        // the tile choice of the next-item ranking, for the pass's rows
      const int tc_chunks = (h->md.L + 1 + TC_KC - 1) / TC_KC, tc_tiles = (I + TC_N - 1) / TC_N;
      k_tc_split<TC_M><<<dim3((n + TC_M - 1) / TC_M, tc_chunks), 256, 0, rk>>>(x->dYp, n, h->md.ldL, h->md.L, e->dAsplit, tc_chunks, nullptr, 1.0f);
      (seen ? k_rest_tc<true> : k_rest_tc<false>)<<<std::min(tc_tiles, h->n_sm), TC_THREADS, rest_tc_smem_bytes(), rk>>>(
          x->slot, k, prow, dOff, x->dNv, x->dSLo, x->dSHi, x->dSItem, x->dBin, x->dCorr, e->dAsplit, e->dBsplit, u.sd, x->dRowSlot, x->skip);
      h->launches += 3;
    } else {
      (seen ? k_rest_score<true> : k_rest_score<false>)<<<(n_comp + EV_IT - 1) / EV_IT, EV_THREADS, rest_smem_bytes(), rk>>>(
          x->slot, k, prow, dOff, x->dNv, x->dSThr, x->dBin, e->n_cand > 0 ? e->dCand : nullptr, e->n_cand, cs.tie, u.sd, x->dRowSlot, x->dRowKey, x->skip);
      h->launches += 2;
    }
  }
  k_rest_counts<<<M, 32, 0, rk>>>(dOff, x->dNv, x->dSIdx, x->dBin, x->dSCnt, x->dWCnt + rr->wused, rr->tc ? x->dCorr : nullptr);
  k_rest_sums<<<1, 256, 0, rk>>>(M, dOff, x->dNv, x->dSCnt, e->dCut, cs.n_cut, cs.mode, x->dSums);
  h->launches += 2;
  rr->wused += (size_t)np;
  CK(cudaGetLastError());
  return G4R_OK;
}

extern "C" int g4r_eval_rest_pairs(const g4r_schedule* s, int64_t* n_events, int64_t* n_pairs) {
  if (!s || !n_events || !n_pairs) return G4R_ERR_INVALID;
  if (!s->has_pos) { g_create_error = "g4r_eval_rest_pairs: the schedule was not built with mode 1 | G4R_SCHED_POSITIONS"; return G4R_ERR_STATE; }
  return rest_walk(s, n_events, n_pairs, nullptr);
}

extern "C" int g4r_eval_rest(g4r_handle* h, const g4r_schedule* s, const int32_t* cut_off, int32_t n_cut, int32_t mode, double* sums_out,
                             int64_t* n_events, int64_t* n_pairs, int32_t* out_counts, int64_t* out_offsets) {
  if (!h || !s || !cut_off || n_cut <= 0 || n_cut > 64 || !sums_out) return G4R_ERR_INVALID;
  if (!s->has_pos) FAIL(G4R_ERR_STATE, "eval_rest: the schedule was not built with mode 1 | G4R_SCHED_POSITIONS");
  for (int j = 0; j < n_cut; j++) if (cut_off[j] <= 0) FAIL(G4R_ERR_INVALID, "eval_rest: cut-offs must be positive");
  int rc = rest_budget(h, s);
  if (rc) return rc;
  int64_t ne = 0, np = 0; int32_t top = -1;
  rest_walk(s, &ne, &np, nullptr, &top);
  if (top >= h->md.n_items) FAIL(G4R_ERR_INDEX, "Index out of bounds");
  RestRun rr;
  rr.out_counts = out_counts; rr.out_offsets = out_offsets;
  std::vector<double> rec((size_t)n_cut), mrr((size_t)n_cut);
  rc = eval_run(h, s, cut_off, n_cut, mode, rec.data(), mrr.data(), nullptr, nullptr, &rr);
  if (rc) return rc;
  std::vector<double> sums((size_t)REST_METRICS * 64);
  CK(cudaMemcpy(sums.data(), rr.x->dSums, sums.size() * sizeof(double), cudaMemcpyDeviceToHost));
  for (int i = 0; i < REST_METRICS; i++) for (int j = 0; j < n_cut; j++) sums_out[i * n_cut + j] = sums[(size_t)i * n_cut + j];
  if (n_events) *n_events = rr.ev;
  if (n_pairs) *n_pairs = rr.pairs;
  return G4R_OK;
}
