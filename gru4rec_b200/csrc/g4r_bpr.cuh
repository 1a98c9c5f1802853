// g4r_bpr.cuh -- BPR-MF of the reference's baselines.py (BPR, baselines.py:303-418) on the device (DESIGN §3k): the fit as a
// dataflow SGD that applies the reference's updates in its order and equals a strictly sequential run bit for bit, and the
// scoring of evaluate_gpu / evaluate_events (session vectors, float64 score tiles fused with the rank counts, the exclude_seen
// uncount, top-k lists).  Included at the end of g4r_lib.cu after g4r_baselines.cuh (the handle, k_bl_sums, bl_noise,
// cta_bitonic) and g4r_persistent.cuh (ld_acquire_u32).
#pragma once
#include <cub/device/device_radix_sort.cuh>

constexpr int BPR_WARPS = 8;                             // warps per CTA of k_bpr_sgd
constexpr int BPR_WARPS_PER_SM = 4;                      // k_bpr_sgd runs at most this many warps per SM: more only add polling
constexpr unsigned long long BPR_WAIT_NS = 5000000000ull; // a predecessor wait longer than this fails the iteration
constexpr size_t BPR_SCRATCH = (size_t)512 << 20;        // evaluation: session vectors, or scores of a block of events
constexpr size_t BPR_ROW_BYTES = 4 * 4 + 3 * 8 * 2 + 3 * 4 + 4 + 4 + 8;   // the fit's device bytes per training row (92)
constexpr int BT_E = 64, BT_J = 64, BT_K = 16;           // score tile: events x items x factors per shared-memory stage
static_assert(BT_E == BT_J, "k_bpr_tile stages both operands with one loop");

// ---------------------------------------------------------------------------------------------------------------------------
// the fit
// ---------------------------------------------------------------------------------------------------------------------------
// the touches of event t (position in the iteration's order): U row u, I rows p and n (one touch when p == n).  Key (row, t)
// with the item rows after the S session rows; p == n leaves a key past every row, which k_bpr_preds skips.
__global__ void k_bpr_keys(const int* perm, const int* neg, const int* rowS, const int* rowI, int N, unsigned S, unsigned n_rows_all,
                           unsigned long long* keys) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N) return;
  const int e = perm[t];
  const unsigned u = (unsigned)rowS[e], p = (unsigned)rowI[e], n = (unsigned)rowI[neg[t]];
  keys[3 * (size_t)t] = ((unsigned long long)u << 32) | (unsigned)t;
  keys[3 * (size_t)t + 1] = ((unsigned long long)(S + p) << 32) | (unsigned)t;
  keys[3 * (size_t)t + 2] = ((unsigned long long)(n == p ? n_rows_all : S + n) << 32) | (unsigned)t;
}

// sorted keys -> per event and touched row the last earlier event that touched the same row (-1: none), slot 0 U, 1 I[p], 2 I[n]
__global__ void k_bpr_preds(const unsigned long long* srt, long long M, const int* perm, const int* rowI, unsigned S, unsigned n_rows_all,
                            int* pred) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= M) return;
  const unsigned long long key = srt[q];
  const unsigned row = (unsigned)(key >> 32);
  if (row >= n_rows_all) return;
  const int t = (int)(key & 0xffffffffu);
  const int prev = (q > 0 && (unsigned)(srt[q - 1] >> 32) == row) ? (int)(srt[q - 1] & 0xffffffffu) : -1;
  const int slot = row < S ? 0 : (row - S == (unsigned)rowI[perm[t]] ? 1 : 2);
  pred[3 * (size_t)t + slot] = prev;
}

struct BprFitDev {
  const int* perm; const int* neg; const int* rowS; const int* rowI; const int* pred;
  double* U; double* I; const double* bI;
  unsigned* flag; int* level; double* lsig;
  int* next; int* max_level; int* fail;
  int N, F; unsigned tag;
  double lr, ls, li;
};

// a fixed shuffle tree over the lanes' partial sums: every lane ends with the same value (x + y == y + x bitwise)
__device__ __forceinline__ double bpr_warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void st_release_gpu_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// One warp per event, claimed in position order.  Lanes 0 .. 2 wait (gpu-scope acquire) until the flags of the event's at most
// three predecessors carry this iteration's tag; the warp applies the reference's update in float64, writes its level and
// publishes its own flag (gpu-scope release after a warp barrier, which orders every lane's row stores before it).  Every
// predecessor lies earlier in the order, so a warp that is already running claimed it: the wait cannot deadlock.  A wait past
// BPR_WAIT_NS sets *fail and every warp leaves.  NV > 0: F <= 32 NV and each lane keeps its elements of the three rows in
// registers between the dots and the update; NV = 0: any F, the rows are read twice.  The arithmetic is the same either way.
template <int NV>
__global__ void __launch_bounds__(BPR_WARPS * 32) k_bpr_sgd(BprFitDev d, int max_warps) {
  const int lane = threadIdx.x & 31;
  if (blockIdx.x * BPR_WARPS + (threadIdx.x >> 5) >= max_warps) return;
  const int F = d.F;
  for (;;) {
    int t = 0;
    if (lane == 0) t = atomicAdd(d.next, 1);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= d.N) return;
    const int e = d.perm[t];
    const int u = d.rowS[e], p = d.rowI[e], n = d.rowI[d.neg[t]];
    const int myq = lane < 3 ? d.pred[3 * (size_t)t + lane] : -1;
    const double bp = d.bI[p], bn = d.bI[n];
    unsigned long long t0 = 0;
    if (lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (int spin = 0;; spin++) {
      const bool ok = myq < 0 || ld_acquire_u32(d.flag + myq) == d.tag;
      if (__all_sync(0xffffffffu, ok)) break;
      int stop = 0;
      if (lane == 0) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        if (now - t0 > 1000000ull && *(volatile int*)d.fail) stop = 1;
        else if (now - t0 > BPR_WAIT_NS) { atomicExch(d.fail, 1); stop = 1; }
      }
      if (__shfl_sync(0xffffffffu, stop, 0)) return;
      if (spin >= 16) __nanosleep(64);
    }
    __syncwarp();
    const int lvp = myq >= 0 ? __ldcg(d.level + myq) : 0;
    double* Uu = d.U + (size_t)u * F;
    double* Ip = d.I + (size_t)p * F;
    double* In = d.I + (size_t)n * F;
    double s1 = 0.0, s2 = 0.0;
    double ru[NV > 0 ? NV : 1], ra[NV > 0 ? NV : 1], rb[NV > 0 ? NV : 1];
    if (NV > 0) {
#pragma unroll
      for (int v = 0; v < NV; v++) {
        const int f = lane + 32 * v;
        ru[v] = f < F ? __ldcg(Uu + f) : 0.0; ra[v] = f < F ? __ldcg(Ip + f) : 0.0; rb[v] = f < F ? __ldcg(In + f) : 0.0;
      }
#pragma unroll
      for (int v = 0; v < NV; v++)
        if (lane + 32 * v < F) { s1 = __dadd_rn(s1, __dmul_rn(ra[v], ru[v])); s2 = __dadd_rn(s2, __dmul_rn(rb[v], ru[v])); }
    } else {
      for (int f = lane; f < F; f += 32) {
        const double uf = __ldcg(Uu + f);
        s1 = __dadd_rn(s1, __dmul_rn(__ldcg(Ip + f), uf));
        s2 = __dadd_rn(s2, __dmul_rn(__ldcg(In + f), uf));
      }
    }
    s1 = bpr_warp_sum(s1);
    s2 = bpr_warp_sum(s2);
    const double x = __dsub_rn(__dadd_rn(__dsub_rn(s1, s2), bp), bn);
    const double sg = __ddiv_rn(1.0, __dadd_rn(1.0, exp(-x)));
    const double c = __dsub_rn(1.0, sg);
#pragma unroll
    for (int v = 0; v < (NV > 0 ? NV : 1); v++) {
      for (int f = lane + 32 * v; f < F; f += (NV > 0 ? F : 32)) {   // NV > 0: once, at f = lane + 32 v; else every lane's f
        const double uf = NV > 0 ? ru[v] : __ldcg(Uu + f), a = NV > 0 ? ra[v] : __ldcg(Ip + f), b = NV > 0 ? rb[v] : __ldcg(In + f);
        const double du = __dmul_rn(d.lr, __dsub_rn(__dmul_rn(c, __dsub_rn(a, b)), __dmul_rn(d.ls, uf)));
        const double dp = __dmul_rn(d.lr, __dsub_rn(__dmul_rn(c, uf), __dmul_rn(d.li, a)));
        const double dn = __dmul_rn(d.lr, __dsub_rn(__dmul_rn(-c, uf), __dmul_rn(d.li, b)));
        __stcg(Uu + f, __dadd_rn(uf, du));
        if (p == n) __stcg(Ip + f, __dadd_rn(__dadd_rn(a, dp), dn));   // the second add lands on the row the first changed
        else { __stcg(Ip + f, __dadd_rn(a, dp)); __stcg(In + f, __dadd_rn(b, dn)); }
      }
    }
    const int lv = 1 + max(max(__shfl_sync(0xffffffffu, lvp, 0), __shfl_sync(0xffffffffu, lvp, 1)), __shfl_sync(0xffffffffu, lvp, 2));
    if (lane == 0) __stcg(d.level + t, lv);
    __syncwarp();
    if (lane == 0) {
      st_release_gpu_u32(d.flag + t, d.tag);
      d.lsig[t] = log(sg);                                 // off the chain: no successor reads these
      atomicMax(d.max_level, lv);
    }
  }
}

// mean of the iteration's log sigm in a fixed order (one block)
__global__ void __launch_bounds__(1024) k_bpr_mean(const double* v, int N, double* out) {
  __shared__ double red[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double s = 0.0;
  for (int t = tid; t < N; t += 1024) s = __dadd_rn(s, v[t]);
  s = bpr_warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (tid == 0) {
    double a = 0.0;
    for (int w = 0; w < 32; w++) a = __dadd_rn(a, red[w]);
    *out = __ddiv_rn(a, (double)N);
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// scoring: score(j | uF) = (sum over f = 0 .. F-1 in order of I[j, f] * uF[f], each product and sum correctly rounded) + bI[j]
// ---------------------------------------------------------------------------------------------------------------------------
struct BprEvalDev {
  const int* items; const int64_t* off; const int* nh; const int64_t* ev0;
  const double* I; const double* bI; int F, n_items, mode, exclude, k;
  const int* comp; const int* mult; int n_comp;          // competitors: the distinct candidates ascending (NULL: every item)
  const unsigned char* first;                            // first[p]: items[p] does not occur earlier in its session
  long long E0; int nb;                                  // the block: counted events E0 .. E0 + nb
  double* uvec; int64_t* pos; int64_t* st; double* tsc;  // per block event: session vector, input position, session start, target score
  int* counts; double* scores;                           // counts [2 x all counted events]; scores [nb x n_comp] (lists only)
  int* out_items; double* out_scores;                    // [all counted events x k]
};

__device__ __forceinline__ double bpr_dot(const double* a, const double* b, int F) {
  double s = 0.0;
  for (int f = 0; f < F; f++) s = __dadd_rn(s, __dmul_rn(a[f], b[f]));
  return s;
}
// the value an event compares: the score, plus the event's noise in 'tiebreaking'
__device__ __forceinline__ double bpr_cmp(const BprEvalDev& d, double sc, long long e, int j) {
  return d.mode == 3 ? __dadd_rn(sc, bl_noise(e, j)) : sc;
}

// first-occurrence flags of every session's positions (warp per session).  O(L^2 / 32) lane steps for a session of L events, as
// k_bpr_seen's uncount is O(L F) per counted event: exclude_seen costs O(L^2 F) per session (DESIGN §3k, limits)
__global__ void __launch_bounds__(256) k_bpr_first(const int* items, const int64_t* off, int64_t S, unsigned char* first) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  const int64_t st = off[s], en = off[s + 1];
  for (int64_t q = st + lane; q < en; q += 32) {
    const int x = items[q];
    bool f = true;
    for (int64_t r = st; r < q && f; r++) f = items[r] != x;
    first[q] = f ? 1 : 0;
  }
}

// warp per session s0 .. s1: the running float64 sum of its input rows, uF = sum / (inputs so far) for every counted event of
// the block; lanes over the factors, each a sequential sum over the positions
__global__ void __launch_bounds__(256) k_bpr_uvec(BprEvalDev d, int64_t s0, int64_t s1) {
  const int lane = threadIdx.x & 31;
  const int64_t s = s0 + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= s1) return;
  const int64_t st = d.off[s], en = d.off[s + 1];
  const int64_t p0 = st + max(d.nh ? d.nh[s] : 0, 1) - 1;
  const long long e0 = d.ev0[s];
  const int F = d.F;
  for (int f = lane; f < F; f += 32) {
    double acc = 0.0;
    for (int64_t p = st; p + 1 < en; p++) {
      const long long e = e0 + (p - p0);
      if (p >= p0 && e >= d.E0 + d.nb) break;
      acc = __dadd_rn(acc, d.I[(size_t)d.items[p] * F + f]);
      if (p < p0 || e < d.E0) continue;
      d.uvec[(size_t)(e - d.E0) * F + f] = __ddiv_rn(acc, (double)(p - st + 1));
      if (f == lane && lane == 0) { d.pos[e - d.E0] = p; d.st[e - d.E0] = st; }
    }
  }
}

// NARM (g4r_narm.cuh): as k_bpr_uvec, with each counted event's vector the encoder's q[e] (float32, converted exactly)
__global__ void __launch_bounds__(256) k_narm_uvec(BprEvalDev d, const float* qev, int64_t s0, int64_t s1) {
  const int lane = threadIdx.x & 31;
  const int64_t s = s0 + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= s1) return;
  const int64_t st = d.off[s], en = d.off[s + 1];
  const int64_t p0 = st + max(d.nh ? d.nh[s] : 0, 1) - 1;
  const long long e0 = d.ev0[s];
  for (int64_t p = p0; p + 1 < en; p++) {
    const long long e = e0 + (p - p0);
    if (e >= d.E0 + d.nb) break;
    if (e < d.E0) continue;
    for (int f = lane; f < d.F; f += 32) d.uvec[(size_t)(e - d.E0) * d.F + f] = (double)qev[(size_t)e * d.F + f];
    if (lane == 0) { d.pos[e - d.E0] = p; d.st[e - d.E0] = st; }
  }
}

// thread per block event: the target's compared value, by the function the tile uses
__global__ void k_bpr_target(BprEvalDev d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.nb) return;
  const int y = d.items[d.pos[i] + 1];
  const double sc = __dadd_rn(bpr_dot(d.I + (size_t)y * d.F, d.uvec + (size_t)i * d.F, d.F), d.bI[y]);
  d.tsc[i] = bpr_cmp(d, sc, d.E0 + i, y);
}

// Score tile: BT_E events x BT_J competitors per pass, 4 x 4 per thread, the factors staged BT_K at a time; blockIdx.y takes a
// contiguous range of competitor tiles.  Each score is one thread's sequential sum over f; the (#greater, #equal) against the
// event's target are summed in registers and added with integer atomics.  LISTS: the scores also go to the block's scratch.
template <bool LISTS>
__global__ void __launch_bounds__(256) k_bpr_tile(BprEvalDev d, int tiles_per_chunk) {
  __shared__ double sU[BT_E][BT_K + 1];
  __shared__ double sI[BT_J][BT_K + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int eb = blockIdx.x * BT_E;
  const int F = d.F;
  int gt[4] = {0, 0, 0, 0}, eq[4] = {0, 0, 0, 0};
  double tv[4];
  for (int r = 0; r < 4; r++) tv[r] = eb + ty + 16 * r < d.nb ? d.tsc[eb + ty + 16 * r] : 0.0;
  const int n_tiles = (d.n_comp + BT_J - 1) / BT_J;
  const int t_end = min(n_tiles, (blockIdx.y + 1) * tiles_per_chunk);
  for (int tj = blockIdx.y * tiles_per_chunk; tj < t_end; tj++) {
    const int q0 = tj * BT_J;
    double acc[4][4];
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) acc[r][c] = 0.0;
    for (int k0 = 0; k0 < F; k0 += BT_K) {
      __syncthreads();
      for (int x = tid; x < BT_E * BT_K; x += 256) {
        const int r = x / BT_K, kk = x % BT_K, ev = eb + r, f = k0 + kk;
        sU[r][kk] = (ev < d.nb && f < F) ? d.uvec[(size_t)ev * F + f] : 0.0;
        const int q = q0 + r;
        const int j = q < d.n_comp ? (d.comp ? d.comp[q] : q) : -1;
        sI[r][kk] = (j >= 0 && f < F) ? d.I[(size_t)j * F + f] : 0.0;
      }
      __syncthreads();
      const int kn = min(BT_K, F - k0);
      for (int kk = 0; kk < kn; kk++) {
        double a[4], b[4];
        for (int r = 0; r < 4; r++) a[r] = sU[ty + 16 * r][kk];
        for (int c = 0; c < 4; c++) b[c] = sI[tx + 16 * c][kk];
        for (int r = 0; r < 4; r++)
          for (int c = 0; c < 4; c++) acc[r][c] = __dadd_rn(acc[r][c], __dmul_rn(b[c], a[r]));
      }
    }
    for (int c = 0; c < 4; c++) {
      const int q = q0 + tx + 16 * c;
      if (q >= d.n_comp) continue;
      const int j = d.comp ? d.comp[q] : q;
      const int w = d.mult ? d.mult[j] : 1;
      const double bj = d.bI[j];
      for (int r = 0; r < 4; r++) {
        const int ev = eb + ty + 16 * r;
        if (ev >= d.nb) continue;
        const double sc = __dadd_rn(acc[r][c], bj);
        if (LISTS) d.scores[(size_t)ev * d.n_comp + q] = sc;
        const double v = bpr_cmp(d, sc, d.E0 + ev, j);
        gt[r] += v > tv[r] ? w : 0;
        eq[r] += v == tv[r] ? w : 0;
      }
    }
  }
  for (int r = 0; r < 4; r++) {
    for (int o = 8; o > 0; o >>= 1) { gt[r] += __shfl_xor_sync(0xffffffffu, gt[r], o); eq[r] += __shfl_xor_sync(0xffffffffu, eq[r], o); }
    const int ev = eb + ty + 16 * r;
    if (tx == 0 && ev < d.nb && (gt[r] || eq[r])) {
      atomicAdd(d.counts + 2 * (d.E0 + ev), gt[r]);
      atomicAdd(d.counts + 2 * (d.E0 + ev) + 1, eq[r]);
    }
  }
}

// exclude_seen, warp per block event: takes back out what the tile counted for the session's distinct items so far (from the
// same score values), marks them ineligible in the list scratch (NaN), and writes (-1, -1) when the target is among them
template <bool LISTS>
__global__ void __launch_bounds__(256) k_bpr_seen(BprEvalDev d) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= d.nb) return;
  const int64_t st = d.st[i], p = d.pos[i];
  const int y = d.items[p + 1];
  const double t = d.tsc[i];
  const long long e = d.E0 + i;
  int gt = 0, eq = 0, miss = 0;
  for (int64_t r = st + lane; r <= p; r += 32) {
    const int j = d.items[r];
    miss |= j == y;
    if (!d.first[r]) continue;
    int q = j;
    if (d.comp) {
      if (d.mult[j] == 0) continue;
      q = sorted_lb(d.comp, d.n_comp, j);
    }
    const int w = d.mult ? d.mult[j] : 1;
    const double sc = __dadd_rn(bpr_dot(d.I + (size_t)j * d.F, d.uvec + (size_t)i * d.F, d.F), d.bI[j]);
    const double v = bpr_cmp(d, sc, e, j);
    gt += v > t ? w : 0;
    eq += v == t ? w : 0;
    if (LISTS) d.scores[(size_t)i * d.n_comp + q] = __longlong_as_double(0x7ff8000000000000ll);
  }
  for (int o = 16; o > 0; o >>= 1) {
    gt += __shfl_xor_sync(0xffffffffu, gt, o); eq += __shfl_xor_sync(0xffffffffu, eq, o); miss |= __shfl_xor_sync(0xffffffffu, miss, o);
  }
  if (lane == 0) {
    int* c = d.counts + 2 * e;
    if (miss) { c[0] = -1; c[1] = -1; }
    else { c[0] -= gt; c[1] -= eq; }
  }
}

// order-preserving key of a float64 score (+0 and -0 alike); NaN marks an ineligible competitor
__device__ __forceinline__ unsigned long long bpr_key(double s) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(__dadd_rn(s, 0.0));
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// CTA per block event: the k best eligible competitors by (score desc, index asc) -- a radix select on (key, then competitor
// position, which orders like the item index), the selected entries sorted in shared memory; padded with -1 / NaN
__global__ void __launch_bounds__(KF_THREADS) k_bpr_select(BprEvalDev d) {
  __shared__ double sKs[KF_KEEP_MAX];
  __shared__ int sKi[KF_KEEP_MAX];
  __shared__ unsigned sHist[256];
  __shared__ int sBin, sNeed, sFull, sN, sKn;
  const int i = blockIdx.x, tid = threadIdx.x, K = d.k, NC = d.n_comp;
  const double* row = d.scores + (size_t)i * NC;
  if (tid == 0) { sN = 0; sKn = 0; }
  __syncthreads();
  int ne = 0;
  for (int q = tid; q < NC; q += KF_THREADS) ne += isnan(row[q]) ? 0 : 1;
  atomicAdd(&sN, ne);
  __syncthreads();
  const int n_el = sN;
  unsigned long long prefix = 0ull, mask = 0ull;
  unsigned jprefix = 0u, jmask = 0u;
  int need = K, full = 1;
  if (n_el > K) {
    full = 0;
    for (int shift = 56; shift >= 0 && !full; shift -= 8) {
      for (int q = tid; q < 256; q += KF_THREADS) sHist[q] = 0u;
      __syncthreads();
      for (int q = tid; q < NC; q += KF_THREADS) {
        const double s = row[q];
        if (isnan(s)) continue;
        const unsigned long long key = bpr_key(s);
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
    if (!full) {                                         // keys equal to the boundary key: the `need` smallest positions
      for (int shift = 24; shift >= 0 && !full; shift -= 8) {
        for (int q = tid; q < 256; q += KF_THREADS) sHist[q] = 0u;
        __syncthreads();
        for (int q = tid; q < NC; q += KF_THREADS) {
          const double s = row[q];
          if (!isnan(s) && bpr_key(s) == prefix && ((unsigned)q & jmask) == jprefix) atomicAdd(&sHist[((unsigned)q >> shift) & 255u], 1u);
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
  for (int q = tid; q < NC; q += KF_THREADS) {
    const double s = row[q];
    if (isnan(s)) continue;
    bool keep = true;
    if (n_el > K) {
      const unsigned long long key = bpr_key(s) & mask;
      keep = key > prefix || (key == prefix && (jmask == 0u || ((unsigned)q & jmask) <= jprefix));
    }
    if (keep) { const int x = atomicAdd(&sKn, 1); sKs[x] = s; sKi[x] = d.comp ? d.comp[q] : q; }
  }
  __syncthreads();
  const int n = sKn;
  int P = 1;
  while (P < n) P <<= 1;
  for (int q = n + tid; q < P; q += KF_THREADS) { sKs[q] = -INFINITY; sKi[q] = 0x7fffffff; }
  cta_bitonic<false>(sKs, sKi, P);
  const long long e = d.E0 + i;
  for (int q = tid; q < K; q += KF_THREADS) {
    d.out_items[(size_t)e * K + q] = q < n ? sKi[q] : -1;
    d.out_scores[(size_t)e * K + q] = q < n ? sKs[q] : __longlong_as_double(0x7ff8000000000000ll);
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// C ABI (include/g4r.h)
// ---------------------------------------------------------------------------------------------------------------------------
static bool bpr_finite(const double* v, size_t n) {
  for (size_t i = 0; i < n; i++) if (!std::isfinite(v[i])) return false;
  return true;
}

static void bpr_free_fit(g4r_baselines* h) {
  for (void* p : h->bpr_mem) cudaFree(p);
  h->bpr_mem.clear();
  h->dU = nullptr; h->dRowS = h->dRowI = h->dPerm = h->dNeg = h->dPred = h->dLevel = h->dCtr = nullptr;
  h->dKeys = h->dKeys2 = nullptr; h->dFlag = nullptr; h->dLsig = nullptr; h->dCub = nullptr;
  h->bpr_rows = 0; h->bpr_sessions = 0; h->bpr_cub_bytes = 0;
}

template <class T>
static cudaError_t bpr_take(g4r_baselines* h, T** p, size_t n) {
  cudaError_t e = bl_alloc(p, n);
  if (e == cudaSuccess) h->bpr_mem.push_back(*p); else *p = nullptr;
  return e;
}

extern "C" int g4r_bl_bpr_begin(g4r_baselines* h, const int32_t* row_session, const int32_t* row_item, int64_t n_rows, int64_t n_sessions,
                                const double* U, const double* I, const double* bI) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BPR) FAIL(G4R_ERR_STATE, "g4r_bl_bpr_begin: the handle is not a BPR");
  if (!row_session || !row_item || !U || !I || !bI || n_rows < 1 || n_sessions < 1)
    FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_begin: null argument, or no rows / sessions");
  const int NI = h->n_items, F = h->n_keep;
  if (n_rows > INT32_MAX / 3 || n_sessions >= INT32_MAX || (uint64_t)n_sessions + (uint64_t)NI >= 0xffffffffull)
    FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_begin: need n_rows <= (2^31 - 1) / 3, n_sessions < 2^31 - 1 and n_sessions + n_items < 2^32 - 1");
  // a negative draw is a row index below n_items (the reference's randint(n_items)): every such row must exist
  if (n_rows < NI) FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_begin: need n_rows >= n_items (the negative draws index rows below n_items)");
  for (int64_t r = 0; r < n_rows; r++) {
    if (row_session[r] < 0 || row_session[r] >= n_sessions) FAIL(G4R_ERR_INDEX, "g4r_bl_bpr_begin: session index out of range");
    if (row_item[r] < 0 || row_item[r] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_bpr_begin: item index out of range");
  }
  if (!bpr_finite(U, (size_t)n_sessions * F) || !bpr_finite(I, (size_t)NI * F) || !bpr_finite(bI, NI))
    FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_begin: U, I and bI must be finite");
  const size_t N = (size_t)n_rows;
  const unsigned long long rows_all = (unsigned long long)n_sessions + NI;      // keys: (row, position), rows below 2^(end_bit - 32)
  int end_bit = 33;
  while (end_bit < 64 && (rows_all >> (end_bit - 32)) != 0ull) end_bit++;
  cudaSetDevice(h->device);
  size_t cub_bytes = 0;
  CK(cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)(3 * N), 0, end_bit,
                                    h->stream));
  // per row: rowS, rowI, perm, neg (4 each), two buffers of 3 sort keys (48), 3 predecessors (12), flag, level (4 each), lsig (8)
  const size_t need = (size_t)n_sessions * F * 8 + N * BPR_ROW_BYTES + cub_bytes + ((size_t)64 << 20);
  bpr_free_fit(h);
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    h->err = "g4r_bl_bpr_begin: the fit needs " + std::to_string(need) + " bytes of device memory (U alone " +
             std::to_string((size_t)n_sessions * F * 8) + "), " + std::to_string(free_b) + " are free";
    return G4R_ERR_CUDA;
  }
  cudaStream_t st = h->stream;
  h->ready = false;
  CK(bpr_take(h, &h->dU, (size_t)n_sessions * F));
  CK(bpr_take(h, &h->dRowS, N)); CK(bpr_take(h, &h->dRowI, N));
  CK(bpr_take(h, &h->dPerm, N)); CK(bpr_take(h, &h->dNeg, N));
  CK(bpr_take(h, &h->dKeys, 3 * N)); CK(bpr_take(h, &h->dKeys2, 3 * N)); CK(bpr_take(h, &h->dPred, 3 * N));
  CK(bpr_take(h, &h->dFlag, N)); CK(bpr_take(h, &h->dLevel, N)); CK(bpr_take(h, &h->dLsig, N + 1));
  CK(bpr_take(h, &h->dCtr, 4)); CK(bpr_take(h, &h->dCub, cub_bytes));
  h->bpr_cub_bytes = cub_bytes;
  CK(cudaMemcpyAsync(h->dU, U, (size_t)n_sessions * F * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dI, I, (size_t)NI * F * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dBI, bI, (size_t)NI * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dRowS, row_session, N * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dRowI, row_item, N * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(h->dFlag, 0, N * 4, st));
  CK(cudaStreamSynchronize(st));
  h->bpr_rows = (int64_t)N; h->bpr_sessions = n_sessions; h->bpr_tag = 0; h->bpr_end_bit = end_bit;
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_bpr_iterate(g4r_baselines* h, const int32_t* perm, const int32_t* negrow, double learning_rate, double lambda_session,
                                  double lambda_item, int32_t max_warps, double* mean_log_sigm, int64_t* max_level, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BPR) FAIL(G4R_ERR_STATE, "g4r_bl_bpr_iterate: the handle is not a BPR");
  if (!h->dU) FAIL(G4R_ERR_STATE, "g4r_bl_bpr_iterate: no fit begun (g4r_bl_bpr_begin)");
  if (!perm || !negrow || max_warps < 1) FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_iterate: null argument or max_warps < 1");
  if (!std::isfinite(learning_rate) || !std::isfinite(lambda_session) || !std::isfinite(lambda_item))
    FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_iterate: learning_rate and the lambdas must be finite");
  const int N = (int)h->bpr_rows, NI = h->n_items;
  const int neg_end = std::min(NI, N);                   // g4r_bl_bpr_begin requires n_items <= n_rows; rowI has n_rows entries
  {
    std::vector<char> seen(N, 0);
    for (int t = 0; t < N; t++) {
      if (perm[t] < 0 || perm[t] >= N || seen[perm[t]]) FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_iterate: perm must be a permutation of 0 .. n_rows - 1");
      seen[perm[t]] = 1;
      if (negrow[t] < 0 || negrow[t] >= neg_end) FAIL(G4R_ERR_INDEX, "g4r_bl_bpr_iterate: negrow must be in 0 .. min(n_items, n_rows) - 1");
    }
  }
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  if (++h->bpr_tag == 0) { CK(cudaMemsetAsync(h->dFlag, 0, (size_t)N * 4, st)); h->bpr_tag = 1; }
  CK(cudaMemcpyAsync(h->dPerm, perm, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dNeg, negrow, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  const unsigned S = (unsigned)h->bpr_sessions, rows_all = S + (unsigned)NI;
  CK(cudaEventRecord(h->ev0, st));
  k_bpr_keys<<<(N + 255) / 256, 256, 0, st>>>(h->dPerm, h->dNeg, h->dRowS, h->dRowI, N, S, rows_all, h->dKeys);
  size_t cb = h->bpr_cub_bytes;
  CK(cub::DeviceRadixSort::SortKeys(h->dCub, cb, h->dKeys, h->dKeys2, 3 * N, 0, h->bpr_end_bit, st));
  CK(cudaMemsetAsync(h->dPred, 0xff, (size_t)3 * N * 4, st));
  k_bpr_preds<<<(unsigned)((3ll * N + 255) / 256), 256, 0, st>>>(h->dKeys2, 3ll * N, h->dPerm, h->dRowI, S, rows_all, h->dPred);
  CK(cudaMemsetAsync(h->dCtr, 0, 4 * sizeof(int), st));
  BprFitDev d{};
  d.perm = h->dPerm; d.neg = h->dNeg; d.rowS = h->dRowS; d.rowI = h->dRowI; d.pred = h->dPred;
  d.U = h->dU; d.I = h->dI; d.bI = h->dBI;
  d.flag = h->dFlag; d.level = h->dLevel; d.lsig = h->dLsig;
  d.next = h->dCtr; d.max_level = h->dCtr + 1; d.fail = h->dCtr + 2;
  d.N = N; d.F = h->n_keep; d.tag = h->bpr_tag;
  d.lr = learning_rate; d.ls = lambda_session; d.li = lambda_item;
  using Fn = void (*)(BprFitDev, int);
  const int F = h->n_keep;
  const Fn fn = F <= 32 ? k_bpr_sgd<1> : F <= 64 ? k_bpr_sgd<2> : F <= 96 ? k_bpr_sgd<3> : F <= 128 ? k_bpr_sgd<4> : k_bpr_sgd<0>;
  const long long warps = std::min<long long>((long long)max_warps, (long long)BPR_WARPS_PER_SM * h->n_sm);
  fn<<<(unsigned)((warps + BPR_WARPS - 1) / BPR_WARPS), BPR_WARPS * 32, 0, st>>>(d, (int)warps);
  k_bpr_mean<<<1, 1024, 0, st>>>(h->dLsig, N, h->dLsig + N);
  CK(cudaGetLastError());
  CK(cudaEventRecord(h->ev1, st));
  int ctr[4] = {0, 0, 0, 0};
  double mean = 0.0;
  CK(cudaMemcpyAsync(ctr, h->dCtr, sizeof(ctr), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&mean, h->dLsig + N, sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (ctr[2]) {
    h->ready = false;
    FAIL(G4R_ERR_CUDA, "g4r_bl_bpr_iterate: a predecessor wait of k_bpr_sgd exceeded its bound; the model is undefined");
  }
  if (mean_log_sigm) *mean_log_sigm = mean;
  if (max_level) *max_level = ctr[1];
  if (device_ms) CK(cudaEventElapsedTime(device_ms, h->ev0, h->ev1));
  return G4R_OK;
}

extern "C" int g4r_bl_bpr_export(g4r_baselines* h, double* U, double* I) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BPR || !h->ready || (U && !h->dU)) FAIL(G4R_ERR_STATE, "g4r_bl_bpr_export: no fitted BPR (U exists only after g4r_bl_bpr_begin)");
  cudaSetDevice(h->device);
  if (U) CK(cudaMemcpyAsync(U, h->dU, (size_t)h->bpr_sessions * h->n_keep * 8, cudaMemcpyDeviceToHost, h->stream));
  if (I) CK(cudaMemcpyAsync(I, h->dI, (size_t)h->n_items * h->n_keep * 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

extern "C" int g4r_bl_bpr_import(g4r_baselines* h, const double* I, const double* bI) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BPR) FAIL(G4R_ERR_STATE, "g4r_bl_bpr_import: the handle is not a BPR");
  if (!I || !bI) FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_import: null argument");
  const int NI = h->n_items, F = h->n_keep;
  if (!bpr_finite(I, (size_t)NI * F) || !bpr_finite(bI, NI)) FAIL(G4R_ERR_INVALID, "g4r_bl_bpr_import: I and bI must be finite");
  cudaSetDevice(h->device);
  bpr_free_fit(h);
  CK(cudaMemcpyAsync(h->dI, I, (size_t)NI * F * 8, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->dBI, bI, (size_t)NI * 8, cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->ready = true;
  return G4R_OK;
}

// BPR's ranking of a g4r_bl_evaluate call: the counted events in blocks of bounded scratch.  qev (NARM): the counted events'
// vectors [n_ev x F] on the device, which replace the session means
static int bpr_blocks(g4r_baselines* h, BlCall& c, const float* qev) {
  const int NI = h->n_items, F = h->n_keep;
  const int64_t n_ev = c.n_ev, n_sessions = c.n_sessions;
  cudaStream_t st = h->stream;
  BprEvalDev d{};
  d.I = h->dI; d.bI = h->dBI; d.F = F; d.n_items = NI; d.mode = c.mode; d.exclude = c.exclude; d.k = c.k;
  d.items = c.d_items; d.off = c.d_off; d.nh = c.d_nh; d.ev0 = c.d_ev0;
  d.mult = c.d_mult; d.comp = c.d_cdist; d.n_comp = c.cdist.empty() ? NI : (int)c.cdist.size();
  unsigned char* first = nullptr;
  if (d.exclude) {
    CK(c.bb.take(&first, c.n_events));
    if (n_sessions > 0) k_bpr_first<<<(unsigned)((n_sessions + 7) / 8), 256, 0, st>>>(d.items, d.off, n_sessions, first);
    d.first = first;
  }
  d.counts = c.counts; d.out_items = c.out_items; d.out_scores = c.out_scores;
  CK(cudaMemsetAsync(d.counts, 0, (size_t)2 * n_ev * sizeof(int), st));
  const int k = c.k;
  int64_t blk = std::max<int64_t>(1, std::min<int64_t>(65536, (int64_t)(BPR_SCRATCH / ((size_t)8 * F))));
  if (k) blk = std::max<int64_t>(1, std::min<int64_t>(blk, (int64_t)(BPR_SCRATCH / ((size_t)8 * d.n_comp))));
  blk = std::min<int64_t>(blk, std::max<int64_t>(n_ev, 1));
  CK(c.bb.take(&d.uvec, (size_t)blk * F)); CK(c.bb.take(&d.pos, blk)); CK(c.bb.take(&d.st, blk)); CK(c.bb.take(&d.tsc, blk));
  if (k) CK(c.bb.take(&d.scores, (size_t)blk * d.n_comp));
  const std::vector<int64_t>& ev0 = c.ev0;
  const int n_tiles = (d.n_comp + BT_J - 1) / BT_J;
  for (int64_t E0 = 0; E0 < n_ev; E0 += blk) {
    const int nb = (int)std::min<int64_t>(blk, n_ev - E0);
    d.E0 = E0; d.nb = nb;
    // the sessions with counted events in [E0, E0 + nb)
    const int64_t s0 = std::upper_bound(ev0.begin(), ev0.begin() + n_sessions + 1, (int64_t)E0) - ev0.begin() - 1;
    const int64_t s1 = std::lower_bound(ev0.begin(), ev0.begin() + n_sessions + 1, (int64_t)(E0 + nb)) - ev0.begin();
    if (qev) k_narm_uvec<<<(unsigned)((s1 - s0 + 7) / 8), 256, 0, st>>>(d, qev, s0, s1);
    else k_bpr_uvec<<<(unsigned)((s1 - s0 + 7) / 8), 256, 0, st>>>(d, s0, s1);
    k_bpr_target<<<(nb + 255) / 256, 256, 0, st>>>(d);
    const unsigned gx = (unsigned)((nb + BT_E - 1) / BT_E);
    const int chunks = std::max(1, std::min(n_tiles, (int)((4 * h->n_sm + gx - 1) / gx)));
    const int per = (n_tiles + chunks - 1) / chunks;
    const dim3 grid(gx, (unsigned)((n_tiles + per - 1) / per));
    if (k) k_bpr_tile<true><<<grid, 256, 0, st>>>(d, per);
    else k_bpr_tile<false><<<grid, 256, 0, st>>>(d, per);
    if (d.exclude) {
      if (k) k_bpr_seen<true><<<(nb + 7) / 8, 256, 0, st>>>(d);
      else k_bpr_seen<false><<<(nb + 7) / 8, 256, 0, st>>>(d);
    }
    if (k) k_bpr_select<<<nb, KF_THREADS, 0, st>>>(d);
    CK(cudaGetLastError());
  }
  return G4R_OK;
}

static int bpr_rank(g4r_baselines* h, BlCall& c) { return bpr_blocks(h, c, nullptr); }
