// g4r_sknn.cuh -- session-based kNN (S-KNN with cosine similarity, V-SKNN-style position weights, DESIGN §3o; STAN-style time
// and position decays, §3p; VSTAN-style vector similarity, match-position neighbour weights and IDF, §3r) on the device: the
// index of the training sessions and the event-parallel ranking of evaluate_gpu / evaluate_events, one CTA per counted event.
// Included at the end of g4r_lib.cu after g4r_baselines.cuh (the handle, BlEvalDev, bl_w, bl_noise, bl_zero_eq, bl_emit,
// cta_bitonic, k_bl_sums, BlBufs).
#pragma once

constexpr int SK_THREADS = 256;
constexpr int SK_SAMPLE_MAX = 8192;                     // sample_size bound: the sample, its sims and the merge buffer in shared memory
constexpr int SK_CHUNK = 4 * SK_THREADS;                // posting-list entries merged into the sample per step
constexpr size_t SK_SCRATCH = (size_t)1 << 30;          // global scratch of one evaluation call (per-CTA slices)

struct SknnEvalDev {
  BlEvalDev bl;                                         // events, modes, candidates, exclude_seen, counts and lists
  long long n_ev; int64_t n_sess;
  const int64_t* s_off; const int* s_item;              // training sessions by recency rank: distinct items ascending
  const int64_t* i_off; const int* i_sess;              // every item's sessions, as ranks ascending (recency order)
  int sample, sim, nbr;                                 // sample_size, 0 cosine / 1 vector, k (neighbours)
  // STAN (§3p): per entry of s_item the 1-based position of the item's last occurrence in its session; the decay tables W1
  // (prefix distance), W2 (per session, by rank) and W3 (distance inside a neighbour)
  const int* s_pos; const double* w1; const double* w2; const double* w3;
  // per-CTA slices of global scratch: the prefix (c_cap entries) and the neighbours' (item, neighbour) pairs (z_cap entries)
  unsigned long long* c_key; int* c_flag; int* c_item; double* c_w; int c_cap;
  unsigned long long* z_key; int* u_item; double* u_sc; double* l_sc; int* l_item; int z_cap;
  // VSTAN (§3r): F per item (IDF) and W4 (prefix distance of the neighbour's most recent shared item)
  const double* f; const double* w4;
};

// the instances of k_sknn_rank
constexpr int SK_SKNN = 0, SK_STAN = 1, SK_VSTAN = 2;

// in-place bitonic sort of P (a power of two) 64-bit keys, ascending, in memory the whole CTA reads
__device__ void sk_bitonic_u64(unsigned long long* a, int P) {
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < P; t += blockDim.x) {
        const int u = t ^ stride;
        if (u <= t) continue;
        const unsigned long long x = a[t], y = a[u];
        if ((y < x) == ((t & size) == 0)) { a[t] = y; a[u] = x; }
      }
    }
  __syncthreads();
}

__device__ __forceinline__ int sk_pow2(int n) { int P = 1; while (P < n) P <<= 1; return P; }

// CTA-wide, every thread calls it: the position of a flagged thread among this round's flagged threads in thread order; *total
// their number
__device__ __forceinline__ int sk_rank_flag(bool f, int* sW, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, f);
  __syncthreads();
  if (lane == 0) sW[warp] = __popc(m);
  __syncthreads();
  int before = 0, tot = 0;
  for (int w = 0; w < SK_THREADS / 32; w++) { const int c = sW[w]; before += w < warp ? c : 0; tot += c; }
  total = tot;
  return before + __popc(m & ((1u << lane) - 1u));
}

__device__ __forceinline__ long long sk_sum(long long v, long long* sRed) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5] = v;
  __syncthreads();
  long long t = 0;
  for (int w = 0; w < SK_THREADS / 32; w++) t += sRed[w];
  return t;
}

// j among the prefix's items: a search of its (item, position) keys sorted ascending
__device__ __forceinline__ bool sk_seen(const unsigned long long* key, int n, int j) {
  const unsigned long long v = (unsigned long long)(unsigned)j << 32;
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (key[m] < v) lo = m + 1; else hi = m; }
  return lo < n && (int)(key[lo] >> 32) == j;
}
// score of item j: its entry among the U scored items (ascending), else 0
__device__ __forceinline__ double sk_score(const int* ui, const double* us, int U, int j) {
  const int p = sorted_lb(ui, U, j);
  return (p < U && ui[p] == j) ? us[p] : 0.0;
}
// j among the U scored items (ascending)
__device__ __forceinline__ bool sk_scored(const int* ui, int U, int j) {
  const int p = sorted_lb(ui, U, j);
  return p < U && ui[p] == j;
}

// One CTA per counted event (grid-stride over the events):
//  1. the prefix c = items[start .. p]: its (item, position) keys sorted, the last occurrence of every item flagged, and the
//     distinct items compacted in order of that position with their weights pos / t;
//  2. the sample: the first `sample` ranks of the union of those items' posting lists, merged list by list into a sorted set in
//     shared memory (a list contributes at most `sample` entries, and none past the set's largest once it is full);
//  3. each candidate's similarity (thread per candidate; c's items in position order searched in the session's sorted items);
//  4. the candidates sorted by (sim desc, rank asc); the first nbr are the neighbours;
//  5. (item, neighbour) pairs of the neighbours' items sorted, each item's sims summed in neighbour order;
//  6. (#greater, #equal) of the target, and with k > 0 its top-k list.
// STAN (§3p) changes three steps: the weights of step 1 are W1[t - p], step 3 is the W1 sum over sqrt(|I(c)| |I(n)|) times W2[n],
// and step 5 first finds each neighbour's most recent shared item r(n) and multiplies each summand by W3[|q_n(j) - q_n(r(n))|].
// Its scored items may score exactly 0 (underflow): they are counted as scored items and listed with the zero-score items.
// VSTAN (§3r) is STAN plus: step 1 keeps each compacted item's prefix distance t - p in c_flag (free once read), step 3 leaves the
// norm out for 'vector' (d.sim), the r(n) pre-pass turns sim2(n) into g(n) = sim2(n) W4[t - p_r(n)] in place in sS after the sort,
// and step 5 multiplies each item's neighbour-order sum once by F[j].
template <int V>
__global__ void __launch_bounds__(SK_THREADS) k_sknn_rank(SknnEvalDev d) {
  constexpr bool STAN = V != SK_SKNN, VSTAN = V == SK_VSTAN;
  extern __shared__ __align__(16) unsigned char sk_smem[];
  __shared__ int sW[SK_THREADS / 32];
  __shared__ long long sRed[SK_THREADS / 32];
  __shared__ int sZ;
  const BlEvalDev& b = d.bl;
  const int S = d.sample, PS = sk_pow2(S), tid = threadIdx.x, lane = tid & 31;
  double* sS = (double*)sk_smem;                        // [PS] sims
  int* bufA = (int*)(sS + PS);                          // [PS] sample (ranks)
  int* bufB = bufA + PS;                                // [PS] merge output
  int* sX = bufB + PS;                                  // [SK_CHUNK] new entries of a list chunk
  unsigned long long* ck = d.c_key + (size_t)blockIdx.x * d.c_cap;
  int* cf = d.c_flag + (size_t)blockIdx.x * d.c_cap;
  int* ci = d.c_item + (size_t)blockIdx.x * d.c_cap;
  double* cw = d.c_w + (size_t)blockIdx.x * d.c_cap;
  unsigned long long* zk = d.z_key + (size_t)blockIdx.x * d.z_cap;
  int* ui = d.u_item + (size_t)blockIdx.x * d.z_cap;
  double* us = d.u_sc + (size_t)blockIdx.x * d.z_cap;
  for (long long e = blockIdx.x; e < d.n_ev; e += gridDim.x) {
    int64_t lo = 0, hi = d.n_sess;                      // the session: last s with ev0[s] <= e
    while (lo < hi) { const int64_t m = (lo + hi + 1) >> 1; if (b.ev0[m] <= e) lo = m; else hi = m - 1; }
    const int64_t s = lo, st = b.off[s];
    const int64_t p = st + max(b.nh ? b.nh[s] : 0, 1) - 1 + (e - b.ev0[s]);
    const int t = (int)(p - st + 1), Pc = sk_pow2(t), y = b.items[p + 1];
    // 1. the prefix
    for (int q = tid; q < Pc; q += SK_THREADS)
      ck[q] = q < t ? ((unsigned long long)(unsigned)b.items[st + q] << 32 | (unsigned)q) : ~0ull;
    sk_bitonic_u64(ck, Pc);
    for (int q = tid; q < t; q += SK_THREADS) cf[(int)(ck[q] & 0xffffffffu)] = (q + 1 == t || (ck[q + 1] >> 32) != (ck[q] >> 32)) ? 1 : 0;
    __syncthreads();
    int D = 0;
    for (int q0 = 0; q0 < t; q0 += SK_THREADS) {
      const int q = q0 + tid;
      const bool f = q < t && cf[q];
      int tot;
      const int r = sk_rank_flag(f, sW, tot);
      if (f) {
        ci[D + r] = b.items[st + q]; cw[D + r] = STAN ? d.w1[t - 1 - q] : __ddiv_rn((double)(q + 1), (double)t);
        if (VSTAN) cf[D + r] = t - 1 - q;                // D + r <= q: this round's flags are read before sk_rank_flag's barrier
      }
      D += tot;
    }
    __syncthreads();
    // 2. the sample
    int* cand = bufA;
    int* nxt = bufB;
    int nB = 0;
    for (int m = 0; m < D; m++) {
      const int i = ci[m];
      const int64_t l0 = d.i_off[i];
      const int64_t n_i = d.i_off[i + 1] - l0;
      const int len = n_i < S ? (int)n_i : S;
      for (int a = 0; a < len; a += SK_CHUNK) {
        if (nB == S && d.i_sess[l0 + a] > cand[nB - 1]) break;
        int nX = 0;
        for (int r0 = 0; r0 < SK_CHUNK; r0 += SK_THREADS) {
          const int q = a + r0 + tid;
          const int v = q < len ? d.i_sess[l0 + q] : 0;
          bool keep = q < len && (nB < S || v < cand[nB - 1]);
          if (keep) { const int x = sorted_lb(cand, nB, v); keep = !(x < nB && cand[x] == v); }
          int tot;
          const int r = sk_rank_flag(keep, sW, tot);
          if (keep) sX[nX + r] = v;
          nX += tot;
        }
        __syncthreads();
        if (nX == 0) continue;
        for (int q = tid; q < nB; q += SK_THREADS) { const int pos = q + sorted_lb(sX, nX, cand[q]); if (pos < S) nxt[pos] = cand[q]; }
        for (int q = tid; q < nX; q += SK_THREADS) { const int pos = q + sorted_lb(cand, nB, sX[q]); if (pos < S) nxt[pos] = sX[q]; }
        __syncthreads();
        nB = min(S, nB + nX);
        int* sw = cand; cand = nxt; nxt = sw;
      }
    }
    // 3. similarities
    const int Pn = sk_pow2(max(nB, 1));
    for (int q = tid; q < Pn; q += SK_THREADS) {
      if (q >= nB) { sS[q] = -1.0; cand[q] = 0x7fffffff; continue; }
      const int r = cand[q];
      const int64_t a0 = d.s_off[r];
      const int ns = (int)(d.s_off[r + 1] - a0);
      const int* it = d.s_item + a0;
      double v = 0.0;
      int cnt = 0;
      for (int m = 0; m < D; m++) {
        const int j = ci[m];
        const int x = sorted_lb(it, ns, j);
        if (x < ns && it[x] == j) { cnt++; if (STAN || d.sim) v = __dadd_rn(v, cw[m]); }
      }
      if (STAN) v = __dmul_rn((VSTAN && d.sim) ? v : __ddiv_rn(v, __dsqrt_rn((double)((long long)D * ns))), d.w2[r]);
      else if (!d.sim) v = __ddiv_rn((double)cnt, __dsqrt_rn((double)((long long)D * ns)));
      sS[q] = v;
    }
    // 4. neighbours
    cta_bitonic<false>(sS, cand, Pn);
    const int nK = min(d.nbr, nB);
    // 5. scores (STAN: nxt, free since the merge, holds q_n(r(n)) of neighbour n; c's items are searched from the last position;
    //    VSTAN: sS[n] becomes g(n))
    if (STAN) {
      for (int r = tid; r < nK; r += SK_THREADS) {
        const int64_t a0 = d.s_off[cand[r]];
        const int ns = (int)(d.s_off[cand[r] + 1] - a0);
        const int* it = d.s_item + a0;
        int qr = 0, dr = 0;
        for (int m = D - 1; m >= 0; m--) {
          const int x = sorted_lb(it, ns, ci[m]);
          if (x < ns && it[x] == ci[m]) { qr = d.s_pos[a0 + x]; if (VSTAN) dr = cf[m]; break; }
        }
        nxt[r] = qr;
        if (VSTAN) sS[r] = __dmul_rn(sS[r], d.w4[dr]);
      }
    }
    if (tid == 0) sZ = 0;
    __syncthreads();
    for (int r = tid >> 5; r < nK; r += SK_THREADS / 32) {
      const int64_t a0 = d.s_off[cand[r]];
      const int ns = (int)(d.s_off[cand[r] + 1] - a0);
      int base = 0;
      if (lane == 0) base = atomicAdd(&sZ, ns);
      base = __shfl_sync(0xffffffffu, base, 0);
      for (int q = lane; q < ns; q += 32) zk[base + q] = (unsigned long long)(unsigned)d.s_item[a0 + q] << 32 | (unsigned)r;
    }
    __syncthreads();
    const int Z = sZ, Pz = sk_pow2(max(Z, 1));
    for (int q = Z + tid; q < Pz; q += SK_THREADS) zk[q] = ~0ull;
    sk_bitonic_u64(zk, Pz);
    int U = 0;
    for (int z0 = 0; z0 < Z; z0 += SK_THREADS) {
      const int z = z0 + tid;
      const bool head = z < Z && (z == 0 || (zk[z] >> 32) != (zk[z - 1] >> 32));
      int tot;
      const int r = sk_rank_flag(head, sW, tot);
      if (head) {
        const unsigned j = (unsigned)(zk[z] >> 32);
        double acc = 0.0;
        for (int w = z; w < Z && (unsigned)(zk[w] >> 32) == j; w++) {
          const int n = (int)(zk[w] & 0xffffffffu);
          if (STAN) {
            const int64_t a0 = d.s_off[cand[n]];
            const int x = sorted_lb(d.s_item + a0, (int)(d.s_off[cand[n] + 1] - a0), (int)j);
            acc = __dadd_rn(acc, __dmul_rn(sS[n], d.w3[abs(d.s_pos[a0 + x] - nxt[n])]));
          } else acc = __dadd_rn(acc, sS[n]);
        }
        ui[U + r] = (int)j; us[U + r] = VSTAN ? __dmul_rn(acc, d.f[j]) : acc;
      }
      U += tot;
    }
    __syncthreads();
    // 6. the target's counts
    const bool miss = b.exclude && sk_seen(ck, t, y);
    const double ty = sk_score(ui, us, U, y);
    long long gt = 0, eq = 0, sx = 0;
    if (b.mode == 3) {
      const double tn = __dadd_rn(ty, bl_noise(e, y));
      const int n_comp = b.mult ? b.n_cdist : b.n_items;
      for (int q = tid; q < n_comp; q += SK_THREADS) {
        const int j = b.mult ? b.cdist[q] : q;
        if (b.exclude && sk_seen(ck, t, j)) continue;
        const double sn = __dadd_rn(sk_score(ui, us, U, j), bl_noise(e, j));
        const long long w = bl_w(b, j);
        gt += sn > tn ? w : 0; eq += sn == tn ? w : 0;
      }
    } else {
      for (int q = tid; q < U; q += SK_THREADS) {
        const int j = ui[q];
        const double sc = us[q];
        const long long w = bl_w(b, j);
        sx += w;                                         // scored items are compared here, zeros included
        if (b.exclude && sk_seen(ck, t, j)) continue;
        gt += sc > ty ? w : 0; eq += sc == ty ? w : 0;
      }
      if (b.exclude)
        for (int m = tid; m < D; m += SK_THREADS)
          if (STAN ? !sk_scored(ui, U, ci[m]) : sk_score(ui, us, U, ci[m]) == 0.0) sx += bl_w(b, ci[m]);
    }
    gt = sk_sum(gt, sRed); eq = sk_sum(eq, sRed); sx = sk_sum(sx, sRed);
    if (tid == 0) {
      if (b.mode != 3) eq += bl_zero_eq(b, ty, sx);
      b.counts[2 * e] = miss ? -1 : (int)gt;
      b.counts[2 * e + 1] = miss ? -1 : (int)eq;
    }
    if (b.k) {
      double* ls = d.l_sc + (size_t)blockIdx.x * d.z_cap;
      int* li = d.l_item + (size_t)blockIdx.x * d.z_cap;
      const int Pu = sk_pow2(max(U, 1));
      for (int q = tid; q < Pu; q += SK_THREADS) { ls[q] = q < U ? us[q] : -1.0; li[q] = q < U ? ui[q] : 0x7fffffff; }
      cta_bitonic<false>(ls, li, Pu);
      if (tid < 32) {
        int* o_i = b.out_items + (size_t)e * b.k;
        double* o_s = b.out_scores + (size_t)e * b.k;
        int base = 0;
        for (int q0 = 0; q0 < U && base < b.k; q0 += 32) {        // the positive scored items by (score desc, index asc)
          const int q = q0 + lane;
          const int j = q < U ? li[q] : 0;
          const bool ok = q < U && (!STAN || ls[q] > 0.0) && (!b.mult || b.mult[j] > 0) && !(b.exclude && sk_seen(ck, t, j));
          bl_emit(ok, j, q < U ? ls[q] : 0.0, o_i, o_s, b.k, base);
        }
        const int n_comp = b.mult ? b.n_cdist : b.n_items;          // then the zero-score items, by index
        for (int q0 = 0; q0 < n_comp && base < b.k; q0 += 32) {
          const int q = q0 + lane;
          const int j = q < n_comp ? (b.mult ? b.cdist[q] : q) : 0;
          const bool ok = q < n_comp && (!b.mult || b.mult[j] > 0) && !(b.exclude && sk_seen(ck, t, j)) && sk_score(ui, us, U, j) == 0.0;
          bl_emit(ok, j, 0.0, o_i, o_s, b.k, base);
        }
        for (int q = base + lane; q < b.k; q += 32) { o_i[q] = -1; o_s[q] = __longlong_as_double(0x7ff8000000000000ll); }
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// C ABI (include/g4r.h)
// ---------------------------------------------------------------------------------------------------------------------------
// the index of a SessionKNN (similarity; positions, w2 and w3 null) or a STAN / VSTAN handle: every argument checked on the host before
// any device write, the sessions renumbered by rank and every item's sessions built by a counting sort that visits the ranks in order
static int sk_index(g4r_baselines* h, const std::string& fn, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items,
                    int64_t n_entries, const int32_t* recency, int32_t sample_size, int32_t similarity, const int32_t* positions,
                    const double* w2, const double* w3, int64_t n_w3) {
  const bool stan = h->kind == BL_STAN || h->kind == BL_VSTAN;
  if (!session_offsets || !recency || n_sessions < 1 || n_sessions >= INT32_MAX || n_entries < 0 || (n_entries > 0 && !items))
    FAIL(G4R_ERR_INVALID, fn + ": null argument, or n_sessions outside 1 .. 2^31 - 2");
  if (stan && (!w2 || !w3 || n_w3 < 1 || n_w3 > (1 << 30) || (n_entries > 0 && !positions)))
    FAIL(G4R_ERR_INVALID, fn + ": null positions, w2 or w3, or n_w3 outside 1 .. 2^30");
  if (sample_size < 1 || sample_size > SK_SAMPLE_MAX) FAIL(G4R_ERR_INVALID, fn + ": sample_size must be in 1 .. 8192");
  if (h->n_keep > sample_size) FAIL(G4R_ERR_INVALID, fn + ": k (n_keep) must not exceed sample_size");
  if (!stan && similarity != 0 && similarity != 1) FAIL(G4R_ERR_INVALID, fn + ": similarity must be 0 (cosine) or 1 (vector)");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_entries)) FAIL(G4R_ERR_INVALID, fn + ": session offsets must rise from 0 to n_entries");
  const int NI = h->n_items;
  for (int64_t s = 0; s < n_sessions; s++)
    for (int64_t q = session_offsets[s]; q < session_offsets[s + 1]; q++) {
      if (items[q] < 0 || items[q] >= NI) FAIL(G4R_ERR_INDEX, fn + ": item index out of range");
      if (q > session_offsets[s] && items[q] <= items[q - 1]) FAIL(G4R_ERR_INVALID, fn + ": a session's items must be distinct and ascending");
    }
  if (stan) {
    // a session of L events has its distinct items' last positions distinct in 1 .. L, and L <= n_w3 (W3 covers 0 .. L - 1)
    std::vector<int64_t> mark(n_w3 + 1, -1);
    for (int64_t s = 0; s < n_sessions; s++)
      for (int64_t q = session_offsets[s]; q < session_offsets[s + 1]; q++) {
        if (positions[q] < 1 || positions[q] > n_w3) FAIL(G4R_ERR_INVALID, fn + ": positions must be in 1 .. n_w3 (the longest session's length)");
        if (mark[positions[q]] == s) FAIL(G4R_ERR_INVALID, fn + ": two items of a session at one position");
        mark[positions[q]] = s;
      }
    for (int64_t s = 0; s < n_sessions; s++)
      if (!(w2[s] >= 0.0 && w2[s] <= 1.0)) FAIL(G4R_ERR_INVALID, fn + ": w2 entries must be in [0, 1]");
    for (int64_t q = 0; q < n_w3; q++)
      if (!(w3[q] >= 0.0 && w3[q] <= 1.0)) FAIL(G4R_ERR_INVALID, fn + ": w3 entries must be in [0, 1]");
  }
  const int64_t S = n_sessions;
  std::vector<int64_t> by_rank(S, -1);
  for (int64_t s = 0; s < S; s++) {
    if (recency[s] < 0 || recency[s] >= S) FAIL(G4R_ERR_INDEX, fn + ": recency rank out of range");
    if (by_rank[recency[s]] >= 0) FAIL(G4R_ERR_INVALID, fn + ": the recency ranks must be a permutation of 0 .. n_sessions - 1");
    by_rank[recency[s]] = s;
  }
  // the sessions renumbered by rank, and every item's sessions: a counting sort that visits the ranks in order
  std::vector<int64_t> off(S + 1, 0), ioff(NI + 1, 0);
  std::vector<int> sit(n_entries), isess(n_entries), spos(stan ? n_entries : 0);
  std::vector<double> rw2(stan ? S : 0);
  std::vector<int64_t> lens(S);
  for (int64_t r = 0; r < S; r++) {
    const int64_t s = by_rank[r], a = session_offsets[s], n = session_offsets[s + 1] - a;
    std::copy(items + a, items + a + n, sit.begin() + off[r]);
    if (stan) { std::copy(positions + a, positions + a + n, spos.begin() + off[r]); rw2[r] = w2[s]; }
    off[r + 1] = off[r] + n;
    lens[r] = n;
    for (int64_t q = a; q < a + n; q++) ioff[items[q] + 1]++;
  }
  for (int i = 0; i < NI; i++) ioff[i + 1] += ioff[i];
  {
    std::vector<int64_t> fill(ioff.begin(), ioff.end() - 1);
    for (int64_t r = 0; r < S; r++)
      for (int64_t q = off[r]; q < off[r + 1]; q++) isess[fill[sit[q]]++] = (int)r;
  }
  const int K = std::min<int64_t>(h->n_keep, S);
  std::nth_element(lens.begin(), lens.begin() + (K - 1), lens.end(), std::greater<int64_t>());
  int64_t zmax = 0;
  for (int q = 0; q < K; q++) zmax += lens[q];
  cudaSetDevice(h->device);
  h->ready = false;
  for (void* p : h->sknn_mem) cudaFree(p);
  h->sknn_mem.clear();
  h->dSkOff = h->dSkIoff = nullptr; h->dSkItem = h->dSkIsess = h->dStPos = nullptr; h->dStW2 = h->dStW3 = nullptr;
  if (h->kind == BL_VSTAN) {                            // a fit clears g4r_bl_vstan_set's settings
    for (void* p : {(void*)h->dVsF, (void*)h->dVsW4}) if (p) cudaFree(p);
    h->dVsF = h->dVsW4 = nullptr; h->vs_n_w4 = 0; h->vs_set = false;
  }
  auto take = [&](auto** p, size_t n) { cudaError_t e = bl_alloc(p, n); if (e == cudaSuccess) h->sknn_mem.push_back(*p); else *p = nullptr; return e; };
  CK(take(&h->dSkOff, S + 1)); CK(take(&h->dSkIoff, NI + 1));
  CK(take(&h->dSkItem, n_entries)); CK(take(&h->dSkIsess, n_entries));
  if (stan) { CK(take(&h->dStPos, n_entries)); CK(take(&h->dStW2, S)); CK(take(&h->dStW3, n_w3)); }
  cudaStream_t st = h->stream;
  CK(cudaMemcpyAsync(h->dSkOff, off.data(), (S + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dSkIoff, ioff.data(), (NI + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  if (n_entries) {
    CK(cudaMemcpyAsync(h->dSkItem, sit.data(), n_entries * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->dSkIsess, isess.data(), n_entries * sizeof(int), cudaMemcpyHostToDevice, st));
    if (stan) CK(cudaMemcpyAsync(h->dStPos, spos.data(), n_entries * sizeof(int), cudaMemcpyHostToDevice, st));
  }
  if (stan) {
    CK(cudaMemcpyAsync(h->dStW2, rw2.data(), S * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->dStW3, w3, n_w3 * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  CK(cudaStreamSynchronize(st));
  h->sk_sessions = S; h->sk_zmax = zmax; h->sk_sample = sample_size; h->sk_sim = stan ? 0 : similarity;
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_sknn_fit(g4r_baselines* h, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_entries,
                               const int32_t* recency, int32_t sample_size, int32_t similarity) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SKNN) FAIL(G4R_ERR_STATE, "g4r_bl_sknn_fit: the handle is not a SessionKNN");
  return sk_index(h, "g4r_bl_sknn_fit", session_offsets, n_sessions, items, n_entries, recency, sample_size, similarity, nullptr, nullptr,
                  nullptr, 0);
}

extern "C" int g4r_bl_stan_fit(g4r_baselines* h, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_entries,
                               const int32_t* positions, const int32_t* recency, const double* w2, const double* w3, int64_t n_w3,
                               int32_t sample_size) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_STAN && h->kind != BL_VSTAN) FAIL(G4R_ERR_STATE, "g4r_bl_stan_fit: the handle is not a STAN or VSTAN");
  return sk_index(h, "g4r_bl_stan_fit", session_offsets, n_sessions, items, n_entries, recency, sample_size, 0, positions, w2, w3, n_w3);
}

extern "C" int g4r_bl_stan_set_w1(g4r_baselines* h, const double* w1, int64_t n_w1) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_STAN && h->kind != BL_VSTAN) FAIL(G4R_ERR_STATE, "g4r_bl_stan_set_w1: the handle is not a STAN or VSTAN");
  if (!w1 || n_w1 < 1 || n_w1 > (1 << 30)) FAIL(G4R_ERR_INVALID, "g4r_bl_stan_set_w1: null w1, or n_w1 outside 1 .. 2^30");
  for (int64_t q = 0; q < n_w1; q++)
    if (!(w1[q] >= 0.0 && w1[q] <= 1.0)) FAIL(G4R_ERR_INVALID, "g4r_bl_stan_set_w1: w1 entries must be in [0, 1]");
  cudaSetDevice(h->device);
  if (h->dStW1) cudaFree(h->dStW1);
  h->dStW1 = nullptr; h->st_n_w1 = 0;
  CK(bl_alloc(&h->dStW1, n_w1));
  CK(cudaMemcpyAsync(h->dStW1, w1, n_w1 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->st_n_w1 = n_w1;
  return G4R_OK;
}

extern "C" int g4r_bl_vstan_set(g4r_baselines* h, int32_t similarity, const double* f, int64_t n_f, const double* w4, int64_t n_w4) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_VSTAN) FAIL(G4R_ERR_STATE, "g4r_bl_vstan_set: the handle is not a VSTAN");
  if (similarity != 0 && similarity != 1) FAIL(G4R_ERR_INVALID, "g4r_bl_vstan_set: similarity must be 0 (cosine) or 1 (vector)");
  if (!f || n_f != h->n_items) FAIL(G4R_ERR_INVALID, "g4r_bl_vstan_set: null f, or n_f is not n_items");
  for (int64_t q = 0; q < n_f; q++)
    if (!(std::isfinite(f[q]) && f[q] >= 0.0)) FAIL(G4R_ERR_INVALID, "g4r_bl_vstan_set: f entries must be finite and >= 0");
  if (!w4 || n_w4 < 1 || n_w4 > (1 << 30)) FAIL(G4R_ERR_INVALID, "g4r_bl_vstan_set: null w4, or n_w4 outside 1 .. 2^30");
  for (int64_t q = 0; q < n_w4; q++)
    if (!(w4[q] >= 0.0 && w4[q] <= 1.0)) FAIL(G4R_ERR_INVALID, "g4r_bl_vstan_set: w4 entries must be in [0, 1]");
  cudaSetDevice(h->device);
  for (void* p : {(void*)h->dVsF, (void*)h->dVsW4}) if (p) cudaFree(p);
  h->dVsF = h->dVsW4 = nullptr; h->vs_n_w4 = 0; h->vs_set = false;
  CK(bl_alloc(&h->dVsF, n_f));
  CK(bl_alloc(&h->dVsW4, n_w4));
  CK(cudaMemcpyAsync(h->dVsF, f, n_f * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->dVsW4, w4, n_w4 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->sk_sim = similarity; h->vs_n_w4 = n_w4; h->vs_set = true;
  return G4R_OK;
}

// the ranking of a g4r_bl_evaluate call of a SessionKNN, a STAN or a VSTAN: resident CTAs over the counted events, each with its own
// slices of a global scratch of at most SK_SCRATCH bytes (fewer CTAs when the slices are large; one at least)
static int sknn_rank(g4r_baselines* h, BlCall& c) {
  const int64_t n_ev = c.n_ev, n_sessions = c.n_sessions;
  const int64_t* session_offsets = c.off;
  const std::vector<int64_t>& ev0 = c.ev0;
  const int k = c.k;
  int64_t max_len = 1;
  for (int64_t s = 0; s < n_sessions; s++) max_len = std::max(max_len, session_offsets[s + 1] - session_offsets[s]);
  if (max_len > (1 << 30) || h->sk_zmax > (1 << 30)) FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: a session or the neighbours' items exceed 2^30 entries");
  const bool stan = h->kind == BL_STAN || h->kind == BL_VSTAN, vstan = h->kind == BL_VSTAN;
  if (stan)                                             // W1 (and W4) must cover the prefix distances 0 .. t - 1 of every counted event
    for (int64_t s = 0; s < n_sessions; s++) {
      const int64_t t_max = session_offsets[s + 1] - session_offsets[s] - 1;
      if (ev0[s + 1] > ev0[s] && t_max > h->st_n_w1)
        FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: a counted event's prefix is longer than the STAN W1 table (g4r_bl_stan_set_w1)");
      if (vstan && ev0[s + 1] > ev0[s] && t_max > h->vs_n_w4)
        FAIL(G4R_ERR_INVALID, "g4r_bl_evaluate: a counted event's prefix is longer than the VSTAN W4 table (g4r_bl_vstan_set)");
    }
  cudaStream_t st = h->stream;
  BlBufs& bb = c.bb;
  SknnEvalDev d{};
  d.bl = c.bl(h->n_items);
  d.n_ev = n_ev; d.n_sess = n_sessions;
  d.s_off = h->dSkOff; d.s_item = h->dSkItem; d.i_off = h->dSkIoff; d.i_sess = h->dSkIsess;
  d.sample = h->sk_sample; d.sim = h->sk_sim; d.nbr = h->n_keep;
  d.s_pos = h->dStPos; d.w1 = h->dStW1; d.w2 = h->dStW2; d.w3 = h->dStW3;
  d.f = h->dVsF; d.w4 = h->dVsW4;
  const auto kern = vstan ? k_sknn_rank<SK_VSTAN> : stan ? k_sknn_rank<SK_STAN> : k_sknn_rank<SK_SKNN>;
  int PS = 1;
  while (PS < d.sample) PS <<= 1;
  const size_t smem = (size_t)PS * (sizeof(double) + 2 * sizeof(int)) + SK_CHUNK * sizeof(int);
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, SK_THREADS, smem));
  int cc = 1, zc = 1;
  while (cc < max_len) cc <<= 1;
  while (zc < h->sk_zmax) zc <<= 1;
  d.c_cap = cc; d.z_cap = zc;
  const size_t per_cta = (size_t)cc * (8 + 4 + 4 + 8) + (size_t)zc * (8 + 4 + 8 + (k ? 8 + 4 : 0));
  const int64_t grid = std::max<int64_t>(1, std::min<int64_t>({std::max<int64_t>(n_ev, 1), (int64_t)std::max(occ, 1) * h->n_sm,
                                                                (int64_t)(SK_SCRATCH / per_cta)}));
  CK(bb.take(&d.c_key, (size_t)cc * grid)); CK(bb.take(&d.c_flag, (size_t)cc * grid));
  CK(bb.take(&d.c_item, (size_t)cc * grid)); CK(bb.take(&d.c_w, (size_t)cc * grid));
  CK(bb.take(&d.z_key, (size_t)zc * grid)); CK(bb.take(&d.u_item, (size_t)zc * grid)); CK(bb.take(&d.u_sc, (size_t)zc * grid));
  if (k) { CK(bb.take(&d.l_sc, (size_t)zc * grid)); CK(bb.take(&d.l_item, (size_t)zc * grid)); }
  if (n_ev > 0) {
    kern<<<(unsigned)grid, SK_THREADS, smem, st>>>(d);
    CK(cudaGetLastError());
  }
  return G4R_OK;
}
