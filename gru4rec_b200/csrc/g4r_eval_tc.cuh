// g4r_eval_tc.cuh -- full-catalogue scoring of evaluate_gpu on the Hopper tensor cores (wgmma, sm_90a).
//
// What is computed (reference: yhat = h Wy^T + By, gru4rec.py:502; ranks = (others > targets).sum + 1, evaluation.py:57-64):
// for every lane b of the evaluation batch the number of catalogue items whose score beats / ties the score of the lane's
// target.  The [items x lanes] score matrix (37,483 x 512 at the RSC15 shape: 3.8 GFLOP per mini-batch, the largest dense
// contraction of the whole path) is never written: each 128-lane x 256-item tile is accumulated in registers by
// wgmma.mma_async (kind tf32, m64n128k8 per warpgroup) and reduced to the two counters right there.
//
// fp32 fidelity on TF32 tensor cores: 3xTF32 -- every fp32 operand x is split as hi = tf32(x), lo = tf32(x - hi) and the
// product is accumulated as lo*hi + hi*lo + hi*hi (the dropped lo*lo term and the roundings are ~2^-21 relative), i.e. ~1e-6
// relative on the scores, far inside the 1e-4 bar on Recall / MRR.  The target's own column is excluded explicitly (it is
// the one comparison that must be exact), so a rank can only move where two DIFFERENT items' scores differ by < 1e-6 relative.
//
// Structure (one CTA per SM, 512 threads = four warpgroups, persistent over its item tiles):
//   pre-pass   k_tc_split writes the operands as hi / lo TF32 blocks in the K-major 128-byte-swizzle layout: the item table
//              when Wy / By have changed (kept between calls), the hidden states once per mini-batch; one extra K column carries the item bias (1.0 on the
//              hidden-state side), so the accumulator is the complete pre-activation score
//   loads      thread 0: two bulk copies (cp.async.bulk -> mbarrier complete_tx) per 32-wide K chunk fill a 96 KB stage
//              [A hi | A lo | B hi | B lo]; two stages, a stage is refilled once all four warpgroups have released it
//   MMA        each warpgroup: 12 wgmma per chunk on its 64 x 128 quarter of the tile
//   epilogue   two compares per item against the lane's pre-activation thresholds (k_eval_tgt computes them once per lane),
//              counters thread-local, summed over the four threads of a quad at the end of a lane block
// All waits are mbarrier try_wait loops with a time-out that traps (a wrong phase must not hang the device).
#pragma once

constexpr int TC_M = 128;            // evaluation lanes per tile (two warpgroups of 64 rows)
constexpr int TC_N = 256;            // items per tile (two warpgroups of 128 columns)
constexpr int TC_KC = 32;            // K chunk per pipeline stage (floats)
constexpr int TC_THREADS = 512;      // four consumer warpgroups: rows (wg & 1) * 64, columns (wg >> 1) * 128 of the tile
constexpr int TC_STAGES = 2;
constexpr uint32_t TC_A_BYTES = TC_M * TC_KC * 4;       // 16 KB per hi / lo array
constexpr uint32_t TC_B_BYTES = TC_N * TC_KC * 4;       // 32 KB
constexpr uint32_t TC_STAGE_BYTES = 2 * TC_A_BYTES + 2 * TC_B_BYTES;   // 96 KB
constexpr unsigned long long TC_TIMEOUT_NS = 2000000000ull;

struct TcSmem {
  alignas(1024) unsigned char stage[TC_STAGES][TC_STAGE_BYTES];   // [A hi | A lo | B hi | B lo]
  alignas(8) unsigned long long stage_full[TC_STAGES];    // operand blocks of the stage have landed (TMA complete_tx)
  unsigned long long stage_free[TC_STAGES];    // the four warpgroups' MMAs that read the stage have completed
  int err;
};

__device__ __forceinline__ uint32_t tc_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tc_mbar_init(unsigned long long* bar, unsigned int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(tc_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void tc_mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(tc_smem_u32(bar)) : "memory");
}
// a wait that does not complete within TC_TIMEOUT_NS is a protocol bug: trap (the launch fails with an error) rather than hang
__device__ __forceinline__ bool tc_mbar_wait(unsigned long long* bar, unsigned int parity, int* err) {
  const uint32_t a = tc_smem_u32(bar);
  unsigned long long t0 = 0; unsigned int spins = 0;
  while (true) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n" : "=r"(ok) : "r"(a), "r"(parity) : "memory");
    if (ok) return true;
    if ((++spins & 63u) == 0) {
      unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (t0 == 0) t0 = t;
      if (t - t0 > TC_TIMEOUT_NS) { *(volatile int*)err = 1; asm volatile("trap;"); }
    }
  }
}
__device__ __forceinline__ uint32_t tc_tf32(float x) { uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x)); return r; }
// K-major operand blocks in the 128-byte-swizzle layout: a row is 32 tf32 values = 128 bytes, eight rows form a 1024-byte atom in
// which the 16-byte piece c of row r sits at position c ^ (r % 8) (the tensor core reads a whole 128-byte row per access without
// bank conflicts).  wgmma shared-memory descriptor: SBO (next 8 rows) = 1024 B, LBO unused for swizzled K-major operands (1),
// layout type 1 = 128-byte swizzle; blocks are 1024-byte aligned, a K step of 8 values advances the start address by 32 bytes
// inside the atom, 64 rows further is +8 KB.
__device__ __forceinline__ uint64_t tc_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024u >> 4) << 32) | (1ull << 62);
}
// byte offset of the 16-byte piece (row r, k = 4 * kq .. 4 * kq + 3) inside a block of rows x 32 k-values
__device__ __forceinline__ uint32_t tc_block_off(int r, int kq) { return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((kq ^ (r & 7)) << 4)); }

// ---- warpgroup MMA (wgmma, sm_90a): D[64 x NW] += A[64 x 8] B[NW x 8]^T in TF32, both operands K-major in shared memory, D in
// registers.  Accumulator fragment of thread t of the warpgroup: d[i] = D[16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2)]
// [8 * (i / 4) + 2 * (t % 4) + i % 2] ----
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from touching the accumulator registers across the asynchronous MMAs
template <int NR>
__device__ __forceinline__ void wg_fence_acc(float (&d)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; i++) asm volatile("" : "+f"(d[i]) :: "memory");
}
#define WG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wg_mma_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
               "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
               "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24), WG_D8(32), WG_D8(40), WG_D8(48), WG_D8(56)
               : "l"(a_desc), "l"(b_desc) : "memory");
}
__device__ __forceinline__ void wg_mma_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
               "%24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
               : WG_D8(0), WG_D8(8), WG_D8(16), WG_D8(24)
               : "l"(a_desc), "l"(b_desc) : "memory");
}
#undef WG_D8
// one 32-wide K chunk of a 3xTF32 product for one warpgroup: lo*hi + hi*lo + hi*hi over four steps of 8, then wait for it (the
// operand blocks are zero beyond the live K, so a partial last chunk needs no special case)
template <int NR>
__device__ __forceinline__ void wg_chunk_3xtf32(float (&d)[NR], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
  wg_fence_acc(d);
  wg_fence();
#pragma unroll
  for (int j = 0; j < TC_KC / 8; j++) {
    const uint32_t o = (uint32_t)j * 32u;      // 8 values along K = 32 bytes inside the swizzle atom
    wg_mma_tf32(d, tc_desc(a_lo + o), tc_desc(b_hi + o));
    wg_mma_tf32(d, tc_desc(a_hi + o), tc_desc(b_lo + o));
    wg_mma_tf32(d, tc_desc(a_hi + o), tc_desc(b_hi + o));
  }
  wg_commit();
  wg_wait0();
  wg_fence_acc(d);
}

// Pre-split operand blocks in global memory (written for the item table whenever it has changed, once per mini-batch for the hidden
// states): block (rb, c) = rows [rb * RB, +RB) x k [32 c, +32) as [hi | lo], each in the K-major 128-byte-swizzle layout
// (tc_block_off).  The scoring kernel then feeds the tensor cores with plain bulk copies (TMA) -- no register staging on the
// critical path.
// The contraction runs over K + 1 values: column K holds `one` on the hidden-state side and the item bias on the table side
// (bias != nullptr), so the accumulator is the complete pre-activation score.  Table rows past the catalogue are all zero: no pad
// score can be kept out of the counts by its value (a flat activation gives a lower threshold of -inf), so the epilogue bounds the
// columns of the last item tile instead.
template <int RB>
__global__ void __launch_bounds__(256) k_tc_split(const float* __restrict__ src, int nrows, int ld, int K, unsigned char* __restrict__ dst, int n_chunk,
                                                  const float* __restrict__ bias, float one) {
  const int rb = blockIdx.x, c = blockIdx.y;
  unsigned char* hi = dst + ((size_t)rb * n_chunk + c) * 2 * (RB * TC_KC * 4);
  unsigned char* lo = hi + RB * TC_KC * 4;
  const int k0 = c * TC_KC;
  for (int i = threadIdx.x; i < RB * 8; i += blockDim.x) {
    const int r = i % RB, cc = i / RB;            // rows fastest: consecutive threads write consecutive 16-byte pieces
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    const int row = rb * RB + r;
    if (row < nrows && k0 + cc * 4 < K) v = ld4(src + (size_t)row * ld + k0 + cc * 4);
    if (K - (k0 + cc * 4) >= 0 && K - (k0 + cc * 4) < 4) {       // the extra column (K % 4 == 0 is not required)
      const float x = bias ? (row < nrows ? bias[row] : 0.f) : one;
      const int u = K - (k0 + cc * 4);
      if (u == 0) v = make_float4(x, 0.f, 0.f, 0.f); else if (u == 1) v.y = x, v.z = 0.f, v.w = 0.f; else if (u == 2) v.z = x, v.w = 0.f; else v.w = x;
    }
    const uint32_t off = tc_block_off(r, cc);
    uint4 h, l;
    h.x = tc_tf32(v.x); h.y = tc_tf32(v.y); h.z = tc_tf32(v.z); h.w = tc_tf32(v.w);
    l.x = tc_tf32(v.x - __uint_as_float(h.x)); l.y = tc_tf32(v.y - __uint_as_float(h.y));
    l.z = tc_tf32(v.z - __uint_as_float(h.z)); l.w = tc_tf32(v.w - __uint_as_float(h.w));
    *reinterpret_cast<uint4*>(hi + off) = h;
    *reinterpret_cast<uint4*>(lo + off) = l;
  }
}
__device__ __forceinline__ void tc_bulk_copy(void* sdst, const void* gsrc, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(tc_smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(tc_smem_u32(bar)) : "memory");
}

// Ranking compares act(x) with the target score t = act(x_t).  act is monotone non-decreasing, so for every lane there are two
// pre-activation thresholds with  act(x) > t  <=>  x > hi  and  act(x) == t  <=>  lo <= x <= hi : they are found once per lane by
// bisection over the ordered fp32 bit patterns with the very act_fwd the fp32 kernels use (64 evaluations per lane), and the
// per-item work drops to two compares.
__device__ __forceinline__ uint32_t tc_fkey(float f) { const uint32_t u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float tc_fkey_inv(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
// x_t = the target's own pre-activation (act(x_t) == t): both thresholds are normally within a few ulps of it, so the search
// gallops away from key(x_t) (1, 2, 4, ... keys) and bisects the last bracket -- a handful of evaluations outside the flat
// regions of the activation, at most ~64 inside them.
__device__ __forceinline__ void tc_thresholds(const ActSpec a, bool elem_act, float t, float x_t, float& lo, float& hi) {
  if (!elem_act) { lo = hi = t; return; }
  const uint32_t kmin = tc_fkey(-INFINITY), kmax = tc_fkey(INFINITY), k0 = min(max(tc_fkey(x_t), kmin), kmax);
  // upper: first key above k0 whose activation exceeds t (kmax + 1 if none); invariant act(l - 1) <= t
  uint32_t l = k0 + 1u, r = kmax + 1u;
  for (uint32_t d = 1u; l < r; d <<= 1) {
    const uint32_t m = (kmax - l < d) ? kmax : l + d - 1u;          // probe
    if (act_fwd(a, tc_fkey_inv(m)) > t) { r = m; break; }
    l = m + 1u;
    if (d >= 0x80000000u) break;
  }
  while (l < r) { const uint32_t m = l + ((r - l) >> 1); if (act_fwd(a, tc_fkey_inv(m)) > t) r = m; else l = m + 1u; }
  hi = tc_fkey_inv(l - 1u);
  // lower: smallest key whose activation still reaches t; invariant act(r2) >= t
  uint32_t r2 = k0, l2 = kmin;
  for (uint32_t d = 1u; l2 < r2; d <<= 1) {
    const uint32_t m = (r2 - kmin < d) ? kmin : r2 - d;
    if (act_fwd(a, tc_fkey_inv(m)) >= t) { r2 = m; if (d >= 0x80000000u) break; } else { l2 = m + 1u; break; }
  }
  while (l2 < r2) { const uint32_t m = l2 + ((r2 - l2) >> 1); if (act_fwd(a, tc_fkey_inv(m)) >= t) r2 = m; else l2 = m + 1u; }
  lo = tc_fkey_inv(r2);
}

// The wgmma sweep of the scoring kernels (k_eval_tc, k_topk_tc): one persistent CTA per SM loops over (lane block of 128) x (its
// item tiles of 256) x (32-wide K chunks).  Asplit: hidden-state blocks of 128 lanes, Bsplit: item-table blocks of 256 items
// (k_tc_split), K = L + 1 with the bias column.  Warpgroup wg accumulates rows (wg & 1) * 64 .. + 63 x columns (wg >> 1) * 128
// .. + 127 of the tile in registers, so a thread holds two lanes x 32 items.  Thread 0 also feeds the stages: it issues the bulk
// copies of a stage as soon as all four warpgroups have finished the MMAs that read it.
//   lane_block(b)      at the start of every lane block: b is the thread's first lane, b + 8 its second
//   tile(d, c0, last)  after every tile: d[i] holds lane b + 8 * ((i / 2) % 2) x item c0 + 8 * (i / 4) + i % 2 (columns past the
//                      catalogue included); last: the CTA's last tile of the lane block
template <class LaneBlock, class Tile>
__device__ __forceinline__ void tc_sweep(int M, int I, int K, const unsigned char* __restrict__ Asplit, const unsigned char* __restrict__ Bsplit,
                                         LaneBlock&& lane_block, Tile&& tile) {
  extern __shared__ __align__(1024) unsigned char tc_raw[];
  TcSmem& sm = *reinterpret_cast<TcSmem*>(tc_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int n_tiles = (I + TC_N - 1) / TC_N;         // item tiles
  const int n_lb = (M + TC_M - 1) / TC_M;            // lane blocks
  const int n_chunk = (K + TC_KC - 1) / TC_KC;
  const int my_tiles = blockIdx.x < n_tiles ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const unsigned int total = (unsigned int)(n_lb * my_tiles * n_chunk);     // (lane block, tile, chunk) sequence of this CTA
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
  const int wr = (wg & 1) * 64, wc = (wg >> 1) * 128;          // this warpgroup's rows / columns of the tile
  const int rq = (warp & 3) * 16 + (lane >> 2);                 // first of the thread's two rows inside the warpgroup's 64
  unsigned int it = 0;
  for (int lb = 0; lb < n_lb; lb++) {
    lane_block(lb * TC_M + wr + rq);
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; i++) d[i] = 0.f;
      for (int c = 0; c < n_chunk; c++, it++) {
        const uint32_t st = it % TC_STAGES, use = it / TC_STAGES;
        tc_mbar_wait(&sm.stage_full[st], use & 1u, &sm.err);                         // operand blocks have landed
        const uint32_t a_hi = tc_smem_u32(sm.stage[st]) + wr * 128, a_lo = a_hi + TC_A_BYTES;
        const uint32_t b_hi = tc_smem_u32(sm.stage[st]) + 2 * TC_A_BYTES + wc * 128, b_lo = b_hi + TC_B_BYTES;
        wg_chunk_3xtf32(d, a_hi, a_lo, b_hi, b_lo);
        if ((tid & 127) == 0) tc_mbar_arrive(&sm.stage_free[st]);
        if (tid == 0 && it + TC_STAGES < total) { tc_mbar_wait(&sm.stage_free[st], use & 1u, &sm.err); issue(it + TC_STAGES); }
        __syncwarp();
      }
      tile(d, t * TC_N + wc + 2 * (lane & 3), t + (int)gridDim.x >= n_tiles);
    }
  }
}

// cnt[b*2 + 0] += #items with score > target score of lane b; cnt[b*2 + 1] += #items with score == target (the target itself
// counts as one tie, exactly as in the fp32 kernel where its score equals the target score bit for bit).  Each thread counts its
// two lanes x 32 items of a tile thread-locally; the four threads of a quad sum their counts after the lane block's last tile.
// SEEN: the items of a lane's seen list are taken back out the way the target's column is -- the seen items among the columns the
// thread holds become a bit mask, and the same d[i] that was counted is uncounted, so no seen item is ever counted, exactly.  The
// CTA visits a lane block's tiles in increasing column order, so each lane keeps a cursor into its list with the next seen item
// already loaded: a tile without a seen item costs no load, a cursor behind the tile jumps by a binary search (O(log cap + seen
// items in the tile) per lane and tile at worst)
template <bool SEEN = false>
__global__ void __launch_bounds__(TC_THREADS, 1) k_eval_tc(int slot, int s, const float* __restrict__ tgt, int tgt_stride, int* cnt,
                                                           const unsigned char* __restrict__ Asplit, const unsigned char* __restrict__ Bsplit,
                                                           SeenDev sd = SeenDev{}) {
  const ModelDev& md = MD;
  const int M = md.wM[s], I = md.n_items, lane = threadIdx.x & 31;
  int bb[2], yit[2]; bool vrow[2]; float lo[2], hi[2];
  int cgt[2], cge[2];
  const int* sl_l[2]; int sl_n[2], sl_p[2], sl_nx[2];              // SEEN: the two lanes' lists, cursors and next seen items
  auto lane_block = [&](int b) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      bb[h] = b + 8 * h;
      vrow[h] = bb[h] < M;
      yit[h] = vrow[h] ? md.wY[(size_t)s * md.B + bb[h]] : -1;
      lo[h] = vrow[h] ? tgt[tgt_stride + bb[h]] : INFINITY; hi[h] = vrow[h] ? tgt[2 * tgt_stride + bb[h]] : INFINITY;   // k_eval_tgt
      cgt[h] = 0; cge[h] = 0;
      if (SEEN) {
        const int sl = vrow[h] ? md.wSlot[(size_t)s * md.B + bb[h]] : 0;
        sl_l[h] = sd.list + (size_t)sl * sd.cap; sl_n[h] = vrow[h] ? sd.n[sl] : 0;
        sl_p[h] = 0; sl_nx[h] = sl_n[h] > 0 ? sl_l[h][0] : INT_MAX;
      }
    }
  };
  auto tile = [&](const float (&d)[64], int c0, bool last) {
    // two compares per item against the lane's pre-activation thresholds; columns past the catalogue (last tile) do not count
    const int n_live = I - c0;
#pragma unroll
    for (int i = 0; i < 64; i++) {
      const int h = (i >> 1) & 1;
      const bool live = (i >> 2) * 8 + (i & 1) < n_live;
      cgt[h] += (live && d[i] > hi[h]) ? 1 : 0;
      cge[h] += (live && d[i] >= lo[h]) ? 1 : 0;
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int rel = yit[h] - c0;                                 // the target's own column, if this thread holds it
      if (rel >= 0 && rel < 128 && (rel & 7) < 2) {               // rare: take it back out, it counts as exactly one tie
        float xs = 0.f;
#pragma unroll
        for (int i = 0; i < 64; i++) if (((i >> 1) & 1) == h && (i >> 2) * 8 + (i & 1) == rel) xs = d[i];
        cgt[h] -= (xs > hi[h]) ? 1 : 0;
        cge[h] -= (xs >= lo[h]) ? 1 : 0;
        cge[h] += 1;                                               // == (self: not above) + one tie
      }
    }
    if (SEEN) {
      unsigned int xm[2];                                          // bit 2 (i / 4) + i % 2: column of d[i] is a seen item
#pragma unroll
      for (int h = 0; h < 2; h++) {
        xm[h] = 0u;
        if (sl_nx[h] < c0) {                                       // seen items in other CTAs' tiles: jump past them
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
      if (xm[0] | xm[1]) {
#pragma unroll
        for (int i = 0; i < 64; i++) {
          const int h = (i >> 1) & 1;
          if ((xm[h] >> ((i >> 2) * 2 + (i & 1))) & 1u) { cgt[h] -= (d[i] > hi[h]) ? 1 : 0; cge[h] -= (d[i] >= lo[h]) ? 1 : 0; }
        }
      }
    }
    if (!last) return;
#pragma unroll
    for (int h = 0; h < 2; h++) {                                  // the four threads of a quad share the two rows
      int g = cgt[h], e = cge[h] - cgt[h];                         // lo <= x <= hi
      g += __shfl_xor_sync(0xffffffffu, g, 1); g += __shfl_xor_sync(0xffffffffu, g, 2);
      e += __shfl_xor_sync(0xffffffffu, e, 1); e += __shfl_xor_sync(0xffffffffu, e, 2);
      if ((lane & 3) == 0 && vrow[h]) { if (g) atomicAdd(&cnt[bb[h] * 2], g); if (e) atomicAdd(&cnt[bb[h] * 2 + 1], e); }
    }
  };
  tc_sweep(M, I, md.L + 1, Asplit, Bsplit, lane_block, tile);
}
