// g4r_tcstep.cuh -- the training step on the 5th-generation tensor cores for the LARGE shared-embedding shapes
// (constrained_embedding, one GRU layer, hidden size >= 160, batch <= 256: paramfiles/{rees46,coveo,diginetica,yoochoose,
// retailrocket}_*_best.py of the reference -- B = 48..240, L = 224..512, 2048 negative samples).  At these shapes a mini-batch is
// ~4 GFLOP of dense contractions (gru4rec.py:460-461 gates, :493 sampled scores, and their gradients from T.grad, :383-384);
// the generic kernels run them on FP32 FFMA tiles.  Here every contraction is a wgmma GEMM (Hopper tensor cores):
//
//   operands  fp32 values are split into hi = tf32(x), lo = tf32(x - hi) ("3xTF32": lo*hi + hi*lo + hi*hi accumulated in fp32
//             reproduces the fp32 product to ~2^-21 relative) and stored as [hi | lo] blocks of 128 rows x 32 k-values in the
//             K-major 128-byte-swizzle layout by small "prep" kernels that also do the gathers
//             (Wy[item] rows of the score columns, H through the lane slots), transposes and elementwise products (H * r);
//   GEMM      128 x 256 output tiles (128 x 128 where the product has at most 128 columns); K is split over the CTAs of a
//             thread-block cluster.  Per CTA: thread 0 streams the operand blocks with bulk copies into a shared-memory ring
//             (mbarrier complete_tx), four warpgroups issue wgmma.mma_async kind tf32 (m64, N = NT / 2, k8) on their quarter of the
//             tile with the accumulator in registers; the partial tile goes through L2, and after a cluster barrier each CTA adds
//             the K splits of its band of rows in K order and applies the fused epilogue (gates + sigmoid + the H*r operand,
//             candidate + GRU update + dropout + reset + the score operand, score + bias, dSy rows, b1 = elementwise GRU backward +
//             operands, da_r, dL/d(input));
//             the two dense-gradient products leave their partial tiles to an elementwise kernel that does the optimizer step;
//   schedule  three streams joined by events (captured into the step graph), programmatic dependent launch along the main chain;
//   the rest  row statistics + dL/do (one kernel per step), and the deterministic sparse updates reuse the generic phases
//             (g4r_kernels.cuh) -- same numerics, same duplicate rules.
// Included from g4r_lib.cu after g4r_eval.cuh (uses its mbarrier / wgmma helpers).
#pragma once
#include <cooperative_groups.h>

constexpr int TS_RB = 128;                               // rows per operand block
constexpr uint32_t TS_BLK = TS_RB * TC_KC * 4;           // bytes of one hi (or lo) block: 16 KB
constexpr int TS_THREADS = 512;                          // four MMA warpgroups (64 rows x NT / 2 columns each); all 16 warps run the reduce / epilogue




// programmatic dependent launch: a kernel launched with the attribute may start (and set itself up) while its predecessor in the
// stream still runs; it consumes the predecessor's results only after pdl_wait().  No-ops for ordinary launches.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void ts_put4(unsigned char* base, int n_chunk, int row, int k, float4 v) {
  const int rb = row / TS_RB, r = row % TS_RB, c = k / TC_KC, kq = (k % TC_KC) >> 2;
  unsigned char* hi = base + ((size_t)rb * n_chunk + c) * 2 * TS_BLK + tc_block_off(r, kq);
  uint4 h, l;
  h.x = tc_tf32(v.x); h.y = tc_tf32(v.y); h.z = tc_tf32(v.z); h.w = tc_tf32(v.w);
  l.x = tc_tf32(v.x - __uint_as_float(h.x)); l.y = tc_tf32(v.y - __uint_as_float(h.y));
  l.z = tc_tf32(v.z - __uint_as_float(h.z)); l.w = tc_tf32(v.w - __uint_as_float(h.w));
  *reinterpret_cast<uint4*>(hi) = h;
  *reinterpret_cast<uint4*>(hi + TS_BLK) = l;
}
// fills a [rows_pad x K_pad] operand: f(row, k) -> the four values (row, k .. k+3); k_fast: consecutive threads walk k (sources
// with k contiguous in memory) else rows (transposed / gathered sources)
template <class F>
__device__ __forceinline__ void ts_fill(unsigned char* base, int rows_pad, int K_pad, bool k_fast, F f) {
  const int n_chunk = K_pad / TC_KC, kq_n = K_pad / 4;
  const long long total = (long long)rows_pad * kq_n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int row, kq;
    if (k_fast) { row = (int)(i / kq_n); kq = (int)(i % kq_n); } else { kq = (int)(i / rows_pad); row = (int)(i % rows_pad); }
    ts_put4(base, n_chunk, row, kq * 4, f(row, kq * 4));
  }
}
__device__ __forceinline__ float4 ts_zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }
// column sums over the lanes with 8 row groups per column and a fixed-order merge: out(col) is called once per column
template <class FLoad, class FOut>
__device__ __forceinline__ void ts_colsum(int n_cols, int n_rows, FLoad ld, FOut out) {
  __shared__ float red[8][33];
  const int cg = threadIdx.x & 31, rg = threadIdx.x >> 5;
  for (int c0 = blockIdx.x * 32; c0 < n_cols; c0 += gridDim.x * 32) {
    const int c = c0 + cg;
    float a = 0.f;
    if (c < n_cols) for (int b = rg; b < n_rows; b += 8) a += ld(b, c);
    red[rg][cg] = a;
    __syncthreads();
    if (rg == 0 && c < n_cols) { float t = 0.f; for (int k = 0; k < 8; k++) t += red[k][cg]; out(c, t); }
    __syncthreads();
  }
}


struct TsGemm {
  const unsigned char* A; const unsigned char* Bm;
  float* P;              // partial tiles [ksplit][m_tiles * 128][ldP]
  int fused;                 // 1: the K splits are a cluster, reduce + epilogue in the kernel; 0: k_ts_epi does it
  unsigned long long* dbg;   // per-CTA phase timestamps (G4R_TS_STAMP=1), else nullptr
  int chunks;            // K_pad / 32 (both operands)
  int m_tiles, n_tiles, NT, ksplit, ldP;
  int epi;
};

// ---- P1: gather of the input rows (shared table, embedding dropout, optimizer-state snapshots: phase_gather_in), A1 = [in0 | H(slot)]
// (lanes x 2L), the in0 half of A2 = [in0 | Hold * r], compact copy of the old hidden state (gru4rec.py:459-461 operands); the
// Hold * r half of A2 comes from the gate epilogue ----
__device__ __forceinline__ float4 ts_in0_quad(const ModelDev& md, int s, int b, int k, int item) {
  float4 v = ld4(md.Wy + (size_t)item * md.ld_in0 + k);
  if (md.p_drop_e > 0.f) {
    const uint32_t e = (uint32_t)(b * md.in0_dim + k); const float keep = 1.0f - md.p_drop_e; const uint32_t gs = md.wG[s];
    v.x *= drop_scale(md.drop_seed, gs, G4R_STREAM_EMBED, e, keep); v.y *= drop_scale(md.drop_seed, gs, G4R_STREAM_EMBED, e + 1, keep);
    v.z *= drop_scale(md.drop_seed, gs, G4R_STREAM_EMBED, e + 2, keep); v.w *= drop_scale(md.drop_seed, gs, G4R_STREAM_EMBED, e + 3, keep);
  }
  return v;
}
__global__ void __launch_bounds__(256) k_ts_prep_fwd(int slot, const int* base, int off, TsBuf tb) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL, L4 = L / 4;
  const int* __restrict__ wX = md.wX + (size_t)s * md.B;
  pdl_trigger();
  if (blockIdx.y == 0) {          // A1, in0 half of A2, in0 itself
    const int n_chunk = tb.Lk2 / TC_KC;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < M * 2 * L4; i += gridDim.x * blockDim.x) {
      const int b = i / (2 * L4), k = (i % (2 * L4)) * 4;
      if (k < L) {
        const float4 v = ts_in0_quad(md, s, b, k, wX[b]);
        st4(md.in0 + (size_t)b * md.ld_in0 + k, v);
        ts_put4(tb.A1, n_chunk, b, k, v);
        ts_put4(tb.A2, n_chunk, b, k, v);
      } else {
        const int sl = (md.wF[(size_t)s * md.B + b] & 2) ? -1 : md.wSlot[(size_t)s * md.B + b];
        const float4 hv = sl >= 0 ? ld4(ly.H + (size_t)sl * ldL + (k - L)) : ts_zero4();
        st4(ly.Hold + (size_t)b * ldL + (k - L), hv);
        ts_put4(tb.A1, n_chunk, b, k, hv);
      }
    }
  } else {                        // raw rows (no dropout) and optimizer-state snapshots for the input-row update
    const int ld = md.ld_in0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < M * (ld / 4); i += gridDim.x * blockDim.x) {
      const int b = i / (ld / 4), c = (i % (ld / 4)) * 4;
      const size_t src = (size_t)wX[b] * ld + c, dst = (size_t)b * ld + c;
      st4(md.Sx + dst, ld4(md.Wy + src));
      if (md.Wy_acc) st4(md.snapAcc + dst, ld4(md.Wy_acc + src));
      if (md.Wy_vel) st4(md.snapVel + dst, ld4(md.Wy_vel + src));
    }
  }
}
// ---- P2: weight operands (they change every step: dense update) ----
//   W1 (n < 2L, k < 2L): k < L ? Wx[k][L + n] : Wrz[k - L][n]      gates        (gru4rec.py:460)
//   W2 (n <  L, k < 2L): k < L ? Wx[k][n]     : Wh[k - L][n]       candidate    (gru4rec.py:461)
//   W3 (n <  L, k <  L): Wh[n][k]                                   d(H*r) = da_h Wh^T
//   W4 (n <  L, k < 3L): Wx[n][k]                                   dL/d(input) = dvec Wx^T
__global__ void __launch_bounds__(256) k_ts_prep_w(int slot, TsBuf tb) {
  const ModelDev& md = MD;
  const LayerDev& ly = md.layer[0];
  const int L = ly.L;
  const float* __restrict__ Wx = ly.Wx; const float* __restrict__ Wh = ly.Wh; const float* __restrict__ Wrz = ly.Wrz;
  if (blockIdx.y == 0) {
    ts_fill(tb.W1, (2 * L + TS_RB - 1) / TS_RB * TS_RB, tb.Lk2, false, [&](int n, int k) -> float4 {
      float v[4];
      for (int u = 0; u < 4; u++) { const int kk = k + u; v[u] = (n < 2 * L && kk < 2 * L) ? (kk < L ? Wx[(size_t)kk * ly.ld3 + L + n] : Wrz[(size_t)(kk - L) * ly.ld2 + n]) : 0.f; }
      return make_float4(v[0], v[1], v[2], v[3]);
    });
  } else if (blockIdx.y == 1) {
    ts_fill(tb.W2, (L + TS_RB - 1) / TS_RB * TS_RB, tb.Lk2, false, [&](int n, int k) -> float4 {
      float v[4];
      for (int u = 0; u < 4; u++) { const int kk = k + u; v[u] = (n < L && kk < 2 * L) ? (kk < L ? Wx[(size_t)kk * ly.ld3 + n] : Wh[(size_t)(kk - L) * ly.ldL + n]) : 0.f; }
      return make_float4(v[0], v[1], v[2], v[3]);
    });
  } else if (blockIdx.y == 2) {
    ts_fill(tb.W3, (L + TS_RB - 1) / TS_RB * TS_RB, tb.Lk1, true, [&](int n, int k) -> float4 { return (n < L && k < L) ? ld4(Wh + (size_t)n * ly.ldL + k) : ts_zero4(); });
  } else {
    ts_fill(tb.W4, (L + TS_RB - 1) / TS_RB * TS_RB, tb.Lk3, true, [&](int n, int k) -> float4 { return (n < L && k < 3 * L) ? ld4(Wx + (size_t)n * ly.ld3 + k) : ts_zero4(); });
  }
}
// ---- P3: item-table operands of the score product and of dL/dh (they depend on the previous step's sparse update only) ----
//   B3 (j, k < L) = Wy[item_j][k];  B5 (c < L, k = j) = Wy[item_j][c];  bias[j] = By[item_j] - logq * log(P0 ...) (gru4rec.py:486-495)
__global__ void __launch_bounds__(256) k_ts_prep_tab(int slot, const int* base, int off, TsBuf tb) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL;
  const int N = M + (md.wSti[s] >= 0 ? md.S : 0);
  const int* __restrict__ pItem = md.pItem + (size_t)s * md.NP;
  const float* __restrict__ Wy = md.Wy;
  if (blockIdx.y == 0) {
    ts_fill(tb.B3, tb.Nk, tb.Lk1, true, [&](int j, int k) -> float4 { return (j < N && k < L) ? ld4(Wy + (size_t)pItem[j] * ldL + k) : ts_zero4(); });
  } else if (blockIdx.y == 1) {
    ts_fill(tb.B5, (L + TS_RB - 1) / TS_RB * TS_RB, tb.Nk, false, [&](int c, int k) -> float4 {
      float v[4];
      for (int u = 0; u < 4; u++) { const int j = k + u; v[u] = (c < L && j < N) ? Wy[(size_t)pItem[j] * ldL + c] : 0.f; }
      return make_float4(v[0], v[1], v[2], v[3]);
    });
  } else {
    const int* __restrict__ pPos = md.pPos + (size_t)s * md.NP;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += gridDim.x * blockDim.x) {
      const int item = pItem[j];
      float bz = md.By[item];
      if (md.logq > 0.f) bz -= (pPos[j] < M) ? md.logP0t[item] : md.logP0s[item];
      tb.bias[j] = bz;
    }
  }
}
// ---- P4: left operand of the dense-gradient product, A8 (m < 3L, k = b) = [Hold*r ; Hold ; in0]^T (known once the gates are) ----
__global__ void __launch_bounds__(256) k_ts_prep_a8(int slot, const int* base, int off, TsBuf tb) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL;
  const int R3 = (3 * L + TS_RB - 1) / TS_RB * TS_RB;
  ts_fill(tb.A8, R3, tb.Bk, false, [&](int mrow, int k) -> float4 {
    float v[4];
    for (int u = 0; u < 4; u++) {
      const int b = k + u;
      float x = 0.f;
      if (mrow < 3 * L && b < M) {
        if (mrow < L) x = ly.Hold[(size_t)b * ldL + mrow] * ly.r[(size_t)b * ldL + mrow];
        else if (mrow < 2 * L) x = ly.Hold[(size_t)b * ldL + mrow - L];
        else x = md.in0[(size_t)b * md.ld_in0 + mrow - 2 * L];
      }
      v[u] = x;
    }
    return make_float4(v[0], v[1], v[2], v[3]);
  });
}
// ---- P5: B4 (c < L, k = b) = h[b][c] (right operand of dSy) ----
__global__ void __launch_bounds__(256) k_ts_prep_yt(int slot, const int* base, int off, TsBuf tb) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL;
  ts_fill(tb.B4, (L + TS_RB - 1) / TS_RB * TS_RB, tb.Bk, false, [&](int c, int k) -> float4 {
    float v[4];
    for (int u = 0; u < 4; u++) { const int b = k + u; v[u] = (c < L && b < M) ? ly.y[(size_t)b * ldL + c] : 0.f; }
    return make_float4(v[0], v[1], v[2], v[3]);
  });
}

// ---- row statistics of the losses from the lane-major score matrix (same merge as phase_score / phase_stats), then dL/do of the
// same row in place and as the left operand A5 (b, k = j) of the dL/dh product: a row needs only its own statistics ----
__global__ void __launch_bounds__(256) k_ts_loss(int slot, const int* base, int off, TsBuf tb) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const int M = md.wM[s];
  const int N = M + (md.wSti[s] >= 0 ? md.S : 0);
  const int b = blockIdx.x;
  pdl_wait(); pdl_trigger();
  if (b >= M) return;
  __shared__ float sW[8 * 8];
  __shared__ float sRS[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* orow = tb.O + (size_t)b * tb.ldO;
  const int tc = md.pTcol[(size_t)s * md.B + b];
  const bool pw = loss_pairwise(md.loss);
  const float t = pw ? act_fwd(md.fact, orow[tc]) : 0.f;
  float m = -INFINITY, Z = 0.f, A = 0.f, Q = 0.f, D = 0.f, T = 0.f, has = 0.f;
  for (int j = tid * 4; j < N; j += blockDim.x * 4) {
    const float4 v = ld4(orow + j);
    stat_add_elem(md, v.x, j == tc, t, m, Z, A, Q, D, T, has);
    if (j + 1 < N) stat_add_elem(md, v.y, j + 1 == tc, t, m, Z, A, Q, D, T, has);
    if (j + 2 < N) stat_add_elem(md, v.z, j + 2 == tc, t, m, Z, A, Q, D, T, has);
    if (j + 3 < N) stat_add_elem(md, v.w, j + 3 == tc, t, m, Z, A, Q, D, T, has);
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {   // fixed butterfly order
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), Z2 = __shfl_xor_sync(0xffffffffu, Z, o), A2 = __shfl_xor_sync(0xffffffffu, A, o),
                Q2 = __shfl_xor_sync(0xffffffffu, Q, o), D2 = __shfl_xor_sync(0xffffffffu, D, o), T2 = __shfl_xor_sync(0xffffffffu, T, o),
                h2 = __shfl_xor_sync(0xffffffffu, has, o);
    stat_combine(md, m, Z, A, Q, D, T, has, m2, Z2, A2, Q2, D2, T2, h2);
  }
  if (lane == 0) { float* w = sW + warp * 8; w[0] = m; w[1] = Z; w[2] = A; w[3] = Q; w[4] = D; w[5] = T; w[6] = has; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; w++) { const float* q = sW + w * 8; stat_combine(md, m, Z, A, Q, D, T, has, q[0], q[1], q[2], q[3], q[4], q[5], q[6]); }
    if (loss_softmaxneg(md.loss)) stat_merge(m, Z, A, Q, D, 0.f, 0.f, 0.f, 0.f, 0.f);   // the zeroed diagonal takes part in the max (gru4rec.py:200-202)
    stats_finalize(md, b, M, N, m, Z, A, Q, D, T, t);
  }
  __syncthreads();
  if (tid < 8) sRS[tid] = md.RS[(size_t)b * G4R_NSTAT + tid];
  __syncthreads();
  const int n_chunk = tb.Nk / TC_KC;
  for (int j = tid * 4; j < tb.Nk; j += blockDim.x * 4) {      // the K padding of A5 beyond the live columns is rewritten with zeros
    float4 v = ts_zero4();
    if (j < N) {
      v = ld4(orow + j);
      v.x = loss_grad_elem(md, sRS, v.x, j == tc, M, N);
      v.y = j + 1 < N ? loss_grad_elem(md, sRS, v.y, j + 1 == tc, M, N) : 0.f;
      v.z = j + 2 < N ? loss_grad_elem(md, sRS, v.z, j + 2 == tc, M, N) : 0.f;
      v.w = j + 3 < N ? loss_grad_elem(md, sRS, v.w, j + 3 == tc, M, N) : 0.f;
      st4(orow + j, v);
    }
    ts_put4(tb.A5, n_chunk, b, j, v);
  }
}
// ---- P6: A4 (j, k = b) = G[b][j] (left operand of dSy); dby[j] = sum_b G[b][j] ----
__global__ void __launch_bounds__(256) k_ts_prep_g(int slot, const int* base, int off, TsBuf tb) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const int M = md.wM[s];
  const int N = M + (md.wSti[s] >= 0 ? md.S : 0);
  const float* __restrict__ G = tb.O;
  if (blockIdx.y == 0) {
    ts_fill(tb.A4, tb.Nk, tb.Bk, false, [&](int j, int k) -> float4 {
      float v[4];
      for (int u = 0; u < 4; u++) { const int b = k + u; v[u] = (j < N && b < M) ? G[(size_t)b * tb.ldO + j] : 0.f; }
      return make_float4(v[0], v[1], v[2], v[3]);
    });
  } else {
    ts_colsum(N, M, [&](int b, int j) { return G[(size_t)b * tb.ldO + j]; }, [&](int j, float t) { md.DBY[j] = t; });
  }
}
// ---- P7: right operands of the dense-gradient products (k = b): B8a rows [0, Lp) = da_h^T, [Lp, 2 Lp) = da_z^T (known after b1),
// B8b rows [0, L) = da_r^T (known after b2) ----
__global__ void __launch_bounds__(256) k_ts_prep_b8(int slot, const int* base, int off, TsBuf tb, int part) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L;
  if (part == 0) {
    ts_fill(tb.B8a, 2 * tb.Lp, tb.Bk, false, [&](int n, int k) -> float4 {
      const int seg = n / tb.Lp, c = n % tb.Lp;
      float v[4];
      for (int u = 0; u < 4; u++) { const int b = k + u; v[u] = (c < L && b < M) ? ly.dvec[(size_t)b * ly.ld3 + (seg ? 2 * L : 0) + c] : 0.f; }
      return make_float4(v[0], v[1], v[2], v[3]);
    });
  } else {
    ts_fill(tb.B8b, (L + TS_RB - 1) / TS_RB * TS_RB, tb.Bk, false, [&](int n, int k) -> float4 {
      float v[4];
      for (int u = 0; u < 4; u++) { const int b = k + u; v[u] = (n < L && b < M) ? ly.dvec[(size_t)b * ly.ld3 + L + n] : 0.f; }
      return make_float4(v[0], v[1], v[2], v[3]);
    });
  }
}
// ---- dBh = sum_b dvec (gru4rec.py:462 bias gradient) with its update ----
__global__ void __launch_bounds__(256) k_ts_bh(int slot, const int* base, int off) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s];
  pdl_wait(); pdl_trigger();
  ts_colsum(3 * ly.L, M, [&](int b, int c) { return ly.dvec[(size_t)b * ly.ld3 + c]; },
            [&](int c, float g) { dense_update(md, ly.Bh + c, ly.Bh_acc ? ly.Bh_acc + c : nullptr, ly.Bh_vel ? ly.Bh_vel + c : nullptr, g, (size_t)ly.ld3); });
}

// ---------------------------------------------------------------------------------------------------------------------
// the GEMM: D[128 x NT tile] = A[128 x K] B[NT x K]^T, 3xTF32.  The parallelism comes from splitting K over the CTAs of a
// thread-block CLUSTER: each CTA accumulates its K slice in registers, writes the partial tile to L2, and after a cluster barrier
// every CTA sums one band of rows over all peers (fixed order) and applies the fused epilogue with coalesced accesses.
// (TsGemm.fused == 0: k_ts_epi reduces the partial tiles instead -- the dense-update products, whose epilogue is a full optimizer
// step per element and wants the whole GPU.)
// ---------------------------------------------------------------------------------------------------------------------
enum { TS_EPI_F1 = 0, TS_EPI_F2, TS_EPI_SCORE, TS_EPI_DSY, TS_EPI_DH, TS_EPI_B2, TS_EPI_B3, TS_EPI_DENSE_A, TS_EPI_DENSE_B };
// live extent of a product at this step (dynamic mini-batch size / column count)
template <int EPI>
__device__ __forceinline__ void ts_limits(const ModelDev& md, const TsBuf& tb, int M, int N, int& m_lim, int& n_lim) {
  const int L = md.layer[0].L;
  if (EPI == TS_EPI_F1) { m_lim = M; n_lim = 2 * L; }
  else if (EPI == TS_EPI_SCORE) { m_lim = M; n_lim = (N + 3) & ~3; }
  else if (EPI == TS_EPI_DSY) { m_lim = N; n_lim = L; }
  else if (EPI == TS_EPI_DENSE_A) { m_lim = 3 * L; n_lim = 2 * tb.Lp; }
  else if (EPI == TS_EPI_DENSE_B) { m_lim = 3 * L; n_lim = L; }
  else { m_lim = M; n_lim = L; }
}
// does the tile [m0, m0 + 128) x [n0, n0 + NT) hold any live output?
template <int EPI>
__device__ __forceinline__ bool ts_tile_live(const ModelDev& md, const TsBuf& tb, int M, int N, int m0, int n0) {
  int m_lim, n_lim;
  ts_limits<EPI>(md, tb, M, N, m_lim, n_lim);
  if (m0 >= m_lim || n0 >= n_lim) return false;
  const int L = md.layer[0].L;
  if (EPI == TS_EPI_DENSE_A || EPI == TS_EPI_DENSE_B) {
    const int blo = m0 / L, bhi = min(m0 + TS_RB - 1, 3 * L - 1) / L;      // feature blocks (H*r | H | in0) the tile's rows touch
    if (EPI == TS_EPI_DENSE_B) return bhi >= 1;                            // da_r: dWrz and dWx only
    if (n0 % tb.Lp >= L) return false;
    return n0 / tb.Lp == 0 ? (blo == 0 || bhi == 2) : bhi >= 1;            // da_h: dWh, dWx;  da_z: dWrz, dWx
  }
  return true;
}
// fused epilogue of four consecutive columns (m, n .. n+3) of a product; every live extent along n is a multiple of 4 (L % 4 == 0)
template <int EPI>
__device__ __forceinline__ void ts_epilogue4(const ModelDev& md, const TsBuf& tb, int s, int m, int n, float4 v) {
  const LayerDev& ly = md.layer[0];
  const int L = ly.L, ldL = ly.ldL;
  if (EPI == TS_EPI_F1) {          // rz = sigmoid(vec[:, L:] + H Wrz) (gru4rec.py:460); the r half also makes the Hold * r part of A2
    const float4 bh = ldn4(ly.Bh + L + n);
    const float4 g = make_float4(sigmoidf_(v.x + bh.x), sigmoidf_(v.y + bh.y), sigmoidf_(v.z + bh.z), sigmoidf_(v.w + bh.w));
    if (n < L) {
      st4(ly.r + (size_t)m * ldL + n, g);
      const float4 ho = ldn4(ly.Hold + (size_t)m * ldL + n);
      ts_put4(tb.A2, tb.Lk2 / TC_KC, m, L + n, make_float4(ho.x * g.x, ho.y * g.y, ho.z * g.z, ho.w * g.w));
    } else st4(ly.z + (size_t)m * ldL + (n - L), g);
  } else if (EPI == TS_EPI_F2) {   // h~ = act((H * r) Wh + vec[:, :L]); h = (1 - z) H + z h~; dropout; reset (gru4rec.py:461-466); h is also A3
    const float4 bh = ldn4(ly.Bh + n), z = ldn4(ly.z + (size_t)m * ldL + n), ho = ldn4(ly.Hold + (size_t)m * ldL + n);
    const float a[4] = {v.x + bh.x, v.y + bh.y, v.z + bh.z, v.w + bh.w}, zv[4] = {z.x, z.y, z.z, z.w}, hov[4] = {ho.x, ho.y, ho.z, ho.w};
    float ht[4], hn[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      ht[u] = act_fwd(md.hact, a[u]);
      hn[u] = (1.0f - zv[u]) * hov[u] + zv[u] * ht[u];
      if (md.p_drop_h > 0.f) hn[u] *= drop_scale(md.drop_seed, md.wG[s], 0u, (uint32_t)(m * L + n + u), 1.0f - md.p_drop_h);
    }
    const float4 h4 = make_float4(hn[0], hn[1], hn[2], hn[3]);
    st4(ly.ah + (size_t)m * ldL + n, make_float4(a[0], a[1], a[2], a[3]));
    st4(ly.ht + (size_t)m * ldL + n, make_float4(ht[0], ht[1], ht[2], ht[3]));
    st4(ly.y + (size_t)m * ldL + n, h4);
    st4(ly.H + (size_t)md.wSlot[(size_t)s * md.B + m] * ldL + n, (md.wF[(size_t)s * md.B + m] & 1) ? ts_zero4() : h4);
    ts_put4(tb.A3, tb.Lk1 / TC_KC, m, n, h4);
  } else if (EPI == TS_EPI_SCORE) { // o = h Sy^T + by (- logq correction) (gru4rec.py:493-495), lane-major
    const float4 bz = ldn4(tb.bias + n);
    st4(tb.O + (size_t)m * tb.ldO + n, make_float4(v.x + bz.x, v.y + bz.y, v.z + bz.z, v.w + bz.w));
  } else if (EPI == TS_EPI_DSY) {  // dSy_j = sum_b g[b][j] h[b]
    st4(md.DSY + (size_t)m * ldL + n, v);
  } else if (EPI == TS_EPI_DH) {   // b1: v = dL/dh; elementwise GRU backward (SURVEY appendix A); da_h / da_z go to dvec and into A6 = da_h, A7 = dvec
    const size_t o = (size_t)m * ldL + n;
    const float4 ht = ldn4(ly.ht + o), ho = ldn4(ly.Hold + o), z = ldn4(ly.z + o), ah = ldn4(ly.ah + o);
    const float dyv[4] = {v.x, v.y, v.z, v.w}, htv[4] = {ht.x, ht.y, ht.z, ht.w}, hov[4] = {ho.x, ho.y, ho.z, ho.w}, zv[4] = {z.x, z.y, z.z, z.w},
                ahv[4] = {ah.x, ah.y, ah.z, ah.w};
    float dah[4], dz[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      float dh = dyv[u];
      if (md.p_drop_h > 0.f) dh *= drop_scale(md.drop_seed, md.wG[s], 0u, (uint32_t)(m * L + n + u), 1.0f - md.p_drop_h);
      dah[u] = dh * zv[u] * act_der(md.hact, ahv[u], htv[u]);
      dz[u] = dh * (htv[u] - hov[u]) * zv[u] * (1.f - zv[u]);
    }
    const float4 a4 = make_float4(dah[0], dah[1], dah[2], dah[3]), z4 = make_float4(dz[0], dz[1], dz[2], dz[3]);
    st4(ly.dvec + (size_t)m * ly.ld3 + n, a4);
    st4(ly.dvec + (size_t)m * ly.ld3 + 2 * L + n, z4);
    ts_put4(tb.A6, tb.Lk1 / TC_KC, m, n, a4);
    ts_put4(tb.A7, tb.Lk3 / TC_KC, m, n, a4);
    ts_put4(tb.A7, tb.Lk3 / TC_KC, m, 2 * L + n, z4);
  } else if (EPI == TS_EPI_B2) {   // da_r = (da_h Wh^T) * H * r (1 - r); completes dvec and its operand A7
    const float4 r = ldn4(ly.r + (size_t)m * ldL + n), ho = ldn4(ly.Hold + (size_t)m * ldL + n);
    const float4 d = make_float4(v.x * ho.x * r.x * (1.f - r.x), v.y * ho.y * r.y * (1.f - r.y), v.z * ho.z * r.z * (1.f - r.z), v.w * ho.w * r.w * (1.f - r.w));
    st4(ly.dvec + (size_t)m * ly.ld3 + L + n, d);
    ts_put4(tb.A7, tb.Lk3 / TC_KC, m, L + n, d);
  } else if (EPI == TS_EPI_B3) {   // dL/d(gathered input row) = (dvec Wx^T) * embedding-dropout mask
    if (md.p_drop_e > 0.f) {
      const uint32_t e = (uint32_t)(m * L + n); const float keep = 1.0f - md.p_drop_e;
      v.x *= drop_scale(md.drop_seed, md.wG[s], G4R_STREAM_EMBED, e, keep); v.y *= drop_scale(md.drop_seed, md.wG[s], G4R_STREAM_EMBED, e + 1, keep);
      v.z *= drop_scale(md.drop_seed, md.wG[s], G4R_STREAM_EMBED, e + 2, keep); v.w *= drop_scale(md.drop_seed, md.wG[s], G4R_STREAM_EMBED, e + 3, keep);
    }
    st4(md.dSx + (size_t)m * md.ld_in0 + n, v);
  } else {   // dense gradients + update: rows m = [H*r | H | in0] features; columns = da_h | da_z (A) or da_r (B)  (dWh, dWrz, dWx, gru4rec.py:390-406)
    int col;                       // column of dvec = [da_h | da_r | da_z]
    if (EPI == TS_EPI_DENSE_A) { const int c = n % tb.Lp; if (c >= L) return; col = n / tb.Lp ? 2 * L + c : c; }
    else col = L + n;
    float* p; float* acc; float* vel; size_t ast;
    if (m < L) { if (col >= L) return; const size_t o = (size_t)m * ldL + col; p = ly.Wh + o; acc = ly.Wh_acc ? ly.Wh_acc + o : nullptr; vel = ly.Wh_vel ? ly.Wh_vel + o : nullptr; ast = (size_t)L * ldL; }
    else if (m < 2 * L) { if (col < L) return; const size_t o = (size_t)(m - L) * ly.ld2 + (col - L); p = ly.Wrz + o; acc = ly.Wrz_acc ? ly.Wrz_acc + o : nullptr; vel = ly.Wrz_vel ? ly.Wrz_vel + o : nullptr; ast = (size_t)L * ly.ld2; }
    else { const size_t o = (size_t)(m - 2 * L) * ly.ld3 + col; p = ly.Wx + o; acc = ly.Wx_acc ? ly.Wx_acc + o : nullptr; vel = ly.Wx_vel ? ly.Wx_vel + o : nullptr; ast = (size_t)L * ly.ld3; }
    const float g4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int u = 0; u < 4; u++) dense_update(md, p + u, acc ? acc + u : nullptr, vel ? vel + u : nullptr, g4[u], ast);
  }
}
// sum of the K splits written to global memory (fixed order) + fused epilogue; consecutive threads on consecutive column quads
template <int EPI>
__global__ void __launch_bounds__(256) k_ts_epi(int slot, const int* base, int off, TsGemm g, TsBuf tb) {
  const ModelDev& md = MD; const int s = STEP_IDX;
  const int M = md.wM[s];
  const int N = M + (md.wSti[s] >= 0 ? md.S : 0);
  int m_lim, n_lim;
  ts_limits<EPI>(md, tb, M, N, m_lim, n_lim);
  const int n4 = n_lim >> 2;
  const size_t ps = (size_t)g.m_tiles * TS_RB * g.ldP;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)m_lim * n4; i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / n4), n = (int)(i % n4) * 4;
    if (!ts_tile_live<EPI>(md, tb, M, N, m / TS_RB * TS_RB, n / g.NT * g.NT)) continue;      // that tile was never computed
    const float* p = g.P + (size_t)m * g.ldP + n;
    float4 v = ld4(p);
    for (int k = 1; k < g.ksplit; k++) { const float4 w = ld4(p + k * ps); v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w; }
    ts_epilogue4<EPI>(md, tb, s, m, n, v);
  }
}

constexpr uint32_t TS_SMEM_OPER = 192 * 1024;
struct TsSmem {
  alignas(1024) unsigned char stage[TS_SMEM_OPER];
  alignas(8) unsigned long long stage_full[4];
  unsigned long long stage_free[4];
  int err;
};
__device__ __forceinline__ void ts_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

#define TS_STAMP(i) do { if (g.dbg) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); g.dbg[(size_t)blockIdx.x * 16 + (i)] = t_; } } while (0)
// main loop of one CTA: its K slice of the 128 x NT tile, warpgroup wg accumulating rows (wg & 1) * 64 .. + 63 x columns
// (wg >> 1) * NT / 2 .. in registers (NR = NT / 4 floats per thread); thread 0 also issues the bulk copies of the stage ring.
// On return the stages are free and the partial tile is in sT [128 x (NT + 4)] (row-major, in the stage memory).
template <int NR>
__device__ __forceinline__ void ts_mainloop(TsSmem& sm, const TsGemm& g, int mt, int nt, int c_beg, int c_end, float* sT) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int NT = 4 * NR;
  const int nb = NT / TS_RB;                                  // 128-row operand blocks per N tile
  const uint32_t b_bytes = (uint32_t)NT * TC_KC * 4;          // one hi (or lo) slab of the N tile
  const uint32_t stage_bytes = 2 * TS_BLK + 2 * b_bytes;      // 64 KB (NT = 128, 3 stages) or 96 KB (NT = 256, 2 stages)
  const uint32_t n_stage = TS_SMEM_OPER / stage_bytes;
  const unsigned int total = c_end > c_beg ? (unsigned int)(c_end - c_beg) : 0u;
  auto issue = [&](unsigned int it) {
    const int c = c_beg + (int)it;
    unsigned char* dst = sm.stage + (it % n_stage) * stage_bytes;
    unsigned long long* bar = &sm.stage_full[it % n_stage];
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(tc_smem_u32(bar)), "r"(stage_bytes) : "memory");
    tc_bulk_copy(dst, g.A + ((size_t)mt * g.chunks + c) * 2 * TS_BLK, 2 * TS_BLK, bar);
    for (int q = 0; q < nb; q++) {                  // smem: [hi of all blocks | lo of all blocks]
      const unsigned char* bsrc = g.Bm + ((size_t)(nt * nb + q) * g.chunks + c) * 2 * TS_BLK;
      tc_bulk_copy(dst + 2 * TS_BLK + q * TS_BLK, bsrc, TS_BLK, bar);
      tc_bulk_copy(dst + 2 * TS_BLK + b_bytes + q * TS_BLK, bsrc + TS_BLK, TS_BLK, bar);
    }
  };
  if (tid == 0) { for (unsigned int it = 0; it < total && it < n_stage; it++) issue(it); TS_STAMP(2); }
  __syncwarp();
  const int wr = (wg & 1) * 64, wc = (wg >> 1) * (NT / 2);
  float d[NR];
#pragma unroll
  for (int i = 0; i < NR; i++) d[i] = 0.f;                    // a K split without chunks contributes zeros
  for (unsigned int it = 0; it < total; it++) {
    const uint32_t st = it % n_stage, use = it / n_stage;
    tc_mbar_wait(&sm.stage_full[st], use & 1u, &sm.err);
    if (it == 0 && tid == 0) TS_STAMP(3);
    const uint32_t a_hi = tc_smem_u32(sm.stage + st * stage_bytes) + wr * 128, a_lo = a_hi + TS_BLK;
    const uint32_t b_hi = tc_smem_u32(sm.stage + st * stage_bytes) + 2 * TS_BLK + wc * 128, b_lo = b_hi + b_bytes;
    wg_chunk_3xtf32(d, a_hi, a_lo, b_hi, b_lo);
    if ((tid & 127) == 0) tc_mbar_arrive(&sm.stage_free[st]);
    if (tid == 0 && it + n_stage < total) { tc_mbar_wait(&sm.stage_free[st], use & 1u, &sm.err); issue(it + n_stage); }
    __syncwarp();
  }
  if (tid == 0) TS_STAMP(4);
  __syncthreads();                                            // every warpgroup is done with the stages: they become sT
  const int ldt = NT + 4;
  const int r0 = wr + (warp & 3) * 16 + (lane >> 2), cq = wc + 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < NR; i += 2)
    *reinterpret_cast<float2*>(sT + (size_t)(r0 + 8 * ((i >> 1) & 1)) * ldt + cq + (i >> 2) * 8) = make_float2(d[i], d[i + 1]);
}
template <int EPI>
__global__ void __launch_bounds__(TS_THREADS, 1) k_ts_gemm(int slot, const int* base, int off, TsGemm g, TsBuf tb) {
  extern __shared__ __align__(1024) unsigned char ts_raw[];
  TsSmem& sm = *reinterpret_cast<TsSmem*>(ts_raw);
  const ModelDev& md = MD; const int s = STEP_IDX;
  const int tid = threadIdx.x;
  const int M = md.wM[s];
  const int N = M + (md.wSti[s] >= 0 ? md.S : 0);
  // the cluster = the K splits of one tile (consecutive blocks): all of them take the same early exit
  const int ks = blockIdx.x % g.ksplit, nt = (blockIdx.x / g.ksplit) % g.n_tiles, mt = blockIdx.x / (g.ksplit * g.n_tiles);
  const int m0 = mt * TS_RB, n0 = nt * g.NT;
  if (tid == 0) TS_STAMP(0);
  if (!ts_tile_live<EPI>(md, tb, M, N, m0, n0)) { pdl_wait(); return; }     // dynamic batch size / column count; unused blocks of the dense-gradient products
  const int cps = (g.chunks + g.ksplit - 1) / g.ksplit;
  const int c_beg = ks * cps, c_end = min(g.chunks, c_beg + cps);
  if (tid == 0) {
    for (int i = 0; i < 4; i++) { tc_mbar_init(&sm.stage_free[i], 4); tc_mbar_init(&sm.stage_full[i], 1); }
    sm.err = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) TS_STAMP(1);
  pdl_wait();               // everything above overlapped the previous kernel of the stream; its results are visible from here on
  pdl_trigger();
  if (EPI == TS_EPI_DH && blockIdx.x == 0 && tid == 0) {    // cost of the step = loss / batch_size (gru4rec.py:577); the row losses are final
    float c = 0.f;
    for (int bb = 0; bb < M; bb++) c += md.RS[(size_t)bb * G4R_NSTAT + 6];
    c = __fdiv_rn(c, (float)md.B);
    md.cost[s] = c;
    if (c != c) atomicExch(md.nanflag, 1);
  }
  // split K through global memory (L2): the register tiles are transposed through shared memory (the operand stages are free once
  // the accumulation is complete) and all warps store the tile as whole 512-byte row pieces
  {
    float* sT = reinterpret_cast<float*>(sm.stage);
    if (g.NT == 256) ts_mainloop<64>(sm, g, mt, nt, c_beg, c_end, sT); else ts_mainloop<32>(sm, g, mt, nt, c_beg, c_end, sT);
    __syncthreads();
    if (tid == 0) TS_STAMP(6);
    const int ldt = g.NT + 4, q4 = g.NT / 4;
    float* ptile = g.P + ((size_t)ks * g.m_tiles * TS_RB + m0) * g.ldP + n0;
    for (int idx = tid; idx < TS_RB * q4; idx += TS_THREADS) {
      const int row = idx / q4, c = (idx % q4) * 4;
      *reinterpret_cast<float4*>(ptile + (size_t)row * g.ldP + c) = *reinterpret_cast<const float4*>(sT + (size_t)row * ldt + c);
    }
  }
  if (g.fused) {
    // the K splits of a tile are the CTAs of one cluster (co-resident): after the cluster barrier (release / acquire) CTA `ks` adds
    // the splits of its band of rows in K order -- the same sum whatever the schedule -- and applies the epilogue, consecutive
    // threads on consecutive column quads
    __threadfence();
    ts_cluster_sync();
    if (tid == 0) TS_STAMP(7);
    int m_lim, n_lim;
    ts_limits<EPI>(md, tb, M, N, m_lim, n_lim);
    const int rpc = TS_RB / g.ksplit, q4 = g.NT / 4, total = rpc * q4;
    const size_t ps = (size_t)g.m_tiles * TS_RB * g.ldP;
    for (int i0 = tid; i0 < total; i0 += TS_THREADS * 4) {       // four quads per thread at a time: all their loads are in flight together
      float4 acc[4]; int mm[4], nn[4]; bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int idx = i0 + u * TS_THREADS;
        mm[u] = m0 + ks * rpc + idx / q4; nn[u] = n0 + (idx % q4) * 4;
        ok[u] = idx < total && mm[u] < m_lim && nn[u] < n_lim;
        acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      for (int k = 0; k < g.ksplit; k++) {
#pragma unroll
        for (int u = 0; u < 4; u++) if (ok[u]) {
          const float4 w = __ldcg(reinterpret_cast<const float4*>(g.P + k * ps + (size_t)mm[u] * g.ldP + nn[u]));
          if (k == 0) acc[u] = w; else { acc[u].x += w.x; acc[u].y += w.y; acc[u].z += w.z; acc[u].w += w.w; }
        }
      }
#pragma unroll
      for (int u = 0; u < 4; u++) if (ok[u]) ts_epilogue4<EPI>(md, tb, s, mm[u], nn[u], acc[u]);
    }
    if (tid == 0) TS_STAMP(8);
  }
}
