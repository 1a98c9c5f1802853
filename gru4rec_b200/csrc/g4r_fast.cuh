// g4r_fast.cuh -- role-specialised persistent kernel for the headline shape family:
//   no-embedding mode, one GRU layer, L <= 120 (step_mode 3: L <= 128), batch <= 32, every score-column chunk <= 32 columns.
// (step_mode 2; anything else runs k_persistent / the per-phase kernels, which share all numerics.)
//
// Why: at B=32, L=100 a mini-batch is ~8 dependent phases over ~6 MB; time is memory/barrier latency.  This kernel
//  * gives each "column CTA" one chunk of score columns (step_mode 2: the CTAs after the G GRU CTAs, chunk c on CTA G + c;
//    step_mode 3: every CTA, chunk c on CTA c); the chunk's Wy / Adagrad / momentum rows and the target rows are
//    PREFETCHED with TMA bulk copies (cp.async.bulk -> mbarrier complete_tx) while the GRU phases of the previous step
//    run, so the score phase starts with its operands already in shared memory;
//  * combines the row statistics of lane b on column CTA b right after the score->gradient barrier;
//  * (step_mode 2) puts only the partial dL/dh before the b1 barrier: dSy and the update of the chunk's rows follow b1, gated for
//    the next prefetch by `rows_done`; the GRU CTAs take no part in the column phases, so none of this is on their chain;
//  * runs the GRU phases on a group of G CTAs (step_mode 2: weights resident in shared memory, one group barrier per
//    mini-batch; see FastSmemR); the other CTAs only wait for `h_ready`;
//  * uses monotonic release/acquire counters (no resets, no separate fences) for all synchronisation.
//
// What is computed (reference hidasib/GRU4Rec, same formulas as the generic phases in g4r_kernels.cuh):
//   F1 / F2   GRU layer in no-embedding mode, gru4rec.py:459-466 (vec = Wx0[X] + Bh, column blocks h~ | r | z, :460-462),
//             hidden dropout and the reset of finished sessions (:464-466)
//   scores    o = h Sy^T + by (- logq log P), gru4rec.py:480-496; final activations :189-223
//   stats     row statistics of the losses, gru4rec.py:225-248 (softmax_neg with the zeroed diagonal :199-203)
//   lossgrad  dL/do of SURVEY appendix A (the reference differentiates symbolically, :383-384), dSy, dby, partial dL/dh
//   update    sparse Adagrad (+momentum) with the duplicate rules of gru4rec.py:335-340,407-431 on the chunk's rows,
//             dense Adagrad (+momentum) of Wh / Wrz / Bh, :330-334,390-406, input rows Wx0[X] :407-431
#pragma once

constexpr int FK_THREADS = 512;
constexpr int FK_NW = FK_THREADS / 32;   // warps per CTA
constexpr int FK_G = 48;            // CTAs that run the GRU phases
constexpr int FK_CT = 32;           // max columns per chunk
constexpr int FK_Q = FK_CT / FK_NW;  // columns per warp
constexpr int FK_B = 32;            // max lanes
static_assert(FK_THREADS / 16 == FK_B, "statistics mapping: 16 threads per lane");
constexpr int FK_LDS = 132;         // shared row stride (floats) for L <= 128: conflict-free 16-byte accesses


__device__ __forceinline__ void red_release_add(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int atom_acqrel_add(unsigned int* p, unsigned int v) {
  unsigned int old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ void wait_ge(const unsigned int* p, unsigned int target) {
  while (ld_acquire_u32(p) < target) { }
}
// ---- mbarrier + TMA bulk copy (1-D, no tensor map): rows of ld*4 bytes, 16-byte aligned ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned int bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned int parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni WAIT_DONE;\n\t"
      "bra.uni WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_row(void* sdst, const void* gsrc, unsigned int bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

struct FastSmem {
  // column role
  alignas(128) float sY[FK_B * FK_LDS];          // h of the step (all lanes)
  float sS[FK_CT * FK_LDS];         // Wy rows of the chunk (TMA)
  float sAcc[FK_CT * FK_LDS];       // Adagrad rows (TMA)
  float sVel[FK_CT * FK_LDS];       // momentum rows (TMA)
  float sTW[FK_B * FK_LDS];         // target rows (TMA; pairwise losses)
  float sD[FK_CT * FK_LDS];         // dSy rows
  float sG[FK_CT * FK_B];           // dL/do
  float sO[FK_CT * FK_B];           // scores o
  float sRS[FK_B * 8];
  float sPart[FK_NW * FK_B * 8];
  float sT[FK_B];                   // target activations
  float sBias[FK_CT], sByP[FK_CT], sByA[FK_CT], sByV[FK_CT], sDby[FK_CT], sTB[FK_B];
  int sIt[2][FK_CT], sPos[2][FK_CT], sTc[2][FK_B], sYit[2][FK_B], sCb[2][2];
  int sFlag[4];
  alignas(8) unsigned long long mbar;
  // GRU role: thin-slab phases (every GRU CTA owns a few output columns / rows and stages the full 32-lane operand)
  alignas(16) float gA[FK_B * 388];             // staged [32 x <=384] operand (H, Hold*r, da_h, dvec)
  alignas(16) float gW[8 * FK_LDS + FK_NW * FK_B * 5 + 16 * FK_B];      // this CTA's weight slab (<= 8 columns/rows of length <= 128) + reduction scratch
  int gIdx[3 * FK_B];               // slot, item, flags of the lanes
};

// loads the index metadata of step s into buffer `buf` (plain loads; consumed much later)
template <class SM>
__device__ __forceinline__ void fk_load_idx(const ModelDev& md, SM& sm, int s, int n_steps, int chunk, int buf) {
  const int tid = threadIdx.x;
  if (s >= n_steps) return;
  const int M = md.wM[s];
  const int* cbeg = md.pCbeg + (size_t)s * (md.NCH + 1);
  const bool hc = chunk < md.NCH;
  const int cb = hc ? cbeg[chunk] : 0, ce = hc ? cbeg[chunk + 1] : 0;
  if (tid < FK_CT) {
    int it = 0, pos = 0;
    if (cb + tid < ce) { it = md.pItem[(size_t)s * md.NP + cb + tid]; pos = md.pPos[(size_t)s * md.NP + cb + tid]; }
    sm.sIt[buf][tid] = it; sm.sPos[buf][tid] = pos;
  }
  if (tid >= 32 && tid < 32 + FK_B) {
    const int b = tid - 32;
    sm.sTc[buf][b] = b < M ? md.pTcol[(size_t)s * md.B + b] : -1;
    sm.sYit[buf][b] = b < M ? md.wY[(size_t)s * md.B + b] : 0;
  }
  if (tid == 64) { sm.sCb[buf][0] = cb; sm.sCb[buf][1] = ce; }
}

// issue the TMA prefetch of step s (rows are final once the previous step's updates are complete)
template <class SM>
__device__ __forceinline__ void fk_prefetch_rows(const ModelDev& md, SM& sm, int s, int n_steps, int buf, bool pw) {
  if (s >= n_steps) return;
  const int tid = threadIdx.x;
  const int M = md.wM[s];
  const int cb = sm.sCb[buf][0], ce = sm.sCb[buf][1];
  const int nj = ce - cb;
  const bool ada = md.adapt == G4R_ADAPT_ADAGRAD, mom = md.mom > 0.f;
  const unsigned int rowb = (unsigned int)md.ldL * 4u;
  uint64_t* bar = reinterpret_cast<uint64_t*>(&sm.mbar);
  // bulk copies are issued one per thread-instruction; spreading them over the warps (lane 0 of each) keeps the issue
  // off the critical path (one warp issuing ~80 copies took 2.3 us)
  const int ntab = 1 + (ada ? 1 : 0) + (mom ? 1 : 0);
  const int ncopy = nj * ntab + (pw ? M : 0);
  if (tid == 0) {
    const unsigned int total = rowb * (unsigned int)ncopy;
    if (total > 0) mbar_expect_tx(bar, total);
    else asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
  }
  if ((tid & 31) == 0) {
    // every issuing thread orders the rows' generic-proxy stores (other CTAs' after the caller's acquire, this CTA's after
    // its __syncthreads) before its bulk copies
    asm volatile("fence.proxy.async.global;" ::: "memory");
    for (int i = tid >> 5; i < ncopy; i += FK_NW) {
      if (i < nj * ntab) {
        const int j = i / ntab, t = i % ntab;
        const size_t off = (size_t)sm.sIt[buf][j] * md.ldL;
        if (t == 0) tma_row(sm.sS + j * FK_LDS, md.Wy + off, rowb, bar);
        else if (t == 1 && ada) tma_row(sm.sAcc + j * FK_LDS, md.Wy_acc + off, rowb, bar);
        else tma_row(sm.sVel + j * FK_LDS, md.Wy_vel + off, rowb, bar);
      } else {
        const int b = i - nj * ntab;
        tma_row(sm.sTW + b * FK_LDS, md.Wy + (size_t)sm.sYit[buf][b] * md.ldL, rowb, bar);
      }
    }
  }
  if (false) {
  } else if (tid >= 64 && tid < 64 + FK_CT) {
    const int j = tid - 64;
    if (j < nj) {
      const int it = sm.sIt[buf][j];
      float bz = md.By[it];
      sm.sByP[j] = bz;
      if (md.logq > 0.f) bz -= (sm.sPos[buf][j] < M) ? md.logP0t[it] : md.logP0s[it];
      sm.sBias[j] = bz;
      sm.sByA[j] = ada ? md.By_acc[it] : 0.f;
      sm.sByV[j] = mom ? md.By_vel[it] : 0.f;
    }
  } else if (tid >= 96 && tid < 96 + FK_B) {
    const int b = tid - 96;
    if (pw && b < M) {
      const int it = sm.sYit[buf][b];
      float bz = md.By[it];
      if (md.logq > 0.f) bz -= md.logP0t[it];
      sm.sTB[b] = bz;
    }
  }
}

__device__ __forceinline__ void fk_group_barrier(FastSync* fs, unsigned int& gepoch, unsigned int G = FK_G) {
  __syncthreads();
  gepoch += 1;
  if (threadIdx.x == 0) { red_release_add(&fs->grp, 1u); wait_ge(&fs->grp, gepoch * G); }
  __syncthreads();
}

// ---------------- thin-slab GRU phases (no-embedding mode, one layer, M <= 32, L <= 128) ----------------
// ncu on the 32x32-tile kernels showed ~2000 instructions per warp at ~8.6 cycles each (2 warps per scheduler):
// the GRU phases are instruction-latency bound.  Here the work of a phase is spread over all FK_G CTAs (a few
// output columns each), the reduction dimension is split over the 8 warps, and every thread issues a few dozen FMAs.
template <class SM>
__device__ __forceinline__ void fk_stage_lanes(const ModelDev& md, SM& sm, int s, int M) {
  if (threadIdx.x < FK_B) {
    const int b = threadIdx.x;
    sm.gIdx[b] = b < M ? md.wSlot[(size_t)s * md.B + b] : -1;
    sm.gIdx[FK_B + b] = b < M ? md.wX[(size_t)s * md.B + b] : 0;
    sm.gIdx[2 * FK_B + b] = b < M ? md.wF[(size_t)s * md.B + b] : 0;
  }
  __syncthreads();
}
// acc[j] (j < W) for lane b = tid % 32 over the k-slice of warp tid / 32: sum_k A[b][k] * Wt[j][k]
template <int W>
__device__ __forceinline__ void fk_slab_dot(float (&acc)[W], const float* sAop, int lda, const float* sWt, int K) {
  const int b = threadIdx.x & 31, ks = threadIdx.x >> 5;
  const int kq = (K + 3) / 4;                      // float4 count along k
  const int per = (kq + FK_NW - 1) / FK_NW;
  const int q0 = ks * per, q1 = min(kq, q0 + per);
#pragma unroll
  for (int j = 0; j < W; j++) acc[j] = 0.f;
  for (int q = q0; q < q1; q++) {
    const float4 a = ld4(sAop + b * lda + q * 4);
#pragma unroll
    for (int j = 0; j < W; j++) {
      const float4 w = ld4(sWt + j * FK_LDS + q * 4);
      acc[j] = fmaf(a.x, w.x, acc[j]); acc[j] = fmaf(a.y, w.y, acc[j]); acc[j] = fmaf(a.z, w.z, acc[j]); acc[j] = fmaf(a.w, w.w, acc[j]);
    }
  }
}
// cross-warp reduction of acc[W] per lane: red[ks][b][j] -> thread (b, j) sums the 8 slices in fixed order
template <int W>
__device__ __forceinline__ float fk_slab_reduce(const float (&acc)[W], float* red, int jsel) {
  const int b = threadIdx.x & 31, ks = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < W; j++) red[(ks * FK_B + b) * W + j] = acc[j];
  __syncthreads();
  float v = 0.f;
  if (jsel < W) {
#pragma unroll
    for (int k = 0; k < FK_NW; k++) v += red[(k * FK_B + b) * W + jsel];
  }
  return v;
}
constexpr int FK_W1 = 5;    // rz columns per CTA   (ceil(2*128 / 48) = 6 would also fit; 2L <= 240 with 48 CTAs)
constexpr int FK_W2 = 3;    // h / dHr columns per CTA (L <= 144)

// F1: rz = sigmoid(Wx0[X][L:3L] + Bh[L:3L] + H @ Wrz) for this CTA's FK_W1 columns; CTA 0 also writes Hold
// inrows != nullptr (row-sharded multi-GPU): the gathered input rows Wx0[X] of the step sit in a local [B x ld3] buffer
__device__ void fk_f1(const ModelDev& md, FastSmem& sm, int s, int cta, const unsigned int* wait_ctr, unsigned int wait_target, const float* inrows = nullptr) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL, tid = threadIdx.x;
  const int c0 = cta * FK_W1;
  if (c0 >= 2 * L) return;
  const int W = min(FK_W1, 2 * L - c0);
  fk_stage_lanes(md, sm, s, M);
  // if the helper CTAs' input-row updates are already complete (the usual case), the epilogue operand is fetched before the
  // product instead of after it
  if (tid == 0) sm.sFlag[3] = (!wait_ctr || ld_acquire_u32(wait_ctr) >= wait_target) ? 1 : 0;
  const int kw = ldL / 4;
  // stage H rows (zero for out-of-range lanes) and the transposed weight slab Wt[j][k] = Wrz[k][c0 + j]
  stage_rows4(sm.gA, FK_LDS, FK_B, kw, [&](int rr) -> const float* { const int sl = sm.gIdx[rr]; return sl >= 0 ? ly.H + (size_t)sl * ldL : nullptr; });
  for (int i = tid; i < FK_W1 * FK_LDS; i += FK_THREADS) {
    const int j = i / FK_LDS, k = i % FK_LDS;
    sm.gW[i] = (j < W && k < L) ? ly.Wrz[(size_t)k * ly.ld2 + c0 + j] : 0.f;
  }
  const int b = tid & 31, jsel = tid >> 5;
  __syncthreads();
  const bool early = sm.sFlag[3] != 0;
  float pre = 0.f;
  if (early && jsel < W && b < M) pre = (inrows ? inrows[(size_t)b * ly.ld3 + L + c0 + jsel] : ly.Wx[(size_t)sm.gIdx[FK_B + b] * ly.ld3 + L + c0 + jsel]) + ly.Bh[L + c0 + jsel];
  float acc[FK_W1];
  fk_slab_dot<FK_W1>(acc, sm.gA, FK_LDS, sm.gW, L);
  const float v = fk_slab_reduce<FK_W1>(acc, sm.gW + 8 * FK_LDS, jsel);
  // otherwise the gathered input rows are still in flight on the helper CTAs (previous step's update): wait now, after
  // the H @ Wrz part, then fetch the epilogue operands (gathered row element + bias)
  if (!early) {
    if (tid == 0) wait_ge(wait_ctr, wait_target);
    __syncthreads();
    if (jsel < W && b < M) pre = (inrows ? inrows[(size_t)b * ly.ld3 + L + c0 + jsel] : ly.Wx[(size_t)sm.gIdx[FK_B + b] * ly.ld3 + L + c0 + jsel]) + ly.Bh[L + c0 + jsel];
  }
  if (jsel < W && b < M) {
    const int c = c0 + jsel;
    const float g = sigmoidf_(v + pre);
    if (c < L) ly.r[(size_t)b * ldL + c] = g; else ly.z[(size_t)b * ldL + (c - L)] = g;
  }
  if (cta == 0) {
    for (int i = tid; i < FK_B * kw; i += FK_THREADS) {
      const int rr = i / kw, c4 = i % kw;
      if (rr < M) st4(ly.Hold + (size_t)rr * ldL + c4 * 4, ld4(sm.gA + rr * FK_LDS + c4 * 4));
    }
  }
}
// F2: h~ = act(Wx0[X][0:L] + Bh[0:L] + (H*r) @ Wh), h, dropout, H_new for this CTA's FK_W2 columns
__device__ void fk_f2(const ModelDev& md, FastSmem& sm, int s, int cta, const float* inrows = nullptr) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL, tid = threadIdx.x;
  const int c0 = cta * FK_W2;
  if (c0 >= L) return;
  const int W = min(FK_W2, L - c0);
  fk_stage_lanes(md, sm, s, M);
  const int kw = ldL / 4;
  // stage H*r
  for (int i0 = 0; i0 < FK_B * kw; i0 += 2 * FK_THREADS) {
    float4 hv[2], rv[2];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int i = i0 + u * FK_THREADS + tid;
      hv[u] = make_float4(0.f, 0.f, 0.f, 0.f); rv[u] = hv[u];
      if (i < FK_B * kw) {
        const int rr = i / kw, c4 = i % kw;   // Hold (compact copy written by CTA 0 in F1): H itself is being overwritten
        if (rr < M) { hv[u] = ld4(ly.Hold + (size_t)rr * ldL + c4 * 4); rv[u] = ld4(ly.r + (size_t)rr * ldL + c4 * 4); }
      }
    }
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int i = i0 + u * FK_THREADS + tid;
      if (i < FK_B * kw) st4(sm.gA + (i / kw) * FK_LDS + (i % kw) * 4, make_float4(hv[u].x * rv[u].x, hv[u].y * rv[u].y, hv[u].z * rv[u].z, hv[u].w * rv[u].w));
    }
  }
  for (int i = tid; i < FK_W2 * FK_LDS; i += FK_THREADS) {
    const int j = i / FK_LDS, k = i % FK_LDS;
    sm.gW[i] = (j < W && k < L) ? ly.Wh[(size_t)k * ldL + c0 + j] : 0.f;
  }
  const int b = tid & 31, jsel = tid >> 5;
  float pre = 0.f, z = 0.f, ho = 0.f;
  if (jsel < W && b < M) {
    const int c = c0 + jsel;
    pre = (inrows ? inrows[(size_t)b * ly.ld3 + c] : ly.Wx[(size_t)sm.gIdx[FK_B + b] * ly.ld3 + c]) + ly.Bh[c];
    z = ly.z[(size_t)b * ldL + c];
    ho = ly.Hold[(size_t)b * ldL + c];
  }
  __syncthreads();
  float acc[FK_W2];
  fk_slab_dot<FK_W2>(acc, sm.gA, FK_LDS, sm.gW, L);
  const float v0 = fk_slab_reduce<FK_W2>(acc, sm.gW + 8 * FK_LDS, jsel);
  if (jsel < W && b < M) {
    const int c = c0 + jsel;
    const float v = v0 + pre;
    const float ht = act_fwd(md.hact, v);
    float h = (1.0f - z) * ho + z * ht;
    if (md.p_drop_h > 0.f) h *= drop_scale(md.drop_seed, md.wG[s], 0u, (uint32_t)(b * L + c), 1.0f - md.p_drop_h);
    ly.ah[(size_t)b * ldL + c] = v;
    ly.ht[(size_t)b * ldL + c] = ht;
    ly.y[(size_t)b * ldL + c] = h;
    ly.H[(size_t)sm.gIdx[b] * ldL + c] = (sm.gIdx[2 * FK_B + b] & 1) ? 0.f : h;
  }
}
// B2: d(H*r)[b][c] = sum_j da_h[b][j] Wh[c][j]; da_r = d(H*r) * Hold * r (1-r) for this CTA's FK_W2 columns
__device__ void fk_b2(const ModelDev& md, FastSmem& sm, int s, int cta) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL, tid = threadIdx.x;
  const int c0 = cta * FK_W2;
  if (c0 >= L) return;
  const int W = min(FK_W2, L - c0);
  const int kw = ldL / 4;
  __syncthreads();
  stage_rows4(sm.gA, FK_LDS, FK_B, kw, [&](int rr) -> const float* { return rr < M ? ly.dvec + (size_t)rr * ly.ld3 : nullptr; });
  stage_rows4(sm.gW, FK_LDS, W, kw, [&](int rr) -> const float* { return ly.Wh + (size_t)(c0 + rr) * ldL; });
  const int b = tid & 31, jsel = tid >> 5;
  float ho = 0.f, r = 0.f;
  if (jsel < W && b < M) { ho = ly.Hold[(size_t)b * ldL + c0 + jsel]; r = ly.r[(size_t)b * ldL + c0 + jsel]; }
  __syncthreads();
  float acc[FK_W2];
  fk_slab_dot<FK_W2>(acc, sm.gA, FK_LDS, sm.gW, L);
  const float v = fk_slab_reduce<FK_W2>(acc, sm.gW + 8 * FK_LDS, jsel);
  if (jsel < W && b < M) ly.dvec[(size_t)b * ly.ld3 + L + c0 + jsel] = v * ho * r * (1.f - r);
}
// Input-row update of lane b on a helper (non-GRU) CTA, concurrent with the dense update of the GRU group: it starts when
// the GRU group has passed its B2 barrier (dvec complete) and only touches Wx0 rows, which the dense phase never reads.
template <class SM>
__device__ void fk_sparse_in(const ModelDev& md, SM& sm, int s, int b) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s];
  if (b >= M) return;
  const uint8_t xf = md.wXflag[(size_t)s * md.B + b];
  if (!(xf & 1)) return;                                // not the first position of its duplicate group
  const int ld3 = ly.ld3, tid = threadIdx.x;
  const int item = md.wX[(size_t)s * md.B + b];
  const int* xnext = md.wXnext + (size_t)s * md.B;
  if (tid == 0) { int n = 0; for (int bb = b; bb >= 0 && n < FK_B; bb = xnext[bb]) sm.gIdx[n++] = bb; sm.gIdx[FK_B] = n; }
  __syncthreads();
  const int nmem = sm.gIdx[FK_B];
  const bool ada = md.adapt == G4R_ADAPT_ADAGRAD, mom = md.mom > 0.f;
  float* prow = ly.Wx + (size_t)item * ld3;
  for (int c4 = tid; c4 < ld3 / 4; c4 += FK_THREADS) {
    const float4 p0 = ld4(prow + c4 * 4), z = make_float4(0.f, 0.f, 0.f, 0.f);
    RowChain<float4> u;
    u.begin(p0, p0, ada ? ld4(ly.Wx_acc + (size_t)item * ld3 + c4 * 4) : z, mom ? ld4(ly.Wx_vel + (size_t)item * ld3 + c4 * 4) : z);
    for (int k = 0; k < nmem; k++) u.add(md, ld4(ly.dvec + (size_t)sm.gIdx[k] * ld3 + c4 * 4), ada, mom);
    st4(prow + c4 * 4, u.ps);
    if (ada) st4(ly.Wx_acc + (size_t)item * ld3 + c4 * 4, u.al);
    if (mom) st4(ly.Wx_vel + (size_t)item * ld3 + c4 * 4, u.vl);
  }
}

// Same update when the CTA owns exactly one lane: everything that does not depend on this step's gradients (duplicate
// chain, parameter / Adagrad / momentum row) is fetched BEFORE waiting for the dvec rows, so that only one load round trip
// separates the GRU role's "dvec complete" signal from the row update.
template <class SM>
__device__ void fk_sparse_in_one(const ModelDev& md, SM& sm, int s, int b, const unsigned int* ctr, unsigned int target) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], ld3 = ly.ld3, tid = threadIdx.x;
  const bool act = b < M && (md.wXflag[(size_t)s * md.B + b] & 1);       // first position of its duplicate group
  const int item = act ? md.wX[(size_t)s * md.B + b] : 0;
  const bool ada = md.adapt == G4R_ADAPT_ADAGRAD, mom = md.mom > 0.f;
  if (act && tid == 0) {
    const int* xnext = md.wXnext + (size_t)s * md.B;
    int n = 0; for (int bb = b; bb >= 0 && n < FK_B; bb = xnext[bb]) sm.gIdx[n++] = bb; sm.gIdx[FK_B] = n;
  }
  float* prow = ly.Wx + (size_t)item * ld3;
  const int c4 = tid;
  const bool mine = act && c4 < ld3 / 4;                                   // ld3 / 4 <= 96 quads: one pass
  float4 p0 = make_float4(0.f, 0.f, 0.f, 0.f), a0 = p0, v0 = p0;
  if (mine) {
    p0 = ld4(prow + c4 * 4);
    if (ada) a0 = ld4(ly.Wx_acc + (size_t)item * ld3 + c4 * 4);
    if (mom) v0 = ld4(ly.Wx_vel + (size_t)item * ld3 + c4 * 4);
  }
  if (tid == 0) wait_ge(ctr, target);
  __syncthreads();
  if (mine) {
    const int nmem = sm.gIdx[FK_B];
    RowChain<float4> u;
    u.begin(p0, p0, a0, v0);
    for (int k = 0; k < nmem; k++) u.add(md, ld4(ly.dvec + (size_t)sm.gIdx[k] * ld3 + c4 * 4), ada, mom);
    st4(prow + c4 * 4, u.ps);
    if (ada) st4(ly.Wx_acc + (size_t)item * ld3 + c4 * 4, u.al);
    if (mom) st4(ly.Wx_vel + (size_t)item * ld3 + c4 * 4, u.vl);
  }
}

// B1 (fast kernel): every column CTA (cta of ncta) reduces a contiguous run of dL/dh elements; lanes = consecutive elements (coalesced),
// warps = slices of the chunk partials, cross-warp sum in shared memory in fixed order; then da_h / da_z.
template <bool CL, class SM>
__device__ void fk_b1(const ModelDev& md, SM& sm, int s, int cta, int ncta) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int E = M * ldL;                                  // padded elements (padding columns are zero everywhere)
  const int per = ((E + ncta - 1) / ncta + 31) / 32 * 32; // elements per CTA, multiple of 32
  const int e0 = cta * per;
  float* red = sm.sPart;                                  // [FK_NW][per]  (per <= 256: M * ldL <= 4096 elements over >= 16 CTAs)
  const size_t cs = (size_t)md.B * ldL;
  // forward saves of this thread's output element (per <= 128 <= FK_THREADS: at most one element per thread), fetched up
  // front so that their round trip overlaps the loads of the chunk partials
  float pht = 0.f, pho = 0.f, pz = 0.f, pah = 0.f;
  if (!CL && tid < per && e0 + tid < E && (e0 + tid) % ldL < L) {
    const size_t o = (size_t)((e0 + tid) / ldL) * ldL + (e0 + tid) % ldL;
    pht = ly.ht[o]; pho = ly.Hold[o]; pz = ly.z[o]; pah = ly.ah[o];
  }
  for (int eb = 0; eb < per; eb += 32) {
    const int e = e0 + eb + lane;
    float d = 0.f;
    if (e < E) {
      float v[10];
#pragma unroll
      for (int u = 0; u < 10; u++) { const int ch = warp + FK_NW * u; v[u] = ch < md.NCH ? md.part[(size_t)ch * cs + e] : 0.f; }
      d = (((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]))) + (v[8] + v[9]);
    }
    red[warp * per + eb + lane] = d;
  }
  __syncthreads();
  for (int i = tid; i < per; i += FK_THREADS) {
    const int e = e0 + i;
    if (e >= E) continue;
    const int b = e / ldL, c = e % ldL;
    if (c >= L) continue;
    float dy = 0.f;
#pragma unroll
    for (int w = 0; w < FK_NW; w++) dy += red[w * per + i];
    const size_t o = (size_t)b * ldL + c;
    if (CL) { ly.dy[o] = dy; continue; }     // cluster variant: the GRU cluster owns ht / z / ah and derives da_h, da_z itself
    const float ht = pht, ho = pho, z = pz, ah = pah;
    float dh = dy;
    if (md.p_drop_h > 0.f) dh *= drop_scale(md.drop_seed, md.wG[s], 0u, (uint32_t)(b * L + c), 1.0f - md.p_drop_h);
    const float dz = dh * (ht - ho);
    const float dah = dh * z * act_der(md.hact, ah, ht);
    ly.dvec[(size_t)b * ly.ld3 + c] = dah;
    ly.dvec[(size_t)b * ly.ld3 + 2 * L + c] = dz * z * (1.f - z);
  }
}

// ---------------- GRU group of step_mode 2: resident weights, ownership by hidden unit ----------------
// GRU CTA g owns the four hidden units Kg = [4g, 4g + 4) (one 16-byte quad; the group has ldL / 4 <= 30 CTAs) and keeps,
// for the whole window, the columns Wh[:, Kg], Wrz[:, Kg], Wrz[:, L + Kg], the rows Wh[Kg, :] and Bh of its units with
// their Adagrad / momentum state in shared memory.  Every phase then needs only its own units or data every CTA already
// holds, except F2, which needs Hold * r over all units: one group barrier per mini-batch.  Each Wh element is held by
// two CTAs (row slab of the owner of its row, column slab of the owner of its column); both copies are updated from the
// same operands in the same order and stay bitwise identical, and only the column copies are written back.
constexpr int FR_U = 4;             // hidden units per GRU CTA

struct FastSmemR {
  // column role (same fields as FastSmem); during the GRU phases sD holds da_h and sPart is the reduction scratch
  alignas(128) float sY[FK_B * FK_LDS];
  float sS[FK_CT * FK_LDS];
  float sAcc[FK_CT * FK_LDS];
  float sVel[FK_CT * FK_LDS];
  float sTW[FK_B * FK_LDS];
  float sD[FK_CT * FK_LDS];
  float sG[FK_CT * FK_B];
  float sO[FK_CT * FK_B];
  float sRS[FK_B * 8];
  float sPart[FK_NW * FK_B * 8];
  float sT[FK_B];
  float sBias[FK_CT], sByP[FK_CT], sByA[FK_CT], sByV[FK_CT], sDby[FK_CT], sTB[FK_B];
  int sIt[2][FK_CT], sPos[2][FK_CT], sTc[2][FK_B], sYit[2][FK_B], sCb[2][2];
  int sFlag[4];
  alignas(8) unsigned long long mbar;
  int gIdx[3 * FK_B];                            // slot, item, flags of the lanes
  // GRU role
  alignas(16) float gH[2][FK_B * FK_LDS];        // H rows of the step's lanes (= Hold) | of the next step, by step parity
  float gHr[FK_B * FK_LDS];                      // Hold * r of the step, all units
  float rC[3][3 * FR_U * FK_LDS];                // value | Adagrad | momentum of the resident columns, rows over k: Wh[:, Kg] | Wrz[:, Kg] | Wrz[:, L + Kg]
  float rR[3][FR_U * FK_LDS];                    // value | Adagrad | momentum of the resident rows Wh[Kg, :]
  float rB[3][3 * FR_U];                         // value | Adagrad | momentum of Bh[Kg] | Bh[L + Kg] | Bh[2L + Kg]
  float gR[FK_B * FR_U], gZ[FK_B * FR_U], gDr[FK_B * FR_U], gDz[FK_B * FR_U];   // r, z, da_r, da_z of the own units, [lane][unit]
};
static_assert(sizeof(FastSmemR) <= 232448, "FastSmemR exceeds the 227 KB shared memory of one CTA");
static_assert(FK_NW * FK_B * 8 >= FK_NW * FK_B * 2 * FR_U, "sPart too small for the F1 reduction");

// resident slabs <-> global (once per window each)
__device__ void fr_load_resident(const ModelDev& md, FastSmemR& sm, int k0) {
  const LayerDev& ly = md.layer[0];
  const int L = ly.L, tid = threadIdx.x;
  for (int i = tid; i < 3 * FR_U * FK_LDS; i += FK_THREADS) {
    const int q = i / FK_LDS, k = i % FK_LDS, t = q / FR_U, c = k0 + q % FR_U;
    float p = 0.f, a = 0.f, v = 0.f;
    if (c < L && k < L) {
      const size_t o = t == 0 ? (size_t)k * ly.ldL + c : (size_t)k * ly.ld2 + (t == 2 ? L : 0) + c;
      const float* P = t == 0 ? ly.Wh : ly.Wrz;
      const float* A = t == 0 ? ly.Wh_acc : ly.Wrz_acc;
      const float* V = t == 0 ? ly.Wh_vel : ly.Wrz_vel;
      p = P[o]; if (A) a = A[o]; if (V) v = V[o];
    }
    sm.rC[0][i] = p; sm.rC[1][i] = a; sm.rC[2][i] = v;
  }
  for (int i = tid; i < FR_U * FK_LDS; i += FK_THREADS) {
    const int k = k0 + i / FK_LDS, c = i % FK_LDS;
    float p = 0.f, a = 0.f, v = 0.f;
    if (k < L && c < L) {
      const size_t o = (size_t)k * ly.ldL + c;
      p = ly.Wh[o]; if (ly.Wh_acc) a = ly.Wh_acc[o]; if (ly.Wh_vel) v = ly.Wh_vel[o];
    }
    sm.rR[0][i] = p; sm.rR[1][i] = a; sm.rR[2][i] = v;
  }
  if (tid < 3 * FR_U) {
    const int c = k0 + tid % FR_U;
    float p = 0.f, a = 0.f, v = 0.f;
    if (c < L) { const int o = (tid / FR_U) * L + c; p = ly.Bh[o]; if (ly.Bh_acc) a = ly.Bh_acc[o]; if (ly.Bh_vel) v = ly.Bh_vel[o]; }
    sm.rB[0][tid] = p; sm.rB[1][tid] = a; sm.rB[2][tid] = v;
  }
  __syncthreads();
}
__device__ void fr_store_resident(const ModelDev& md, FastSmemR& sm, int k0) {
  const LayerDev& ly = md.layer[0];
  const int L = ly.L, tid = threadIdx.x;
  __syncthreads();
  for (int i = tid; i < 3 * FR_U * FK_LDS; i += FK_THREADS) {
    const int q = i / FK_LDS, k = i % FK_LDS, t = q / FR_U, c = k0 + q % FR_U;
    if (c < L && k < L) {
      const size_t o = t == 0 ? (size_t)k * ly.ldL + c : (size_t)k * ly.ld2 + (t == 2 ? L : 0) + c;
      float* P = t == 0 ? ly.Wh : ly.Wrz;
      float* A = t == 0 ? ly.Wh_acc : ly.Wrz_acc;
      float* V = t == 0 ? ly.Wh_vel : ly.Wrz_vel;
      P[o] = sm.rC[0][i]; if (A) A[o] = sm.rC[1][i]; if (V) V[o] = sm.rC[2][i];
    }
  }
  if (tid < 3 * FR_U) {
    const int c = k0 + tid % FR_U;
    if (c < L) { const int o = (tid / FR_U) * L + c; ly.Bh[o] = sm.rB[0][tid]; if (ly.Bh_acc) ly.Bh_acc[o] = sm.rB[1][tid]; if (ly.Bh_vel) ly.Bh_vel[o] = sm.rB[2][tid]; }
  }
}

// F1 of step s: r, z of the own units from the staged H rows sH (= Hold); writes r, z, Hold and Hold * r of the own units
__device__ void fr_f1(const ModelDev& md, FastSmemR& sm, int s, int k0, const float* sH, const unsigned int* wait_ctr, unsigned int wait_target) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL, tid = threadIdx.x;
  // if the helper CTAs' input-row updates are already complete (the usual case), the epilogue operand is fetched before the
  // product instead of after it
  if (tid == 0) sm.sFlag[3] = (!wait_ctr || ld_acquire_u32(wait_ctr) >= wait_target) ? 1 : 0;
  __syncthreads();
  const bool early = sm.sFlag[3] != 0;
  const int b = tid & 31, jsel = tid >> 5, j = jsel % FR_U, c = k0 + j;
  const bool isr = jsel < FR_U;
  const bool on = jsel < 2 * FR_U && b < M && c < L;
  const int col = (isr ? L : 2 * L) + c;                 // column of the gate in Wx0 rows and Bh
  const float bias = sm.rB[0][(isr ? 1 : 2) * FR_U + j];
  float pre = 0.f;
  if (early && on) pre = ly.Wx[(size_t)sm.gIdx[FK_B + b] * ly.ld3 + col] + bias;
  float acc[2 * FR_U];
  fk_slab_dot<2 * FR_U>(acc, sH, FK_LDS, sm.rC[0] + FR_U * FK_LDS, L);
  const float v = fk_slab_reduce<2 * FR_U>(acc, sm.sPart, jsel);
  if (!early) {
    if (tid == 0) wait_ge(wait_ctr, wait_target);
    __syncthreads();
    if (on) pre = ly.Wx[(size_t)sm.gIdx[FK_B + b] * ly.ld3 + col] + bias;
  }
  if (jsel < 2 * FR_U) {
    const float g = on ? sigmoidf_(v + pre) : 0.f;
    if (isr) {
      sm.gR[b * FR_U + j] = g;
      if (on) {
        const float ho = sH[b * FK_LDS + c];
        ly.r[(size_t)b * ldL + c] = g;
        ly.Hold[(size_t)b * ldL + c] = ho;
        ly.Hr[(size_t)b * ldL + c] = ho * g;
      }
    } else {
      sm.gZ[b * FR_U + j] = g;
      if (on) ly.z[(size_t)b * ldL + c] = g;
    }
  }
}
// F2 of step s (after the group barrier that completes Hold * r): h~, h, dropout, H_new of the own units
__device__ void fr_f2(const ModelDev& md, FastSmemR& sm, int s, int k0, const float* sHo) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ldL = ly.ldL, tid = threadIdx.x;
  const int b = tid & 31, jsel = tid >> 5, c = k0 + jsel;
  const bool on = jsel < FR_U && b < M && c < L;
  float pre = 0.f;
  if (on) pre = ly.Wx[(size_t)sm.gIdx[FK_B + b] * ly.ld3 + c] + sm.rB[0][jsel];
  stage_rows4(sm.gHr, FK_LDS, FK_B, ldL / 4, [&](int rr) -> const float* { return rr < M ? ly.Hr + (size_t)rr * ldL : nullptr; });
  __syncthreads();
  float acc[FR_U];
  fk_slab_dot<FR_U>(acc, sm.gHr, FK_LDS, sm.rC[0], L);
  const float v0 = fk_slab_reduce<FR_U>(acc, sm.sPart, jsel);
  if (on) {
    const float v = v0 + pre;
    const float ht = act_fwd(md.hact, v);
    const float z = sm.gZ[b * FR_U + jsel], ho = sHo[b * FK_LDS + c];
    float h = (1.0f - z) * ho + z * ht;
    if (md.p_drop_h > 0.f) h *= drop_scale(md.drop_seed, md.wG[s], 0u, (uint32_t)(b * L + c), 1.0f - md.p_drop_h);
    ly.ah[(size_t)b * ldL + c] = v;
    ly.ht[(size_t)b * ldL + c] = ht;
    ly.y[(size_t)b * ldL + c] = h;
    ly.H[(size_t)sm.gIdx[b] * ldL + c] = (sm.gIdx[2 * FK_B + b] & 1) ? 0.f : h;
  }
}
// B2 of step s (dL/dh complete): stages da_h (all units) and da_z (own units), then da_r of the own units from the resident
// rows of Wh; da_r goes to dvec for the helper CTAs and to gDr for the dense update
__device__ void fr_b2(const ModelDev& md, FastSmemR& sm, int s, int k0, const float* sHo) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, ld3 = ly.ld3, tid = threadIdx.x;
  float dz = 0.f;
  if (tid < FK_B * FR_U && tid / FR_U < M && k0 + tid % FR_U < L) dz = ly.dvec[(size_t)(tid / FR_U) * ld3 + 2 * L + k0 + tid % FR_U];
  stage_rows4(sm.sD, FK_LDS, FK_B, ly.ldL / 4, [&](int rr) -> const float* { return rr < M ? ly.dvec + (size_t)rr * ld3 : nullptr; });
  if (tid < FK_B * FR_U) sm.gDz[tid] = dz;
  __syncthreads();
  const int b = tid & 31, jsel = tid >> 5, c = k0 + jsel;
  float acc[FR_U];
  fk_slab_dot<FR_U>(acc, sm.sD, FK_LDS, sm.rR[0], L);
  const float v = fk_slab_reduce<FR_U>(acc, sm.sPart, jsel);
  if (jsel < FR_U) {
    float dar = 0.f;
    if (b < M && c < L) {
      const float ho = sHo[b * FK_LDS + c], r = sm.gR[b * FR_U + jsel];
      dar = v * ho * r * (1.f - r);
      ly.dvec[(size_t)b * ld3 + L + c] = dar;
    }
    sm.gDr[b * FR_U + jsel] = dar;
  }
}
// D of step s: gradients of the resident slabs and Bh from shared memory only (Hold, Hold * r, da_h of all units; da_r,
// da_z of the own units), summed over the lanes in order with fmaf, then updated in place.
// A task is one 16-byte quad of outputs: column tasks (resident column jm, quad q of k), row tasks (resident row j, quad q
// of the columns), then the 3 * FR_U bias entries.
__device__ void fr_dense(const ModelDev& md, FastSmemR& sm, int s, int k0, const float* sHo) {
  const LayerDev& ly = md.layer[0];
  const int M = md.wM[s], L = ly.L, kw = ly.ldL / 4;
  const bool ada = md.adapt == G4R_ADAPT_ADAGRAD, mom = md.mom > 0.f;
  const int ncol = 3 * FR_U * kw, nrow = FR_U * kw;
  for (int t = threadIdx.x; t < ncol + nrow + 3 * FR_U; t += FK_THREADS) {
    if (t < ncol + nrow) {
      const bool colt = t < ncol;
      const int u = colt ? t : t - ncol, q = u % kw, jm = u / kw, j = jm % FR_U;
      // g[e] = sum_b vec[b][e] * sc[b]; resident element o + e (o: offset in rC[*] or rR[*])
      const float* vec; const float* sc; int ss, o;
      if (colt) {
        const int m = jm / FR_U;                 // 0: Wh (Hold * r, da_h) | 1: Wrz r-block (Hold, da_r) | 2: z-block (Hold, da_z)
        vec = (m == 0 ? sm.gHr : sHo) + q * 4;
        if (m == 0) { sc = sm.sD + k0 + j; ss = FK_LDS; } else { sc = (m == 1 ? sm.gDr : sm.gDz) + j; ss = FR_U; }
        o = jm * FK_LDS + q * 4;
      } else {                                   // Wh[k0 + j][4q..]: (Hold * r)[b][k0 + j] * da_h[b][4q..]
        vec = sm.sD + q * 4; sc = sm.gHr + k0 + j; ss = FK_LDS;
        o = j * FK_LDS + q * 4;
      }
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
      for (int b = 0; b < M; b++) {
        const float4 a = ld4(vec + b * FK_LDS);
        const float d = sc[b * ss];
        g.x = fmaf(a.x, d, g.x); g.y = fmaf(a.y, d, g.y); g.z = fmaf(a.z, d, g.z); g.w = fmaf(a.w, d, g.w);
      }
      // column task: unit k0 + j, rows k = 4q + e; row task: row k0 + j, columns 4q + e
      if (k0 + j < L) {
        float* P = colt ? sm.rC[0] : sm.rR[0];
        float* A = colt ? sm.rC[1] : sm.rR[1];
        float* V = colt ? sm.rC[2] : sm.rR[2];
        if (q * 4 + 0 < L) dense_elem(md, ada, mom, g.x, P + o + 0, A + o + 0, V + o + 0);
        if (q * 4 + 1 < L) dense_elem(md, ada, mom, g.y, P + o + 1, A + o + 1, V + o + 1);
        if (q * 4 + 2 < L) dense_elem(md, ada, mom, g.z, P + o + 2, A + o + 2, V + o + 2);
        if (q * 4 + 3 < L) dense_elem(md, ada, mom, g.w, P + o + 3, A + o + 3, V + o + 3);
      }
    } else {
      const int i = t - ncol - nrow, m = i / FR_U, j = i % FR_U;
      if (k0 + j < L) {
        float g = 0.f;
        for (int b = 0; b < M; b++) g = g + (m == 0 ? sm.sD[b * FK_LDS + k0 + j] : (m == 1 ? sm.gDr : sm.gDz)[b * FR_U + j]);
        dense_elem(md, ada, mom, g, sm.rB[0] + i, sm.rB[1] + i, sm.rB[2] + i);
      }
    }
  }
}
// ---------------- loss-gradient tail of the column role (dL/do in sG, the chunk's rows in sS / sAcc / sVel) ----------------
// partial dL/dh[b][quad] = sum_j g[b][j] Sy_j[quad] of this chunk: one thread per (lane, quad)
template <class SM>
__device__ __forceinline__ void fk_part(SM& sm, float* part, int M, int nj, int ldL) {
  const int kw = ldL / 4;
  for (int t = threadIdx.x; t < M * kw; t += FK_THREADS) {
    const int bb = t / kw, q4 = t % kw;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int jj = 0; jj < nj; jj++) {
      const float g = sm.sG[jj * FK_B + bb];
      const float4 w = ld4(sm.sS + jj * FK_LDS + q4 * 4);
      a.x = fmaf(g, w.x, a.x); a.y = fmaf(g, w.y, a.y); a.z = fmaf(g, w.z, a.z); a.w = fmaf(g, w.w, a.w);
    }
    st4(part + (size_t)bb * ldL + q4 * 4, a);
  }
}
// dSy[j][quad] = sum_b g[b][j] y[b][quad] into sD: one thread per (column, 16-byte feature quad), all nj*kw pairs in parallel
template <class SM>
__device__ __forceinline__ void fk_dsy(SM& sm, int M, int nj, int kw) {
  for (int t = threadIdx.x; t < nj * kw; t += FK_THREADS) {
    const int jj = t / kw, q4 = t % kw;
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int bb = 0; bb < M; bb++) {
      const float4 y = ld4(sm.sY + bb * FK_LDS + q4 * 4);
      const float g = sm.sG[jj * FK_B + bb];
      d.x = fmaf(g, y.x, d.x); d.y = fmaf(g, y.y, d.y); d.z = fmaf(g, y.z, d.z); d.w = fmaf(g, y.w, d.w);
    }
    st4(sm.sD + jj * FK_LDS + q4 * 4, d);
  }
}
// sparse update of the chunk's Wy / By rows and their Adagrad / momentum state from shared memory (rows prefetched before
// the step, dSy in sD, dby in sDby): one warp per duplicate group
template <class SM>
__device__ __forceinline__ void fk_update_rows(const ModelDev& md, SM& sm, int buf, int nj, int kw) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ldL = md.ldL;
  const bool ada = md.adapt == G4R_ADAPT_ADAGRAD, mom = md.mom > 0.f;
  for (int j = warp; j < nj; j += FK_NW) {
    const int item = sm.sIt[buf][j];
    if (j > 0 && sm.sIt[buf][j - 1] == item) continue;
    int je = j + 1;
    while (je < nj && sm.sIt[buf][je] == item) je++;
    if (lane < kw) {
      const float4 p0 = ld4(sm.sS + j * FK_LDS + lane * 4), z = make_float4(0.f, 0.f, 0.f, 0.f);
      RowChain<float4> u;
      u.begin(p0, p0, ada ? ld4(sm.sAcc + j * FK_LDS + lane * 4) : z, mom ? ld4(sm.sVel + j * FK_LDS + lane * 4) : z);
      for (int k = j; k < je; k++) u.add(md, ld4(sm.sD + k * FK_LDS + lane * 4), ada, mom);
      const size_t off = (size_t)item * ldL + lane * 4;
      st4(md.Wy + off, u.ps);
      if (ada) st4(md.Wy_acc + off, u.al);
      if (mom) st4(md.Wy_vel + off, u.vl);
    }
    if (lane == 0) {
      RowChain<float> u;
      u.begin(sm.sByP[j], sm.sByP[j], sm.sByA[j], sm.sByV[j]);
      for (int k = j; k < je; k++) u.add(md, sm.sDby[k], ada, mom);
      md.By[item] = u.ps;
      if (ada) md.By_acc[item] = u.al;
      if (mom) md.By_vel[item] = u.vl;
    }
  }
}
// dby of the chunk's columns from sG (fixed shuffle order)
template <class SM>
__device__ __forceinline__ void fk_dby(SM& sm, int M, int nj) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int jj = warp; jj < nj; jj += FK_NW) {
    float a = (lane < M) ? sm.sG[jj * FK_B + lane] : 0.f;
    a = warp_sum(a);
    if (lane == 0) sm.sDby[jj] = a;
  }
}
// ---------------- scores and row statistics of the column role (k_fast_t and k_fast_mg) ----------------
// target activations into sT (pairwise losses: a warp per lane), then this thread's column products y_b . Sy_j into acc
// (lane b = lane, columns jj = warp + FK_NW q)
template <class SM>
__device__ __forceinline__ void fk_scores(const ModelDev& md, SM& sm, float (&acc)[FK_Q], int M, int nj, bool pw) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, kw = md.ldL / 4;
  if (pw) {
    for (int b = warp; b < FK_B; b += FK_NW) {
      if (b < M) {
        float a = 0.f;
        if (lane < kw) {
          const float4 y = ld4(sm.sY + b * FK_LDS + lane * 4), w = ld4(sm.sTW + b * FK_LDS + lane * 4);
          a = fmaf(w.x, y.x, a); a = fmaf(w.y, y.y, a); a = fmaf(w.z, y.z, a); a = fmaf(w.w, y.w, a);
        }
        a = warp_sum(a);
        if (lane == 0) sm.sT[b] = act_fwd(md.fact, a + sm.sTB[b]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < FK_Q; q++) acc[q] = 0.f;
  const float* yr = sm.sY + lane * FK_LDS;
  for (int c4 = 0; c4 < kw; c4++) {
    const float4 y = ld4(yr + c4 * 4);
#pragma unroll
    for (int q = 0; q < FK_Q; q++) {
      if (warp + FK_NW * q < nj) {
        const float4 w = ld4(sm.sS + (warp + FK_NW * q) * FK_LDS + c4 * 4);
        acc[q] = fmaf(y.x, w.x, acc[q]); acc[q] = fmaf(y.y, w.y, acc[q]); acc[q] = fmaf(y.z, w.z, acc[q]); acc[q] = fmaf(y.w, w.w, acc[q]);
      }
    }
  }
}
// scores o = acc + bias into sO, then the chunk statistics of lane b by 16 threads (columns sub, sub + 16) into md.stat: row
// max first, then plain sums -- one expf per column instead of an exp-rescaling merge per element.  The summands are written
// out here rather than taken from loss_terms: through loss_terms the compiler contracts fewer products into FMAs in this
// kernel, and the headline step's results change in the last bit.
template <class SM>
__device__ __forceinline__ void fk_chunk_stats(const ModelDev& md, SM& sm, const float (&acc)[FK_Q], int buf, int M, int cb, int nj,
                                               int chunk, bool has_chunk, bool pw) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int q = 0; q < FK_Q; q++) {
    const int jj = warp + q * FK_NW;
    if (jj < nj && lane < M) sm.sO[jj * FK_B + lane] = acc[q] + sm.sBias[jj];
  }
  __syncthreads();                          // sT and sO complete
  const int b = tid >> 4, sub = tid & 15;   // FK_THREADS / 16 == FK_B lanes
  const bool okb = b < M;
  const int tc = okb ? sm.sTc[buf][b] : -1;
  const float t = (pw && okb) ? sm.sT[b] : 0.f;
  const bool xe = loss_xe(md.loss);
  float yv[2]; bool use[2], ist[2];
  float mloc = -INFINITY;                   // max over the columns the loss weights by their softmax
#pragma unroll
  for (int q = 0; q < 2; q++) {
    const int jj = sub + 16 * q;
    use[q] = okb && jj < nj;
    ist[q] = use[q] && (tc == cb + jj);
    const float o = use[q] ? sm.sO[jj * FK_B + b] : 0.f;
    yv[q] = xe ? o : act_fwd(md.fact, o);
    if (use[q] && (xe || (loss_softmaxneg(md.loss) && !ist[q]))) mloc = fmaxf(mloc, yv[q]);
  }
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, o));
  float Z = 0.f, A = 0.f, Q = 0.f, D = 0.f, T = 0.f, has = 0.f;
#pragma unroll
  for (int q = 0; q < 2; q++) {
    if (!use[q]) continue;
    const float y = yv[q];
    if (ist[q]) has = 1.f;
    if (xe) { Z += expf(y - mloc); if (ist[q]) T = y; }
    else if (md.loss == G4R_LOSS_BPR_MAX) { if (!ist[q]) { const float e = expf(y - mloc), sg = sigmoidf_(t - y); Z += e; A += sg * e; Q += y * y * e; D += sg * (1.f - sg) * e; } }
    else if (md.loss == G4R_LOSS_TOP1_MAX) { if (!ist[q]) { const float e = expf(y - mloc), a1 = sigmoidf_(y - t), b1 = sigmoidf_(y * y); Z += e; A += (a1 + b1) * e; D += a1 * (1.f - a1) * e; } }
    else if (md.loss == G4R_LOSS_BPR) { const float sg = sigmoidf_(t - y); A += -logf(sg); if (!ist[q]) D += 1.f - sg; }
    else { const float a1 = sigmoidf_(y - t), b1 = sigmoidf_(y * y); A += a1 + b1; if (!ist[q]) D += a1 * (1.f - a1); }
  }
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) {
    Z += __shfl_xor_sync(0xffffffffu, Z, o); A += __shfl_xor_sync(0xffffffffu, A, o); Q += __shfl_xor_sync(0xffffffffu, Q, o);
    D += __shfl_xor_sync(0xffffffffu, D, o); T += __shfl_xor_sync(0xffffffffu, T, o); has += __shfl_xor_sync(0xffffffffu, has, o);
  }
  if (has_chunk && okb && sub == 0) {
    float* st = md.stat + ((size_t)chunk * md.B + b) * G4R_NSTAT;
    st4(st, make_float4(mloc, Z, A, Q));
    st4(st + 4, make_float4(D, T, has > 0.f ? 1.f : 0.f, pw ? t : 0.f));
  }
}
// RS[b] of lane b from every chunk's statistics (one CTA per lane): row max over the chunk maxima, one rescale exp per chunk,
// then plain sums (fixed shuffle / warp order)
template <class SM>
__device__ __forceinline__ void fk_row_stats(const ModelDev& md, SM& sm, int b, int M, int N) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float mc = -INFINITY, Z = 0.f, A = 0.f, Q = 0.f, D = 0.f, T = 0.f, has = 0.f, tt = 0.f;
  if (tid < md.NCH) {
    const float* st = md.stat + ((size_t)tid * md.B + b) * G4R_NSTAT;
    const float4 u = ld4(st), v = ld4(st + 4);
    mc = u.x; Z = u.y; A = u.z; Q = u.w; D = v.x; T = v.y; has = v.z;
    if (tid == 0) tt = v.w;
  }
  float mg = mc;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o));
  if (lane == 0) sm.sPart[warp] = mg;
  __syncthreads();
  mg = sm.sPart[0];
  for (int w = 1; w < FK_NW; w++) mg = fmaxf(mg, sm.sPart[w]);
  if (loss_softmaxneg(md.loss)) mg = fmaxf(mg, 0.f);          // the zeroed diagonal takes part in the max (gru4rec.py:200-202)
  if (loss_weighted(md.loss)) {
    const float sc = (mc == -INFINITY) ? 0.f : expf(mc - mg);
    Z *= sc; A *= sc; Q *= sc; D *= sc;
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Z += __shfl_xor_sync(0xffffffffu, Z, o); A += __shfl_xor_sync(0xffffffffu, A, o); Q += __shfl_xor_sync(0xffffffffu, Q, o);
    D += __shfl_xor_sync(0xffffffffu, D, o); T += __shfl_xor_sync(0xffffffffu, T, o); has += __shfl_xor_sync(0xffffffffu, has, o);
  }
  __syncthreads();
  if (lane == 0) { float* w = sm.sPart + 32 + warp * 8; w[0] = Z; w[1] = A; w[2] = Q; w[3] = D; w[4] = T; w[5] = has; w[6] = tt; }
  __syncthreads();
  if (tid == 0) {
    tt = sm.sPart[32 + 6];
    for (int w = 1; w < FK_NW; w++) { const float* q = sm.sPart + 32 + w * 8; Z += q[0]; A += q[1]; Q += q[2]; D += q[3]; T += q[4]; }
    stats_finalize(md, b, M, N, mg, Z, A, Q, D, T, tt);
  }
}
// every lane's RS into sRS; chunk 0 writes the step's cost (the lanes' losses over batch_size)
template <class SM>
__device__ __forceinline__ void fk_cost(const ModelDev& md, SM& sm, int s, int M, int chunk) {
  const int tid = threadIdx.x;
  if (tid < M * 2) st4(sm.sRS + tid * 4, ld4(md.RS + tid * 4));
  __syncthreads();
  if (chunk == 0 && tid == 0) {
    float c = 0.f;
    for (int b = 0; b < M; b++) c += sm.sRS[b * 8 + 6];
    c = __fdiv_rn(c, (float)md.B);
    md.cost[s] = c;
    if (c != c) atomicExch(md.nanflag, 1);
  }
}
// dL/do of the chunk's columns into sG (zero outside the nj x M tile)
template <class SM>
__device__ __forceinline__ void fk_grad(const ModelDev& md, SM& sm, int buf, int M, int N, int cb, int nj) {
  for (int i = threadIdx.x; i < FK_CT * FK_B; i += FK_THREADS) {
    const int jj = i / FK_B, b = i % FK_B;
    sm.sG[i] = (jj < nj && b < M) ? loss_grad_elem(md, sm.sRS + (size_t)b * 8, sm.sO[i], sm.sTc[buf][b] == cb + jj, M, N) : 0.f;
  }
}
#include "g4r_fastc.cuh"

// CL = false: GRU phases on a 48-CTA group with global group barriers (step_mode 2).
// CL = true : launched with thread-block clusters; the GRU phases run on cluster 0 (g4r_fastc.cuh, step_mode 3).
template <bool CL>
__global__ void __launch_bounds__(FK_THREADS, 1) k_fast_t(int slot, int n_steps, FastSync* fs, unsigned long long* tstamp) {
  using SM = typename std::conditional<CL, FastSmemC, FastSmemR>::type;
  extern __shared__ __align__(128) unsigned char fk_raw[];
  SM& sm = *reinterpret_cast<SM*>(fk_raw);
  const ModelDev& md = MD;
  const LayerDev& ly = md.layer[0];
  const int cta = blockIdx.x, ncta = gridDim.x;
  const int tid = threadIdx.x;
  const int G = CL ? (int)cl_size() : md.ldL / 4;   // CTAs of the GRU role (step_mode 2: one quad of hidden units each)
  const bool gru = cta < G;
  // column CTAs: step_mode 2 the CTAs after the GRU group (the host sized NCH <= ncta - G), step_mode 3 every CTA.  Column CTA
  // `chunk` owns chunk `chunk` (those beyond NCH own no columns) and combines the row statistics of lane `chunk`.
  const bool col = CL || !gru;
  const int chunk = CL ? cta : cta - G;
  const int ncol = CL ? ncta : ncta - G;       // arrivals at B2 / B3, rows_done and b1_done per step
  const bool has_chunk = col && chunk < md.NCH;
  const bool pw = loss_pairwise(md.loss);
  const int ldL = md.ldL, B = md.B;
  const int kw = ldL / 4;
  uint64_t* bar = reinterpret_cast<uint64_t*>(&sm.mbar);
  unsigned int bar_epoch = 0, gepoch = 0, stats_target = 0;
  const int in_ctas = min(B, ncta - G);        // helper CTAs [G, G + in_ctas) update the gathered input rows
#ifdef G4R_CF_FINE
#define FK_FTS(s_) ((tstamp && cta == 0 && (s_) < 500 && n_steps >= 1000) ? tstamp + (size_t)((s_) + 500) * 16 : nullptr)
#define FK_STAMP_OK(s_) ((s_) < 500)
#else
#define FK_FTS(s_) ((unsigned long long*)nullptr)
#define FK_STAMP_OK(s_) true
#endif
  // one row of 16 stamps per step: the GRU-phase slots 4-8 from CTA 0, the column-phase slots from the first column CTA
  // (step_mode 3: CTA 0 for both)
#define FK_STAMP(k) do { if (tstamp && cta == ((CL || ((k) >= 4 && (k) <= 8)) ? 0 : G) && tid == 0 && FK_STAMP_OK(s)) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); tstamp[(size_t)s * 16 + (k)] = t_; } } while (0)
  if (tid == 0) { mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  if (col) fk_load_idx(md, sm, 0, n_steps, chunk, 0);
  __syncthreads();
  if (col) fk_prefetch_rows(md, sm, 0, n_steps, 0, pw);
  // GRU forward of step 0
  ClusterCtx cc = {0, 1, 0, 0};
  if constexpr (CL) {
    if (gru) {
      cc = cf_init(md, sm);
      cf_load_resident(md, sm, cc);
      if (n_steps > 0) {
        fk_stage_lanes(md, sm, 0, md.wM[0]);
        cf_f1(md, sm, cc, 0, false, nullptr, 0u, nullptr);
        cf_f2(md, sm, cc, 0, nullptr);
        __syncthreads();
        if (tid == 0) red_release_add(&fs->h_ready, 1u);
      }
    }
  } else {
    if (gru) {
      fr_load_resident(md, sm, 4 * cta);
      if (n_steps > 0) {
        fk_stage_lanes(md, sm, 0, md.wM[0]);
        stage_rows4(sm.gH[0], FK_LDS, FK_B, kw, [&](int rr) -> const float* { const int sl = sm.gIdx[rr]; return sl >= 0 ? ly.H + (size_t)sl * ldL : nullptr; });
        fr_f1(md, sm, 0, 4 * cta, sm.gH[0], nullptr, 0u);
        fk_group_barrier(fs, gepoch, G);
        fr_f2(md, sm, 0, 4 * cta, sm.gH[0]);
        __syncthreads();
        if (tid == 0) red_release_add(&fs->h_ready, 1u);
      }
    }
  }
  for (int s = 0; s < n_steps; s++) {
    const int buf = s & 1;
    const int M = md.wM[s];
    const int sti = md.wSti[s];
    const int N = M + (sti >= 0 ? md.S : 0);
    FK_STAMP(0);
    // indices of the NEXT step (consumed after this step's last barrier)
    if (col) fk_load_idx(md, sm, s + 1, n_steps, chunk, buf ^ 1);
    const bool gru_next = !CL && gru && s + 1 < n_steps;
    if (gru_next && tid < FK_B) {               // lanes of the next step (f2 of this step has used gIdx)
      const int M1 = md.wM[s + 1];
      sm.gIdx[tid] = tid < M1 ? md.wSlot[(size_t)(s + 1) * B + tid] : -1;
      sm.gIdx[FK_B + tid] = tid < M1 ? md.wX[(size_t)(s + 1) * B + tid] : 0;
      sm.gIdx[2 * FK_B + tid] = tid < M1 ? md.wF[(size_t)(s + 1) * B + tid] : 0;
    }
    // ---- wait for h(s) ----
    if (tid == 0) wait_ge(&fs->h_ready, (unsigned int)(s + 1) * (unsigned int)G);
    __syncthreads();
    if constexpr (!CL) {
      if (!col) {
        // ---- step_mode 2 GRU role (no score columns): backward of step s once b1 is done, dense update, forward of s + 1 ----
        const bool nxt = s + 1 < n_steps;
        const int k0 = 4 * cta;
        const float* sHo = sm.gH[s & 1];                  // H rows of step s (staged one step earlier)
        float* hnext = sm.gH[(s + 1) & 1];
        // while the column CTAs run the step: the H rows of step s + 1 (final since every f2(s) has run)
        if (nxt) stage_rows4(hnext, FK_LDS, FK_B, kw, [&](int rr) -> const float* { const int sl = sm.gIdx[rr]; return sl >= 0 ? ly.H + (size_t)sl * ldL : nullptr; });
        __syncthreads();
        if (tid == 0) wait_ge(&fs->b1_done, (unsigned int)(s + 1) * (unsigned int)ncol);
        __syncthreads();
        FK_STAMP(4);
        fr_b2(md, sm, s, k0, sHo);
        __syncthreads();
        if (tid == 0) red_release_add(&fs->dvec_done, 1u);   // dvec of the step complete once all G have arrived
        FK_STAMP(5);
        fr_dense(md, sm, s, k0, sHo);
        FK_STAMP(6);
        if (nxt) {
          fr_f1(md, sm, s + 1, k0, hnext, &fs->in_done, (unsigned int)(s + 1) * (unsigned int)in_ctas);   // waits for the helper CTAs' input-row updates
          fk_group_barrier(fs, gepoch, G);                // all-gather of Hold * r
          FK_STAMP(7);
          fr_f2(md, sm, s + 1, k0, hnext);
          __syncthreads();
          if (tid == 0) red_release_add(&fs->h_ready, 1u);
        }
        FK_STAMP(8);
        continue;
      }
    }
    // ---- column role: stage h(s) ----
    stage_rows4(sm.sY, FK_LDS, FK_B, kw, [&](int rr) -> const float* { return rr < M ? ly.y + (size_t)rr * ldL : nullptr; });
    mbar_wait(bar, (unsigned int)(s & 1));      // prefetched rows of this step have landed
    __syncthreads();
    FK_STAMP(1);
    const int cb = sm.sCb[buf][0], ce = sm.sCb[buf][1];
    const int nj = ce - cb;
    // ---- scores + partial statistics ----
    {
      float acc[FK_Q];
      fk_scores(md, sm, acc, M, nj, pw);
      FK_STAMP(9);
      fk_chunk_stats(md, sm, acc, buf, M, cb, nj, chunk, has_chunk, pw);
    }
    // ---- barrier B2, then lane b's statistics are combined by column CTA b (all lanes in parallel, fixed merge order) ----
    __syncthreads();
    FK_STAMP(10);
    bar_epoch += 1;
    if (tid == 0) { red_release_add(&fs->bar, 1u); wait_ge(&fs->bar, bar_epoch * (unsigned int)ncol); }
    __syncthreads();
    if (chunk < M) {
      fk_row_stats(md, sm, chunk, M, N);
      if (tid == 0) red_release_add(&fs->stats, 1u);
    }
    stats_target += (unsigned int)M;
    if (tid == 0) wait_ge(&fs->stats, stats_target);
    __syncthreads();
    FK_STAMP(2);
    // ---- loss gradient, dSy, partial dL/dh, sparse update of this chunk's rows ----
    fk_cost(md, sm, s, M, chunk);
    FK_STAMP(11);
    fk_grad(md, sm, buf, M, N, cb, nj);
    __syncthreads();
    fk_dby(sm, M, nj);
    FK_STAMP(12);
    float* part = md.part + (size_t)(has_chunk ? chunk : 0) * md.B * ldL;
    if constexpr (CL) {
      // cluster variant: dSy, partial dL/dh and the row update before B3, then b1 and the prefetch of the next step's rows
      if (has_chunk) { fk_dsy(sm, M, nj, kw); fk_part(sm, part, M, nj, ldL); }
      __syncthreads();
      FK_STAMP(13);
      fk_update_rows(md, sm, buf, nj, kw);
      if (has_chunk && nj == 0) for (int i = tid; i < M * ldL; i += FK_THREADS) part[i] = 0.f;
      // ---- barrier B3: all updates and partial dL/dh complete ----
      __syncthreads();
      FK_STAMP(14);
      bar_epoch += 1;
      if (tid == 0) { red_release_add(&fs->bar, 1u); wait_ge(&fs->bar, bar_epoch * (unsigned int)ncta); }
      __syncthreads();
      FK_STAMP(3);
      // ---- b1 on every CTA, then prefetch the next step's rows ----
      fk_b1<CL>(md, sm, s, cta, ncta);
      __syncthreads();
      if (tid == 0) red_release_add(&fs->b1_done, 1u);
      FK_STAMP(15);
      fk_prefetch_rows(md, sm, s + 1, n_steps, buf ^ 1, pw);
      FK_STAMP(4);
      // ---- GRU role: backward, dense update, forward of the next step ----
      if (gru) {
        if (s + 1 < n_steps) fk_stage_lanes(md, sm, s + 1, md.wM[s + 1]);
        cf_backward(md, sm, cc, fs, s, ncta, s + 1 < n_steps, (tstamp && cta == 0 && FK_STAMP_OK(s)) ? tstamp + (size_t)s * 16 : nullptr, FK_FTS(s));
        FK_STAMP(6);
        if (s + 1 < n_steps) {
          cf_f1(md, sm, cc, s + 1, true, &fs->in_done, (unsigned int)(s + 1) * (unsigned int)in_ctas, FK_FTS(s));
          FK_STAMP(7);
          cf_f2(md, sm, cc, s + 1, FK_FTS(s));
          __syncthreads();
          if (tid == 0) red_release_add(&fs->h_ready, 1u);
        } else {
          cl_wait();                                   // matches the arrive left pending by cf_backward
        }
        FK_STAMP(8);
      }
      if (!gru && cta < G + in_ctas) {
        // input-row update of the step's lanes, once dvec is complete (the GRU cluster's grp counter)
        const unsigned int tgt = (unsigned int)(s + 1) * (unsigned int)G;
        if (in_ctas == B && ly.ld3 / 4 <= FK_THREADS) fk_sparse_in_one(md, sm, s, cta - G, &fs->grp, tgt);
        else {
          if (tid == 0) wait_ge(&fs->grp, tgt);
          __syncthreads();
          for (int b = cta - G; b < B; b += in_ctas) { fk_sparse_in(md, sm, s, b); __syncthreads(); }
        }
        __syncthreads();
        if (tid == 0) red_release_add(&fs->in_done, 1u);
      }
    } else {
      // partial dL/dh first: b1 and the GRU phases after it need nothing else from the column role
      if (has_chunk) fk_part(sm, part, M, nj, ldL);
      if (has_chunk && nj == 0) for (int i = tid; i < M * ldL; i += FK_THREADS) part[i] = 0.f;
      // ---- barrier B3: partial dL/dh complete ----
      __syncthreads();
      FK_STAMP(13);
      bar_epoch += 1;
      if (tid == 0) { red_release_add(&fs->bar, 1u); wait_ge(&fs->bar, bar_epoch * (unsigned int)ncol); }
      __syncthreads();
      FK_STAMP(3);
      fk_b1<CL>(md, sm, s, chunk, ncol);
      __syncthreads();
      if (tid == 0) red_release_add(&fs->b1_done, 1u);
      FK_STAMP(15);
      // ---- off the chain: dSy and the update of the chunk's Wy / By rows.  Only the TMA prefetch of the next step reads the
      // updated rows; it waits for rows_done (every column CTA's update) ----
      fk_dsy(sm, M, nj, kw);
      __syncthreads();
      if (chunk < in_ctas) {
        // helper CTA: the input-row update of the step's lanes first, once dvec is complete -- F1 of the next step waits for
        // it (in_done), the chunk's row update only gates the next prefetch.  Wx0 and Wy / By are separate tables here, so
        // the order changes no result.
        const unsigned int tgt = (unsigned int)(s + 1) * (unsigned int)G;
        if (in_ctas == B && ly.ld3 / 4 <= FK_THREADS) fk_sparse_in_one(md, sm, s, chunk, &fs->dvec_done, tgt);
        else {
          if (tid == 0) wait_ge(&fs->dvec_done, tgt);
          __syncthreads();
          for (int b = chunk; b < B; b += in_ctas) { fk_sparse_in(md, sm, s, b); __syncthreads(); }
        }
        __syncthreads();
        if (tid == 0) red_release_add(&fs->in_done, 1u);
      }
      fk_update_rows(md, sm, buf, nj, kw);
      __syncthreads();
      FK_STAMP(14);
      if (tid == 0) red_release_add(&fs->rows_done, 1u);
      if (s + 1 < n_steps) {
        if (tid == 0) wait_ge(&fs->rows_done, (unsigned int)(s + 1) * (unsigned int)ncol);
        __syncthreads();
        fk_prefetch_rows(md, sm, s + 1, n_steps, buf ^ 1, pw);
      }
    }
  }
  if constexpr (CL) { if (gru) cf_store_resident(md, sm, cc); }
  else { if (gru) fr_store_resident(md, sm, 4 * cta); }
#undef FK_STAMP
}
