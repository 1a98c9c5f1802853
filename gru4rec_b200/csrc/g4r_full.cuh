// g4r_full.cuh -- full-softmax training (g4r_config.full_softmax = 1, DESIGN §3n): every training step scores the whole
// catalogue 0 .. n_items-1 instead of the sampled column list Y | samples, and updates every Wy / By row.
//
// The input gather, the GRU forward, the GRU backward, the dense update and phase_sparse_in are the per-phase kernels of the
// one-step path, unchanged.  What replaces score -> stats -> lossgrad:
//   k_full_stats    fp32 tiles of y . Wy^T + By (ev_tiles, FS_IT items per CTA): per (tile, lane) online max / sum-exp and the
//                   target's score -- or k_full_tc_stats, the same on the wgmma 3xTF32 tiles of the evaluation path (tc_sweep over
//                   [hi | lo] splits of y and of Wy | By, both made again every step), per 128 items
//   k_full_rowstat  one CTA per lane merges its tiles in a fixed order and finalises the row statistics (stats_finalize)
//   k_full_grad     the same tiles again (k_full_tc_grad: the same wgmma sweep), bit for bit, and dO = dL/do into an item-major
//                   [n_items][Bld] buffer; CTA 0 sums the cost
//   k_full_dy       dL/dy = dO . Wy from the rows before the update, as fixed K-split partials that k_b1 sums in order
//   k_full_rows     dWy = dO^T . y and dBy per item (K = M lanes, in order), each row updated in the product's epilogue through
//                   g4r_opt.cuh; one CTA owns each row, so there are no atomics
// Included at the end of g4r_lib.cu, after g4r_eval.cuh (ev_tiles).
#pragma once

static_assert(FS_IT == EV_IT, "the full-softmax score tiles are the fp32 evaluation tiles");
static_assert(FS_TC_M == TC_M && FS_TC_N == TC_N && FS_TC_KC == TC_KC, "the full-softmax wgmma tiles are the evaluation's");
constexpr int FR_IT = 32;     // items per CTA of the row update
constexpr int FR_IPT = 4;     // items per thread of the row update: one 16-byte load of y feeds FR_IPT accumulators
constexpr size_t FULL_STATS_SMEM = (size_t)(EV_TILE_FLOATS + 8 * EV_TB * 4) * sizeof(float);
constexpr size_t FULL_GRAD_SMEM = (size_t)EV_TILE_FLOATS * sizeof(float);
static inline size_t full_rows_smem(const ModelDev& md) { return (size_t)FR_IT * md.Bld * sizeof(float); }

// running (max, sum-exp) of a lane's scores and its target score, merged with a second partial (stat_merge's rescaling)
__device__ __forceinline__ void full_merge(float& m, float& Z, float& T, float& has, float m2, float Z2, float T2, float has2) {
  float A = 0.f, Q = 0.f, D = 0.f;
  stat_merge(m, Z, A, Q, D, m2, Z2, 0.f, 0.f, 0.f);
  if (has2 > 0.f) { T = T2; has = 1.f; }
}

__global__ void __launch_bounds__(EV_THREADS) k_full_stats(int slot, const int* base, int off, float* __restrict__ stat) {
  const ModelDev& md = MD;
  const int s = STEP_IDX;
  extern __shared__ __align__(16) float smem[];
  float* sP = smem + EV_TILE_FLOATS;                  // [8 warps][EV_TB][4] partial statistics of the current row block
  const int M = md.wM[s];
  const int i0 = blockIdx.x * EV_IT, ni = min(EV_IT, md.n_items - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ev_tiles(md, smem, M, i0, ni, nullptr, [&](int b0, const float (&acc)[8]) {
    const int b = b0 + lane;
    float m = -INFINITY, Z = 0.f, T = 0.f, has = 0.f;
    if (b < M) {
      const int y = md.wY[(size_t)s * md.B + b];
#pragma unroll
      for (int q = 0; q < 8; q++) {
        const int it = i0 + warp + 8 * q;
        if (warp + 8 * q < ni) {
          const float o = acc[q] + md.By[it];
          full_merge(m, Z, T, has, o, 1.f, o, it == y ? 1.f : 0.f);
        }
      }
    }
    st4(sP + (warp * EV_TB + lane) * 4, make_float4(m, Z, T, has));
    __syncthreads();
    if (tid < EV_TB && b0 + tid < M) {
      float4 r = ld4(sP + tid * 4);
      for (int w = 1; w < 8; w++) { const float4 u = ld4(sP + (w * EV_TB + tid) * 4); full_merge(r.x, r.y, r.z, r.w, u.x, u.y, u.z, u.w); }
      st4(stat + ((size_t)blockIdx.x * md.B + b0 + tid) * 4, r);
    }
  });
}

__global__ void __launch_bounds__(256) k_full_rowstat(int slot, const int* base, int off, const float* __restrict__ stat, int tiles) {
  const ModelDev& md = MD;
  const int s = STEP_IDX;
  const int b = blockIdx.x, M = md.wM[s];
  if (b >= M) return;
  __shared__ float4 sW[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float m = -INFINITY, Z = 0.f, T = 0.f, has = 0.f;
  for (int t = tid; t < tiles; t += blockDim.x) {
    const float4 u = ld4(stat + ((size_t)t * md.B + b) * 4);
    full_merge(m, Z, T, has, u.x, u.y, u.z, u.w);
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {    // fixed butterfly order
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), Z2 = __shfl_xor_sync(0xffffffffu, Z, o);
    const float T2 = __shfl_xor_sync(0xffffffffu, T, o), h2 = __shfl_xor_sync(0xffffffffu, has, o);
    full_merge(m, Z, T, has, m2, Z2, T2, h2);
  }
  if (lane == 0) sW[warp] = make_float4(m, Z, T, has);
  __syncthreads();
  if (tid == 0) {
    float4 r = sW[0];
    for (int w = 1; w < 8; w++) full_merge(r.x, r.y, r.z, r.w, sW[w].x, sW[w].y, sW[w].z, sW[w].w);
    stats_finalize(md, b, M, M, r.x, r.y, 0.f, 0.f, 0.f, r.z, 0.f);
  }
}

__global__ void __launch_bounds__(EV_THREADS) k_full_grad(int slot, const int* base, int off, float* __restrict__ dO) {
  const ModelDev& md = MD;
  const int s = STEP_IDX;
  extern __shared__ __align__(16) float smem[];
  const int M = md.wM[s];
  const int i0 = blockIdx.x * EV_IT, ni = min(EV_IT, md.n_items - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (blockIdx.x == 0 && tid == 0) {
    float c = 0.f;
    for (int b = 0; b < M; b++) c += md.RS[(size_t)b * G4R_NSTAT + 6];
    c = __fdiv_rn(c, (float)md.B);            // cost = loss / batch_size (gru4rec.py:577)
    md.cost[s] = c;
    if (c != c) atomicExch(md.nanflag, 1);
  }
  ev_tiles(md, smem, M, i0, ni, nullptr, [&](int b0, const float (&acc)[8]) {
    const int b = b0 + lane;
    if (b >= M) return;
    const float* rs = md.RS + (size_t)b * G4R_NSTAT;
    const int y = md.wY[(size_t)s * md.B + b];
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int it = i0 + warp + 8 * q;
      if (warp + 8 * q < ni) dO[(size_t)it * md.Bld + b] = loss_grad_elem(md, rs, acc[q] + md.By[it], it == y, M, M);
    }
  });
}

// wgmma kind of k_full_stats: thread (lane b, b + 8) x 32 items of each 256-item tile; the quad's four threads merge in a fixed
// order and write the statistics of the warpgroup's 128 items (statistics tile 2 t + column half)
__global__ void __launch_bounds__(TC_THREADS, 1) k_full_tc_stats(int slot, const int* base, int off, float* __restrict__ stat,
                                                                 const unsigned char* __restrict__ Asplit, const unsigned char* __restrict__ Bsplit) {
  const ModelDev& md = MD;
  const int s = STEP_IDX;
  const int M = md.wM[s], I = md.n_items, lane = threadIdx.x & 31, half = (threadIdx.x >> 7) >> 1;
  int bb[2], yit[2];
  auto lane_block = [&](int b) {
#pragma unroll
    for (int h = 0; h < 2; h++) { bb[h] = b + 8 * h; yit[h] = bb[h] < M ? md.wY[(size_t)s * md.B + bb[h]] : -1; }
  };
  auto tile = [&](const float (&d)[64], int c0, bool) {
    float m[2] = {-INFINITY, -INFINITY}, Z[2] = {0.f, 0.f}, T[2] = {0.f, 0.f}, has[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 64; i++) {
      const int h = (i >> 1) & 1, it = c0 + (i >> 2) * 8 + (i & 1);
      if (it < I) full_merge(m[h], Z[h], T[h], has[h], d[i], 1.f, d[i], it == yit[h] ? 1.f : 0.f);
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m[h], o), Z2 = __shfl_xor_sync(0xffffffffu, Z[h], o);
        const float T2 = __shfl_xor_sync(0xffffffffu, T[h], o), h2 = __shfl_xor_sync(0xffffffffu, has[h], o);
        full_merge(m[h], Z[h], T[h], has[h], m2, Z2, T2, h2);
      }
      const int st = 2 * ((c0 - half * 128) / TC_N) + half;
      if ((lane & 3) == 0 && bb[h] < M) st4(stat + ((size_t)st * md.B + bb[h]) * 4, make_float4(m[h], Z[h], T[h], has[h]));
    }
  };
  tc_sweep(M, I, md.L + 1, Asplit, Bsplit, lane_block, tile);
}

// wgmma kind of k_full_grad: the sweep of k_full_tc_stats again (bit for bit the same scores), dO of every live (lane, item)
__global__ void __launch_bounds__(TC_THREADS, 1) k_full_tc_grad(int slot, const int* base, int off, float* __restrict__ dO,
                                                                const unsigned char* __restrict__ Asplit, const unsigned char* __restrict__ Bsplit) {
  const ModelDev& md = MD;
  const int s = STEP_IDX;
  const int M = md.wM[s], I = md.n_items;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float c = 0.f;
    for (int b = 0; b < M; b++) c += md.RS[(size_t)b * G4R_NSTAT + 6];
    c = __fdiv_rn(c, (float)md.B);            // cost = loss / batch_size (gru4rec.py:577)
    md.cost[s] = c;
    if (c != c) atomicExch(md.nanflag, 1);
  }
  int bb[2], yit[2];
  auto lane_block = [&](int b) {
#pragma unroll
    for (int h = 0; h < 2; h++) { bb[h] = b + 8 * h; yit[h] = bb[h] < M ? md.wY[(size_t)s * md.B + bb[h]] : -1; }
  };
  auto tile = [&](const float (&d)[64], int c0, bool) {
#pragma unroll
    for (int i = 0; i < 64; i++) {
      const int h = (i >> 1) & 1, it = c0 + (i >> 2) * 8 + (i & 1);
      if (it < I && bb[h] < M)
        dO[(size_t)it * md.Bld + bb[h]] = loss_grad_elem(md, md.RS + (size_t)bb[h] * G4R_NSTAT, d[i], it == yit[h], M, M);
    }
  };
  tc_sweep(M, I, md.L + 1, Asplit, Bsplit, lane_block, tile);
}

// blockIdx.x: 32 x 32 output tile of [M lanes x L], blockIdx.y: K split of kchunk items
__global__ void __launch_bounds__(GEMM_THREADS) k_full_dy(int slot, const int* base, int off, const float* __restrict__ dO, int kchunk) {
  const ModelDev& md = MD;
  const int s = STEP_IDX;
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  const int M = md.wM[s], L = md.L, ldL = md.ldL;
  const int ntn = (L + GB - 1) / GB;
  const int m0 = (blockIdx.x / ntn) * GB, n0 = (blockIdx.x % ntn) * GB;
  if (m0 >= M) return;
  const int kb = blockIdx.y * kchunk, K = min(kchunk, md.n_items - kb);
  float acc[GT][GT] = {};
  tile_gemm(acc, TileSrc{dO + (size_t)kb * md.Bld, nullptr, nullptr, 1, md.Bld, m0, 0, M, K, 0},
            TileSrc{md.Wy + (size_t)kb * ldL, nullptr, nullptr, 1, ldL, n0, 0, L, K, 0}, K, sA, sB);
  float* part = md.part + (size_t)blockIdx.y * md.B * ldL;
  const int tx = threadIdx.x % (GB / GT), ty = threadIdx.x / (GB / GT);
#pragma unroll
  for (int i = 0; i < GT; i++)
#pragma unroll
    for (int j = 0; j < GT; j++) {
      const int b = m0 + ty * GT + i, c = n0 + tx * GT + j;
      if (b < M && c < L) part[(size_t)b * ldL + c] = acc[i][j];
    }
}

// one Wy quad of one item: the single-occurrence sparse rule of gru4rec.py:407-431 (acc / velocity / parameter of one member)
__device__ __forceinline__ void full_row_quad(const ModelDev& md, int it, int c4, float4 g, bool ada, bool mom) {
  const size_t o = (size_t)it * md.ldL + c4 * 4;
  float* prow = md.Wy + o;
  if (md.adapt > G4R_ADAPT_ADAGRAD) {
    const float gv[4] = {g.x, g.y, g.z, g.w};
    opt_row_generic(md, prow, md.Wy_acc + o, (size_t)md.n_items * md.ldL, md.Wy_vel ? md.Wy_vel + o : nullptr, nullptr, 4, 1, 0, 1, true,
                    [&](int, int c) { return gv[c]; });
    return;
  }
  const float4 p0 = ld4(prow), z = make_float4(0.f, 0.f, 0.f, 0.f);
  RowChain<float4> u;
  u.begin(p0, p0, ada ? ld4(md.Wy_acc + o) : z, mom ? ld4(md.Wy_vel + o) : z);
  u.add(md, g, ada, mom);
  st4(prow, u.ps);
  if (ada) st4(md.Wy_acc + o, u.al);
  if (mom) st4(md.Wy_vel + o, u.vl);
}

__global__ void __launch_bounds__(256) k_full_rows(int slot, const int* base, int off, const float* __restrict__ dO) {
  const ModelDev& md = MD;
  const int s = STEP_IDX;
  extern __shared__ __align__(16) float sG[];         // [FR_IT][Bld] dL/do of the CTA's items
  const int M = md.wM[s], I = md.n_items, ldL = md.ldL, Bld = md.Bld;
  const int i0 = blockIdx.x * FR_IT, ni = min(FR_IT, I - i0);
  const int tid = threadIdx.x;
  for (int i = tid; i < FR_IT * Bld; i += blockDim.x) {
    const int jj = i / Bld, b = i % Bld;
    sG[i] = (jj < ni && b < M) ? dO[(size_t)(i0 + jj) * Bld + b] : 0.f;
  }
  __syncthreads();
  const bool ada = md.adapt == G4R_ADAPT_ADAGRAD, mom = md.mom > 0.f;
  if (tid < ni) {                                     // By (gru4rec.py:486-489)
    const int it = i0 + tid;
    float g = 0.f;
    for (int b = 0; b < M; b++) g += sG[tid * Bld + b];
    if (md.adapt > G4R_ADAPT_ADAGRAD) {
      opt_row_generic(md, md.By + it, md.By_acc + it, (size_t)I, md.By_vel ? md.By_vel + it : nullptr, nullptr, 1, 1, 0, 1, true, [&](int, int) { return g; });
    } else {
      RowChain<float> u;
      u.begin(md.By[it], md.By[it], ada ? md.By_acc[it] : 0.f, mom ? md.By_vel[it] : 0.f);
      u.add(md, g, ada, mom);
      md.By[it] = u.ps;
      if (ada) md.By_acc[it] = u.al;
      if (mom) md.By_vel[it] = u.vl;
    }
  }
  const float* __restrict__ Y = md.layer[md.n_layers - 1].y;
  const int kw = ldL / 4;
  for (int u = tid; u < (FR_IT / FR_IPT) * kw; u += blockDim.x) {
    const int c4 = u % kw, j0 = (u / kw) * FR_IPT;
    if (j0 >= ni) continue;
    float4 a[FR_IPT];
#pragma unroll
    for (int j = 0; j < FR_IPT; j++) a[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int b = 0; b < M; b++) {                     // dWy[item][k] = sum_b dO[b][item] y[b][k], lanes in order
      const float4 y = ld4(Y + (size_t)b * ldL + c4 * 4);
#pragma unroll
      for (int j = 0; j < FR_IPT; j++) {
        const float g = sG[(j0 + j) * Bld + b];
        a[j].x = fmaf(g, y.x, a[j].x); a[j].y = fmaf(g, y.y, a[j].y); a[j].z = fmaf(g, y.z, a[j].z); a[j].w = fmaf(g, y.w, a[j].w);
      }
    }
#pragma unroll
    for (int j = 0; j < FR_IPT; j++)
      if (j0 + j < ni) full_row_quad(md, i0 + j0 + j, c4, a[j], ada, mom);
  }
}

// shared embedding: every input item is also a score column, and that column's update (the item's last occurrence in the Wy
// list X | 0..I-1) keeps the optimizer state -- phase_sparse_in reads the flag
__global__ void __launch_bounds__(256) k_full_xflag(uint8_t* __restrict__ xflag, const int* __restrict__ wM, int B, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * B; i += (int64_t)gridDim.x * blockDim.x)
    if ((int)(i % B) < wM[i / B]) xflag[i] |= 2;
}
static void full_mark_inputs(g4r_handle* h, int64_t n) {
  if (h->md.mode != 2) return;
  const int64_t nb = std::min<int64_t>(1024, (n * h->md.B + 255) / 256);
  k_full_xflag<<<(unsigned)nb, 256, 0, h->stream>>>(h->dXflag, h->dM, h->md.B, n);
  h->launches++;
}

static int full_opt_in(g4r_handle* h) {
  if (raise_smem_limit((const void*)k_full_stats, FULL_STATS_SMEM) != cudaSuccess || raise_smem_limit((const void*)k_full_grad, FULL_GRAD_SMEM) != cudaSuccess ||
      raise_smem_limit((const void*)k_full_rows, full_rows_smem(h->md)) != cudaSuccess ||
      raise_smem_limit((const void*)k_full_tc_stats, sizeof(TcSmem)) != cudaSuccess || raise_smem_limit((const void*)k_full_tc_grad, sizeof(TcSmem)) != cudaSuccess)
    return G4R_ERR_INVALID;
  return G4R_OK;
}

static int enqueue_full_step(g4r_handle* h, const int* base, int off) {
  const ModelDev& md = h->md;
  const FullDev& f = h->fs;
  cudaStream_t st = h->stream;
  enqueue_forward(h, base, off);
  if (f.tc) {
    // the operands as [hi | lo] TF32 blocks: y of every lane (rows past the step's M are never read back), Wy | By of this step
    const int sweep = std::min((md.n_items + TC_N - 1) / TC_N, h->n_sm);
    LAUNCH(PH_SCORE, k_tc_split<TC_M><<<dim3((md.B + TC_M - 1) / TC_M, f.chunks), 256, 0, st>>>(md.layer[md.n_layers - 1].y, md.B, md.ldL, md.L, f.Asplit, f.chunks, nullptr, 1.0f));
    LAUNCH(PH_SCORE, k_tc_split<TC_N><<<dim3((md.n_items + TC_N - 1) / TC_N, f.chunks), 256, 0, st>>>(md.Wy, md.n_items, md.ldL, md.L, f.Bsplit, f.chunks, md.By, 0.f));
    LAUNCH(PH_SCORE, k_full_tc_stats<<<sweep, TC_THREADS, sizeof(TcSmem), st>>>(h->slot, base, off, f.stat, f.Asplit, f.Bsplit));
    LAUNCH(PH_STATS, k_full_rowstat<<<md.B, 256, 0, st>>>(h->slot, base, off, f.stat, f.tiles));
    LAUNCH(PH_LOSSGRAD, k_full_tc_grad<<<sweep, TC_THREADS, sizeof(TcSmem), st>>>(h->slot, base, off, f.dO, f.Asplit, f.Bsplit));
  } else {
    LAUNCH(PH_SCORE, k_full_stats<<<f.tiles, EV_THREADS, FULL_STATS_SMEM, st>>>(h->slot, base, off, f.stat));
    LAUNCH(PH_STATS, k_full_rowstat<<<md.B, 256, 0, st>>>(h->slot, base, off, f.stat, f.tiles));
    LAUNCH(PH_LOSSGRAD, k_full_grad<<<f.tiles, EV_THREADS, FULL_GRAD_SMEM, st>>>(h->slot, base, off, f.dO));
  }
  const int mn = ((md.B + GB - 1) / GB) * ((md.L + GB - 1) / GB);
  LAUNCH(PH_LOSSGRAD, k_full_dy<<<dim3(mn, f.ks), GEMM_THREADS, 0, st>>>(h->slot, base, off, f.dO, f.kchunk));
  LAUNCH(PH_LOSSGRAD, k_full_rows<<<(md.n_items + FR_IT - 1) / FR_IT, 256, full_rows_smem(md), st>>>(h->slot, base, off, f.dO));
  enqueue_backward(h, base, off, f.ks);
  return G4R_OK;
}
static int64_t full_launches_per_step(const g4r_handle* h) {
  const ModelDev& md = h->md;
  int64_t n = (md.mode != 0 ? 1 : 0) + 5 + (h->fs.tc ? 2 : 0) + 1;     // gather + [2 splits] + stats / rowstat / grad / dy / rows + sparse_in
  for (int li = 0; li < md.n_layers; li++) n += 2 + 2 + (md.layer[li].in_dim > 0 ? 1 : 0) + 1;
  return n;
}
