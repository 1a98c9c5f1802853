// g4r_bptt.cuh -- truncated backpropagation through time (DESIGN §3l): one update per window of T consecutive mini-batches.
//
// A window runs, for each of its steps, the per-phase forward and score phases of the step (k_gather_in .. k_lossgrad, export
// mode: nothing is applied) and saves what the backward needs into the step's slice of the window buffers (BpttDev).  Then the
// gradient flows back through the window, steps in reverse and layers top-down, carried from step t to step t - 1 through each
// layer's hidden state at its physical slot (k_bptt_b1 / b2 / b3).  The dense gradients are products over the window's stacked
// events (k_bptt_dense), and the row tables get one merged update: the rows of all steps in window-position order, duplicate
// groups formed by one sort and applied through g4r_opt.cuh in position order (k_bptt_keys, k_bptt_apply).  Every sum has a
// fixed order; nothing uses atomics.  Included by g4r_lib.cu after the per-phase launch sequence.
#pragma once

// ---- forward saves of step s (upload slot) into window slice t ----
// sections (blockIdx.y): 5 per layer (Hold, r, z, a_h, h~), one input per layer, the top layer's dL/dy (the chunk partials summed
// in chunk order), the dSy rows, the per-step scalars / lanes / row lists
__global__ void __launch_bounds__(256) k_bptt_save(int slot, BpttDev w, int s, int t) {
  const ModelDev& md = MD;
  const int nl = md.n_layers, B = md.B, M = md.wM[s];
  const int sec = blockIdx.y;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
  auto rows = [&](float* dst, const float* src, int ld, int nvalid, int ntot) {
    for (int i = tid; i < ntot * ld; i += nth) dst[i] = (i / ld < nvalid) ? src[i] : 0.f;
  };
  if (sec < 5 * nl) {
    const int li = sec / 5, k = sec % 5;
    const LayerDev& ly = md.layer[li];
    const float* src = k == 0 ? ly.Hold : k == 1 ? ly.r : k == 2 ? ly.z : k == 3 ? ly.ah : ly.ht;
    float* dst = (k == 0 ? w.Hold[li] : k == 1 ? w.R[li] : k == 2 ? w.Z[li] : k == 3 ? w.Ah[li] : w.Ht[li]) + (size_t)t * B * ly.ldL;
    rows(dst, src, ly.ldL, M, B);
    return;
  }
  if (sec < 6 * nl) {
    const int li = sec - 5 * nl;
    const LayerDev& ly = md.layer[li];
    if (ly.in_dim == 0) return;
    rows(w.In[li] + (size_t)t * B * ly.ld_in, ly.in, ly.ld_in, M, B);
    return;
  }
  if (sec == 6 * nl) {
    const size_t cs = (size_t)md.B * md.ldL;
    float* dst = w.Dy + (size_t)t * B * md.ldL;
    for (int i = tid; i < B * md.ldL; i += nth) {
      float d = 0.f;
      if (i / md.ldL < M) for (int c = 0; c < md.NCH; c++) d += md.part[(size_t)c * cs + i];
      dst[i] = d;
    }
    return;
  }
  const int N = M + (md.wSti[s] >= 0 ? md.S : 0);
  if (sec == 6 * nl + 1) { rows(w.DSY + (size_t)t * md.NP * md.ldL, md.DSY, md.ldL, N, N); return; }
  for (int j = tid; j < md.NP; j += nth) {
    w.DBY[(size_t)t * md.NP + j] = j < N ? md.DBY[j] : 0.f;
    w.Item[(size_t)t * md.NP + j] = j < N ? md.pItem[(size_t)s * md.NP + j] : -1;
  }
  for (int b = tid; b < B; b += nth) {
    w.X[(size_t)t * B + b] = b < M ? md.wX[(size_t)s * B + b] : -1;
    w.Slot[(size_t)t * B + b] = b < M ? md.wSlot[(size_t)s * B + b] : 0;
    w.F[(size_t)t * B + b] = b < M ? md.wF[(size_t)s * B + b] : 0;
  }
  if (tid == 0) { w.M[t] = M; w.N[t] = N; w.G[t] = md.wG[s]; }
}

__device__ __forceinline__ float hid_mask(const ModelDev& md, uint32_t gstep, int li, int b, int L, int c) {
  return md.p_drop_h > 0.f ? drop_scale(md.drop_seed, gstep, (uint32_t)li, (uint32_t)(b * L + c), 1.0f - md.p_drop_h) : 1.0f;
}

// ---- backward of step t, layer li: dh = (dy + carry) * mask, carry zeroed where the lane's session ended at step t; da_h, da_z ----
__global__ void __launch_bounds__(256) k_bptt_b1(int slot, BpttDev w, int t, int li) {
  const ModelDev& md = MD;
  const LayerDev& ly = md.layer[li];
  const int B = md.B, M = w.M[t], L = ly.L, ldL = ly.ldL;
  const bool top = li == md.n_layers - 1;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < M * L; e += gridDim.x * blockDim.x) {
    const int b = e / L, c = e % L;
    const size_t o = ((size_t)t * B + b) * ldL + c;
    const float dy = top ? w.Dy[o] : w.Dyl[li][(size_t)b * ldL + c];
    const float cin = (w.F[(size_t)t * B + b] & 1) ? 0.f : w.Carry[li][(size_t)w.Slot[(size_t)t * B + b] * ldL + c];
    const float dh = (dy + cin) * hid_mask(md, w.G[t], li, b, L, c);
    const float ht = w.Ht[li][o], ho = w.Hold[li][o], z = w.Z[li][o], ah = w.Ah[li][o];
    float* dv = w.Dvec[li] + ((size_t)t * B + b) * ly.ld3;
    dv[c] = dh * z * act_der(md.hact, ah, ht);
    dv[2 * L + c] = dh * (ht - ho) * z * (1.f - z);
    w.Dh[li][(size_t)b * ldL + c] = dh;
  }
}

// d(H*r) = da_h Wh^T (kept for the carry); da_r = d(H*r) * H * r (1 - r)
__global__ void __launch_bounds__(GEMM_THREADS) k_bptt_b2(int slot, BpttDev w, int t, int li) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  const ModelDev& md = MD;
  const LayerDev& ly = md.layer[li];
  const int B = md.B, M = w.M[t], L = ly.L;
  const int ntn = (L + GB - 1) / GB;
  const int m0 = (blockIdx.x / ntn) * GB, n0 = (blockIdx.x % ntn) * GB;
  if (m0 >= M) return;
  float* dvec = w.Dvec[li] + (size_t)t * B * ly.ld3;
  float acc[GT][GT] = {};
  tile_gemm(acc, TileSrc{dvec, nullptr, nullptr, ly.ld3, 1, m0, 0, M, L, 1}, TileSrc{ly.Wh, nullptr, nullptr, ly.ldL, 1, n0, 0, L, L, 1}, L, sA, sB);
  const int tx = threadIdx.x % (GB / GT), ty = threadIdx.x / (GB / GT);
#pragma unroll
  for (int i = 0; i < GT; i++)
#pragma unroll
    for (int j = 0; j < GT; j++) {
      const int b = m0 + ty * GT + i, c = n0 + tx * GT + j;
      if (b >= M || c >= L) continue;
      const size_t o = ((size_t)t * B + b) * ly.ldL + c;
      const float r = w.R[li][o];
      w.DHr[li][(size_t)b * ly.ldL + c] = acc[i][j];
      dvec[(size_t)b * ly.ld3 + L + c] = acc[i][j] * w.Hold[li][o] * r * (1.f - r);
    }
}

// tiles [0, nct): the carry to step t - 1 at the lane's physical slot, dh (1 - z) + d(H*r) r + [da_r | da_z] Wrz^T;
// tiles [nct, ..): the gradient wrt the layer input, dvec Wx^T (dL/dy of the layer below, or dSx with the embedding mask)
__global__ void __launch_bounds__(GEMM_THREADS) k_bptt_b3(int slot, BpttDev w, int t, int li, int nct) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  const ModelDev& md = MD;
  const LayerDev& ly = md.layer[li];
  const int B = md.B, M = w.M[t], L = ly.L;
  const float* dvec = w.Dvec[li] + (size_t)t * B * ly.ld3;
  const int tx = threadIdx.x % (GB / GT), ty = threadIdx.x / (GB / GT);
  float acc[GT][GT] = {};
  int job = blockIdx.x;
  if (job < nct) {
    const int ntn = (L + GB - 1) / GB;
    const int m0 = (job / ntn) * GB, n0 = (job % ntn) * GB;
    if (m0 >= M) return;
    tile_gemm(acc, TileSrc{dvec + L, nullptr, nullptr, ly.ld3, 1, m0, 0, M, 2 * L, 1}, TileSrc{ly.Wrz, nullptr, nullptr, ly.ld2, 1, n0, 0, L, 2 * L, 1}, 2 * L, sA, sB);
#pragma unroll
    for (int i = 0; i < GT; i++)
#pragma unroll
      for (int j = 0; j < GT; j++) {
        const int b = m0 + ty * GT + i, c = n0 + tx * GT + j;
        if (b >= M || c >= L) continue;
        const size_t ol = (size_t)b * ly.ldL + c, o = (size_t)t * B * ly.ldL + ol;
        const float v = acc[i][j] + w.Dh[li][ol] * (1.f - w.Z[li][o]) + w.DHr[li][ol] * w.R[li][o];
        w.Carry[li][(size_t)w.Slot[(size_t)t * B + b] * ly.ldL + c] = v;
      }
    return;
  }
  job -= nct;
  const int IN = ly.in_dim;
  const int ntn = (IN + GB - 1) / GB;
  const int m0 = (job / ntn) * GB, n0 = (job % ntn) * GB;
  if (m0 >= M) return;
  tile_gemm(acc, TileSrc{dvec, nullptr, nullptr, ly.ld3, 1, m0, 0, M, 3 * L, 1}, TileSrc{ly.Wx, nullptr, nullptr, ly.ld3, 1, n0, 0, IN, 3 * L, 1}, 3 * L, sA, sB);
  const float retain = 1.0f - md.p_drop_e;
#pragma unroll
  for (int i = 0; i < GT; i++)
#pragma unroll
    for (int j = 0; j < GT; j++) {
      const int b = m0 + ty * GT + i, c = n0 + tx * GT + j;
      if (b >= M || c >= IN) continue;
      float v = acc[i][j];
      if (li > 0) w.Dyl[li - 1][(size_t)b * md.layer[li - 1].ldL + c] = v;
      else {
        if (md.p_drop_e > 0.f) v *= drop_scale(md.drop_seed, w.G[t], G4R_STREAM_EMBED, (uint32_t)(b * IN + c), retain);
        w.DSx[((size_t)t * B + b) * md.ld_in0 + c] = v;
      }
    }
}

// ---- window dense gradients of layer li: products over the K = T * B stacked events (rows past a step's M are zero in dvec) ----
__global__ void __launch_bounds__(GEMM_THREADS) k_bptt_dense(int slot, BpttDev w, int li, int K) {
  __shared__ float sA[GK * (GB + 1)], sB[GK * (GB + 1)];
  const ModelDev& md = MD;
  const LayerDev& ly = md.layer[li];
  const int L = ly.L;
  const DenseJobs dj = dense_jobs(L, ly.in_dim);
  const int tx = threadIdx.x % (GB / GT), ty = threadIdx.x / (GB / GT);
  const float* dvec = w.Dvec[li];
  float acc[GT][GT] = {};
  int job = blockIdx.x;
  float* out; int rows, cols, ldo;
  if (job < dj.nWh) {
    const int ntn = (L + GB - 1) / GB, m0 = (job / ntn) * GB, n0 = (job % ntn) * GB;
    tile_gemm(acc, TileSrc{w.Hold[li], w.R[li], nullptr, 1, ly.ldL, m0, 0, L, K, 0}, TileSrc{dvec, nullptr, nullptr, 1, ly.ld3, n0, 0, L, K, 0}, K, sA, sB);
    out = ly.Wh_g + (size_t)m0 * ly.ldL + n0; rows = L - m0; cols = L - n0; ldo = ly.ldL;
  } else if ((job -= dj.nWh) < dj.nWrz) {
    const int ntn = (2 * L + GB - 1) / GB, m0 = (job / ntn) * GB, n0 = (job % ntn) * GB;
    tile_gemm(acc, TileSrc{w.Hold[li], nullptr, nullptr, 1, ly.ldL, m0, 0, L, K, 0}, TileSrc{dvec + L, nullptr, nullptr, 1, ly.ld3, n0, 0, 2 * L, K, 0}, K, sA, sB);
    out = ly.Wrz_g + (size_t)m0 * ly.ld2 + n0; rows = L - m0; cols = 2 * L - n0; ldo = ly.ld2;
  } else if ((job -= dj.nWrz) < dj.nWx) {
    const int IN = ly.in_dim, ntn = (3 * L + GB - 1) / GB, m0 = (job / ntn) * GB, n0 = (job % ntn) * GB;
    tile_gemm(acc, TileSrc{w.In[li], nullptr, nullptr, 1, ly.ld_in, m0, 0, IN, K, 0}, TileSrc{dvec, nullptr, nullptr, 1, ly.ld3, n0, 0, 3 * L, K, 0}, K, sA, sB);
    out = ly.Wx_g + (size_t)m0 * ly.ld3 + n0; rows = IN - m0; cols = 3 * L - n0; ldo = ly.ld3;
  } else {
    job -= dj.nWx;
    const int c = job * GEMM_THREADS + threadIdx.x;
    if (c < 3 * L) {
      float g = 0.f;
      for (int e = 0; e < K; e++) g += dvec[(size_t)e * ly.ld3 + c];
      ly.Bh_g[c] = g;
    }
    return;
  }
#pragma unroll
  for (int i = 0; i < GT; i++)
#pragma unroll
    for (int j = 0; j < GT; j++) {
      const int rr = ty * GT + i, c = tx * GT + j;
      if (rr < rows && c < cols) out[(size_t)rr * ldo + c] = acc[i][j];
    }
}

// gradient row of window entry `pos` (= t * (B + NP) + r): r < B input row of lane r, else score column r - B
__device__ __forceinline__ const float* bptt_row(const ModelDev& md, const BpttDev& w, int pos) {
  const int W = md.B + md.NP, t = pos / W, r = pos % W;
  if (r >= md.B) return w.DSY + ((size_t)t * md.NP + (r - md.B)) * md.ldL;
  return md.mode == 0 ? w.Dvec[0] + ((size_t)t * md.B + r) * md.layer[0].ld3 : w.DSx + ((size_t)t * md.B + r) * md.ld_in0;
}

// grad_cap: global L2 norm over the window's merged gradient (dense sums, every row of every step); one CTA, fixed order
__global__ void __launch_bounds__(1024) k_bptt_gradnorm(int slot, BpttDev w, int T, const float* dense_flat, size_t dense_count, float* gscale) {
  __shared__ float smem[32];
  const ModelDev& md = MD;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int ldg = md.mode == 0 ? md.layer[0].ld3 : md.ld_in0;
  float a = 0.f;
  for (int t = 0; t < T; t++) {
    const int M = w.M[t], N = w.N[t];
    const float* dsy = w.DSY + (size_t)t * md.NP * md.ldL;
    for (size_t i = tid; i < (size_t)N * md.ldL; i += nt) { const float g = dsy[i]; a += g * g; }
    for (int i = tid; i < N; i += nt) { const float g = w.DBY[(size_t)t * md.NP + i]; a += g * g; }
    const float* G = md.mode == 0 ? w.Dvec[0] + (size_t)t * md.B * ldg : w.DSx + (size_t)t * md.B * ldg;
    for (int i = tid; i < M * ldg; i += nt) { const float g = G[i]; a += g * g; }
  }
  for (size_t i = tid; i < dense_count; i += nt) { const float g = dense_flat[i]; a += g * g; }
  a = warp_sum(a);
  if ((tid & 31) == 0) smem[tid >> 5] = a;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int i = 0; i < (nt >> 5); i++) s += smem[i];
    const float norm = sqrtf(s);
    gscale[0] = norm >= md.grad_cap ? __fdiv_rn(md.grad_cap, norm) : 1.0f;
  }
}

// ---- merged row list of the window: key = (table row id) << 32 | window position; table row id = item * 2 + (score column and
// the input table is not Wy).  Sorted, the duplicates of a row form one run in window-position order ----
__global__ void __launch_bounds__(256) k_bptt_keys(int slot, BpttDev w, int n) {
  const ModelDev& md = MD;
  const int W = md.B + md.NP;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int t = i / W, r = i % W;
    int item = -1, tbl = 0;
    if (r < md.B) { if (r < w.M[t]) item = w.X[(size_t)t * md.B + r]; }
    else if (r - md.B < w.N[t]) { item = w.Item[(size_t)t * md.NP + (r - md.B)]; tbl = md.mode == 2 ? 0 : 1; }
    w.keys[i] = item < 0 ? ~0ULL : (((unsigned long long)((unsigned)item * 2u + (unsigned)tbl)) << 32) | (unsigned)i;
  }
}

// one warp per run of equal rows: the update of gru4rec.py:407-431 with the run's members in window-position order, every
// right-hand side from the values at the start of the window (g4r_opt.cuh); By takes the run's score columns
__global__ void __launch_bounds__(256) k_bptt_apply(int slot, BpttDev w, int n) {
  const ModelDev& md = MD;
  const int lane = threadIdx.x & 31;
  const int e0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e0 >= n) return;
  const unsigned long long* keys = w.keys2;
  const unsigned long long k0 = keys[e0];
  if (k0 == ~0ULL) return;
  const unsigned hi = (unsigned)(k0 >> 32);
  if (e0 > 0 && (unsigned)(keys[e0 - 1] >> 32) == hi) return;          // not the start of its run
  int e1 = e0 + 1;
  while (e1 < n && keys[e1] != ~0ULL && (unsigned)(keys[e1] >> 32) == hi) e1++;
  const int nm = e1 - e0;
  const int item = (int)(hi >> 1);
  const bool out_tbl = (hi & 1u) || md.mode == 2;
  float *tab, *tacc, *tvel; int ld;
  if (out_tbl) { tab = md.Wy; tacc = md.Wy_acc; tvel = md.Wy_vel; ld = md.ldL; }
  else if (md.mode == 0) { tab = md.layer[0].Wx; tacc = md.layer[0].Wx_acc; tvel = md.layer[0].Wx_vel; ld = md.layer[0].ld3; }
  else { tab = md.E; tacc = md.E_acc; tvel = md.E_vel; ld = md.ld_in0; }
  const size_t ast = (size_t)md.n_items * ld;
  float* prow = tab + (size_t)item * ld;
  float* arow = tacc ? tacc + (size_t)item * ld : nullptr;
  float* vrow = tvel ? tvel + (size_t)item * ld : nullptr;
  auto pos = [&](int k) { return (int)(keys[e0 + k] & 0xffffffffu); };
  const int W = md.B + md.NP;
  const bool ada = md.adapt == G4R_ADAPT_ADAGRAD, mom = md.mom > 0.f;
  if (md.adapt > G4R_ADAPT_ADAGRAD) {
    opt_row_generic(md, prow, arow, ast, vrow, nullptr, ld, nm, lane, 32, true, [&](int k, int c) { return bptt_row(md, w, pos(k))[c]; });
  } else {
    const float gsc = grad_scale(md);
    for (int c4 = lane; c4 < ld / 4; c4 += 32) {
      const float4 p0 = ld4(prow + c4 * 4), z = make_float4(0.f, 0.f, 0.f, 0.f);
      RowChain<float4> u;
      u.begin(p0, p0, ada ? ld4(arow + c4 * 4) : z, mom ? ld4(vrow + c4 * 4) : z);
      for (int k = 0; k < nm; k++) {
        float4 g = ld4(bptt_row(md, w, pos(k)) + c4 * 4);
        g.x *= gsc; g.y *= gsc; g.z *= gsc; g.w *= gsc;
        u.add(md, g, ada, mom);
      }
      st4(prow + c4 * 4, u.ps);
      if (ada) st4(arow + c4 * 4, u.al);
      if (mom) st4(vrow + c4 * 4, u.vl);
    }
  }
  if (!out_tbl || lane != 0) return;
  auto dby = [&](int k) { const int p = pos(k), t = p / W; return w.DBY[(size_t)t * md.NP + (p % W - md.B)]; };
  if (md.adapt > G4R_ADAPT_ADAGRAD) {        // no shared table here: every member is a score column
    opt_row_generic(md, md.By + item, md.By_acc + item, (size_t)md.n_items, md.By_vel ? md.By_vel + item : nullptr, nullptr, 1, nm, 0, 1, true,
                    [&](int k, int) { return dby(k); });
    return;
  }
  const float gsc = grad_scale(md);
  const float p0 = md.By[item];
  RowChain<float> u;
  u.begin(p0, p0, ada ? md.By_acc[item] : 0.f, mom ? md.By_vel[item] : 0.f);
  for (int k = 0; k < nm; k++) if (pos(k) % W >= md.B) u.add(md, dby(k) * gsc, ada, mom);
  md.By[item] = u.ps;
  if (ada) md.By_acc[item] = u.al;
  if (mom) md.By_vel[item] = u.vl;
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// step s of the uploaded window: its forward and score phases, saved as step t of the BPTT window
static int bptt_forward(g4r_handle* h, int s, int t) {
  enqueue_forward_scores(h, nullptr, s);
  const int nl = h->md.n_layers;
  LAUNCH(PH_GATHER, k_bptt_save<<<dim3(std::max(1, std::min(h->n_sm, (h->md.B * h->md.ldL + 255) / 256)), 6 * nl + 3), 256, 0, h->stream>>>(h->slot, h->bw, s, t));
  return G4R_OK;
}

// the backward through the window's T saved steps and its one update
static int bptt_finish(g4r_handle* h, int T) {
  const ModelDev& md = h->md;
  const BpttDev& w = h->bw;
  cudaStream_t st = h->stream;
  const int B = md.B, nl = md.n_layers;
  for (int li = 0; li < nl; li++) {
    const LayerDev& ly = md.layer[li];
    CK(cudaMemsetAsync(w.Carry[li], 0, (size_t)B * ly.ldL * sizeof(float), st));
    CK(cudaMemsetAsync(w.Dvec[li], 0, (size_t)T * B * ly.ld3 * sizeof(float), st));
  }
  for (int t = T - 1; t >= 0; t--) {
    for (int li = nl - 1; li >= 0; li--) {
      const LayerDev& ly = md.layer[li];
      LAUNCH(PH_B1, k_bptt_b1<<<std::max(1, std::min(4 * h->n_sm, (B * ly.L + 255) / 256)), 256, 0, st>>>(h->slot, w, t, li));
      LAUNCH(PH_B2, k_bptt_b2<<<tiles2(ly.L, B), GEMM_THREADS, 0, st>>>(h->slot, w, t, li));
      const int nct = t > 0 ? tiles2(ly.L, B) : 0;
      const int nin = ly.in_dim > 0 ? tiles2(ly.in_dim, B) : 0;
      if (nct + nin > 0) LAUNCH(PH_B3, k_bptt_b3<<<nct + nin, GEMM_THREADS, 0, st>>>(h->slot, w, t, li, nct));
    }
  }
  for (int li = 0; li < nl; li++) {
    const DenseJobs dj = dense_jobs(md.layer[li].L, md.layer[li].in_dim);
    LAUNCH(PH_DENSE, k_bptt_dense<<<dj.nWh + dj.nWrz + dj.nWx + dj.nBh, GEMM_THREADS, 0, st>>>(h->slot, w, li, T * B));
  }
  const MgDev& mg = h->mgdev;
  if (md.grad_cap > 0.f) LAUNCH(PH_GRADCAP, k_bptt_gradnorm<<<1, 1024, 0, st>>>(h->slot, w, T, mg.gradFlat, mg.gradCount, h->dGscale));
  const int n = T * (B + md.NP);
  LAUNCH(PH_SPARSE_IN, k_bptt_keys<<<std::max(1, std::min(4 * h->n_sm, (n + 255) / 256)), 256, 0, st>>>(h->slot, w, n));
  size_t cb = h->bptt_cub_bytes;
  CK(cub::DeviceRadixSort::SortKeys(h->bptt_cub, cb, w.keys, w.keys2, n, 0, 64, st));
  h->launches++;
  LAUNCH(PH_SPARSE_IN, k_bptt_apply<<<(n + 7) / 8, 256, 0, st>>>(h->slot, w, n));
  for (const MgTensor& m : h->mg_tensors) LAUNCH(PH_DENSE, k_apply_dense<<<(m.count + 255) / 256, 256, 0, st>>>(h->slot, m.p, m.acc, m.vel, mg.gradFlat + m.goff, m.count));
  CK(cudaGetLastError());
  h->bptt_windows++;
  return G4R_OK;
}

// windows of the uploaded steps [0, n): every bptt steps (the last window may be shorter)
static int bptt_run_uploaded(g4r_handle* h, int n) {
  const int T = h->cfg.bptt;
  for (int k = 0; k < n; k += T) {
    const int Tw = std::min(T, n - k);
    for (int i = 0; i < Tw; i++) { int rc = bptt_forward(h, k + i, i); if (rc) return rc; }
    int rc = bptt_finish(h, Tw);
    if (rc) return rc;
  }
  if (h->gen_len > 0) h->sample_ptr += n;
  h->global_step += (uint32_t)n;
  return G4R_OK;
}

// g4r_train_steps for a window handle: steps [first, first + n) window by window.  A window's steps may straddle a regeneration
// of the sample store: they are uploaded in pieces, and each step's sample ids are in its window slice before the store changes.
static int bptt_train_steps(g4r_handle* h, const g4r_schedule* s, int64_t first, int64_t n, float* cost_out, int64_t* nan_step) {
  const int T = h->cfg.bptt;
  int64_t done = 0;
  std::vector<float> wc(T);
  while (done < n) {
    const int Tw = (int)std::min<int64_t>(T, n - done);
    for (int t = 0; t < Tw;) {
      if (h->gen_len > 0 && (!h->have_store || h->sample_ptr >= h->gen_len)) {
        int rc = g4r_generate_samples(h);
        if (rc) return rc;
      }
      const int64_t got = stage_window(h, s, first + done + t, Tw - t);
      if (got <= 0) FAIL(G4R_ERR_STATE, "empty window");
      int rc = upload_window(h, got);
      if (rc) return rc;
      for (int i = 0; i < (int)got; i++) { rc = bptt_forward(h, i, t + i); if (rc) return rc; }
      if (h->gen_len > 0) h->sample_ptr += got;
      h->global_step += (uint32_t)got;
      CK(cudaMemcpyAsync(h->hCost, h->md.cost, (size_t)got * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));        // the pinned staging buffers are refilled next
      memcpy(wc.data() + t, h->hCost, (size_t)got * sizeof(float));
      t += (int)got;
    }
    int rc = bptt_finish(h, Tw);
    if (rc) return rc;
    CK(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < Tw; i++) {
      if (cost_out) cost_out[done + i] = wc[i];
      if (wc[i] != wc[i]) {
        if (nan_step) *nan_step = first + done + i;
        FAIL(G4R_ERR_NAN, "NaN error!");
      }
    }
    done += Tw;
  }
  return G4R_OK;
}

// a range a window handle accepts: it starts at a window boundary and holds whole windows, or runs to the schedule's end
static bool bptt_aligned(const g4r_handle* h, const g4r_schedule* s, int64_t first, int64_t n) {
  const int T = h->cfg.bptt;
  return first % T == 0 && (n % T == 0 || first + n == s->n_steps);
}
