// g4r_stamp.cuh -- the STAMP short-term attention/memory baseline on the device (DESIGN §3v): per query (a prefix's last max_len
// inputs) the session mean m_s and the last click m_t, the attention a_i = w0 . sig(x_i W1 + m_t W2 + m_s W3 + b_a) without
// normalisation, m_a = sum_i a_i x_i, the two tanh cells h_s = tanh(m_a Ws + bs), h_t = tanh(m_t Wt + bt), q = h_s h_t and
// full-catalogue cross-entropy over E q, trained with NARM's dense Adam; and the eval-mode encoder that feeds per-event vectors to
// BPR's ranking.  Every dense product runs through NARM's k_nm_gemm, the catalogue loss through k_nm_softmax, the input-embedding
// gradient through k_nm_keys / k_nm_scatter; the training samples and batch plan are SR-GNN's, evaluation chunks NARM's planner.
// Every reduction runs in a fixed order (no floating-point atomics), so a fit is bitwise reproducible.  A handle keeps its model
// in the handle's NARM fields and its samples and scratch in SR-GNN's.  Included at the end of g4r_lib.cu after g4r_srgnn.cuh.
#pragma once

constexpr int ST_D_MAX = 1024, ST_LEN_MAX = 512;
constexpr int ST_THREADS = 256;                        // attention and input-gradient CTAs (one per query)
constexpr int ST_EVAL_POS = 16384;                     // positions (and pieces) per evaluation chunk

// offsets of the parameters in the flat float32 vector (DESIGN §3v); W2 and W3 are adjacent, so [W2 ; W3] is one [2d x d] matrix
struct StLayout {
  size_t E, W1, W2, W3, ba, w0, Ws, bs, Wt, bt, n;
};
static StLayout st_layout(int NI, int d) {
  StLayout L;
  const size_t D = d, DD = D * D;
  L.E = 0; L.W1 = (size_t)NI * D; L.W2 = L.W1 + DD; L.W3 = L.W2 + DD; L.ba = L.W3 + DD; L.w0 = L.ba + D; L.Ws = L.w0 + D; L.bs = L.Ws + DD;
  L.Wt = L.bs + D; L.bt = L.Wt + DD; L.n = L.bt + D;
  return L;
}

// one mini-batch (or evaluation chunk): nb pieces, piece b the plen[b] inputs items[pstart[b] ..] at positions poff[b] ..; nq
// queries, query j the inputs at positions qs[j] .. qp[j] (n = qp - qs + 1 of them, the last one the last click).  A training
// sample is one piece with one query over all of it, its target the item after the piece.
struct StDev {
  const int* items; const long long* pstart; const int* plen; const int* poff; int nb, P;
  const int* qs; const int* qp; int nq;
  const float* E;
  int d, train;
  int *PX, *PY;                                          // per position: input item; per query: target
};

// CTA per piece: X[p] = E[input] and PX; a training piece's target
__global__ void __launch_bounds__(ST_THREADS) k_st_gather(StDev g, float* X) {
  const int b = blockIdx.x, n = g.plen[b], p0 = g.poff[b], d = g.d;
  const long long s0 = g.pstart[b];
  for (int z = threadIdx.x; z < n * d; z += blockDim.x) {
    const int t = z / d, c = z % d, it = g.items[s0 + t];
    if (c == 0) g.PX[p0 + t] = it;
    X[(size_t)(p0 + t) * d + c] = g.E[(size_t)it * d + c];
  }
  if (g.train && threadIdx.x == 0) g.PY[b] = g.items[s0 + n];
}

// thread per (query, unit): MC[j] = [m_t ; m_s], m_t = x_n, m_s = (sum over positions in order of x_i) / n
__global__ void k_st_means(StDev g, const float* X, float* MC) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)g.nq * g.d) return;
  const int j = (int)(i / g.d), c = (int)(i % g.d), d = g.d, a = g.qs[j], e = g.qp[j];
  float s = 0.f;
  for (int p = a; p <= e; p++) s = __fadd_rn(s, X[(size_t)p * d + c]);
  MC[(size_t)j * 2 * d + c] = X[(size_t)e * d + c];
  MC[(size_t)j * 2 * d + d + c] = __fdiv_rn(s, (float)(e - a + 1));
}

// sig(x_i W1 + [m_t ; m_s] [W2 ; W3] + b_a) of unit c, from U = X W1 and V = MC [W2 ; W3]
__device__ __forceinline__ float st_sig(float u, float v, float ba) { return nm_sig(__fadd_rn(__fadd_rn(u, v), ba)); }

// CTA per query: a_i = w0 . sig(.) (warp per position, lanes strided over units then sg_warp_sum's fixed tree), m_a = sum over
// positions in order of a_i x_i; a training batch keeps a_i per position (ALPHA; its queries own their positions)
__global__ void __launch_bounds__(ST_THREADS) k_st_att(StDev g, const float* X, const float* U, const float* V, const float* ba, const float* w0,
                                                       float* ALPHA, float* MA) {
  __shared__ float al[ST_LEN_MAX];
  const int j = blockIdx.x, a = g.qs[j], n = g.qp[j] - a + 1, d = g.d, lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* v = V + (size_t)j * d;
  for (int t = w; t < n; t += nw) {
    const size_t p = (size_t)(a + t);
    float s = 0.f;
    for (int c = lane; c < d; c += 32) s = __fmaf_rn(w0[c], st_sig(U[p * d + c], v[c], ba[c]), s);
    s = sg_warp_sum(s);
    if (lane == 0) { al[t] = s; if (ALPHA) ALPHA[p] = s; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < n; t++) s = __fmaf_rn(al[t], X[(size_t)(a + t) * d + c], s);
    MA[(size_t)j * d + c] = s;
  }
}

// thread per (query, unit): h_s = tanh(AS + bs), h_t = tanh(AT + bt), q = h_s h_t into row `row[j]` of Q (j without row)
__global__ void k_st_cells(int nq, int d, const float* AS, const float* AT, const float* bs, const float* bt, float* HS, float* HT, const int* row,
                           float* Q) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nq * d) return;
  const int j = (int)(i / d), c = (int)(i % d);
  const float hs = tanhf(__fadd_rn(AS[i], bs[c])), ht = tanhf(__fadd_rn(AT[i], bt[c]));
  if (HS) { HS[i] = hs; HT[i] = ht; }
  Q[(size_t)(row ? row[j] : j) * d + c] = __fmul_rn(hs, ht);
}

// thread per (query, unit), the cells' backward from DQ: DAS = dq h_t (1 - h_s^2), DAT = dq h_s (1 - h_t^2)
__global__ void k_st_cells_bwd(int nq, int d, const float* DQ, const float* HS, const float* HT, float* DAS, float* DAT) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nq * d) return;
  const float dq = DQ[i], hs = HS[i], ht = HT[i];
  DAS[i] = __fmul_rn(__fmul_rn(dq, ht), __fsub_rn(1.f, __fmul_rn(hs, hs)));
  DAT[i] = __fmul_rn(__fmul_rn(dq, hs), __fsub_rn(1.f, __fmul_rn(ht, ht)));
}

// CTA per query (a training batch: its own positions), the attention's backward from DMA = dL/dm_a: da_i = DMA . x_i;
// DSIG[p] = da_i w0 sig' (dL/dU, and each position's part of dL/dV), DW0[p] = da_i sig (w0's gradient rows), DXA[p] = a_i DMA
// (the m_a part of dL/dx_i); DV[j] = sum over positions in order of DSIG
__global__ void __launch_bounds__(ST_THREADS) k_st_att_bwd(StDev g, const float* X, const float* U, const float* V, const float* ba, const float* w0,
                                                           const float* ALPHA, const float* DMA, float* DSIG, float* DW0, float* DXA, float* DV) {
  __shared__ float da[ST_LEN_MAX];
  const int j = blockIdx.x, a = g.qs[j], n = g.qp[j] - a + 1, d = g.d, lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float *v = V + (size_t)j * d, *dm = DMA + (size_t)j * d;
  for (int t = w; t < n; t += nw) {
    float s = 0.f;
    for (int c = lane; c < d; c += 32) s = __fmaf_rn(dm[c], X[(size_t)(a + t) * d + c], s);
    s = sg_warp_sum(s);
    if (lane == 0) da[t] = s;
  }
  __syncthreads();
  for (int z = threadIdx.x; z < n * d; z += blockDim.x) {
    const int t = z / d, c = z % d;
    const size_t p = (size_t)(a + t);
    const float u = st_sig(U[p * d + c], v[c], ba[c]);
    DSIG[p * d + c] = __fmul_rn(__fmul_rn(da[t], w0[c]), __fmul_rn(u, __fsub_rn(1.f, u)));
    DW0[p * d + c] = __fmul_rn(da[t], u);
    DXA[p * d + c] = __fmul_rn(ALPHA[p], dm[c]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < n; t++) s = __fadd_rn(s, DSIG[(size_t)(a + t) * d + c]);
    DV[(size_t)j * d + c] = s;
  }
}

// CTA per query (a training batch), dL/dx_i of its positions: (DXA + T1) + dm_s / n, and at the last click + (dm_t + DMT), with
// T1 = DSIG W1^T, DMC = [dm_t ; dm_s] = DV [W2 ; W3]^T and DMT = DAT Wt^T
__global__ void __launch_bounds__(ST_THREADS) k_st_dx(StDev g, const float* DXA, const float* T1, const float* DMC, const float* DMT, float* DX) {
  const int j = blockIdx.x, a = g.qs[j], n = g.qp[j] - a + 1, d = g.d;
  const float* dmc = DMC + (size_t)j * 2 * d;
  for (int z = threadIdx.x; z < n * d; z += blockDim.x) {
    const int t = z / d, c = z % d;
    const size_t p = (size_t)(a + t);
    float s = __fadd_rn(__fadd_rn(DXA[p * d + c], T1[p * d + c]), __fdiv_rn(dmc[d + c], (float)n));
    if (t == n - 1) s = __fadd_rn(s, __fadd_rn(dmc[c], DMT[(size_t)j * d + c]));
    DX[p * d + c] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
// the float arrays of a batch of P positions and nq queries; evaluation carries no backward buffers and writes q in place
struct StBuf {
  float *X, *U, *ALPHA;                                  // per position
  float *MC, *V, *MA, *AS, *AT, *HS, *HT, *Q;            // per query
  float *DSIG, *DW0, *DXA, *T1, *DX;                     // the backward, per position
  float *LOSS, *DQ, *DAS, *DAT, *DMA, *DMT, *DV, *DMC;   // per query
};
static size_t st_pos_floats(int d, bool train) { return train ? (size_t)7 * d + 1 : (size_t)2 * d; }
static size_t st_qry_floats(int d, bool train) { return train ? (size_t)17 * d + 1 : (size_t)6 * d; }
// pcap positions and qcap queries of room
static void st_carve(StBuf& B, float* f, long long pcap, long long qcap, int d, bool train) {
  B = StBuf{};
  auto pos = [&](float** q, size_t w) { *q = f; f += (size_t)pcap * w; };
  auto qry = [&](float** q, size_t w) { *q = f; f += (size_t)qcap * w; };
  pos(&B.X, d); pos(&B.U, d);
  qry(&B.MC, 2 * d); qry(&B.V, d); qry(&B.MA, d); qry(&B.AS, d); qry(&B.AT, d);
  if (!train) return;
  qry(&B.HS, d); qry(&B.HT, d); pos(&B.ALPHA, 1); pos(&B.DSIG, d); pos(&B.DW0, d); pos(&B.DXA, d); pos(&B.T1, d); pos(&B.DX, d);
  qry(&B.Q, d); qry(&B.LOSS, 1); qry(&B.DQ, d); qry(&B.DAS, d); qry(&B.DAT, d); qry(&B.DMA, d); qry(&B.DMT, d); qry(&B.DV, d); qry(&B.DMC, 2 * d);
}
constexpr int ST_INTS_POS = 1, ST_INTS_QRY = 2;         // PX; PY and qp (a training batch's qs is its poff)

static unsigned st_grid(long long n) { return (unsigned)((n + 255) / 256); }

// the encoder of a batch or chunk: q of every query into row row[j] of Q (encoder products never split k)
static void st_encode(cudaStream_t st, const StDev& g, const StBuf& B, const float* th, const StLayout& Lo, const int* row, float* Q) {
  const int P = g.P, d = g.d, nq = g.nq;
  k_st_gather<<<g.nb, ST_THREADS, 0, st>>>(g, B.X);
  k_st_means<<<st_grid((long long)nq * d), 256, 0, st>>>(g, B.X, B.MC);
  nm_gemm<NM_ENCODER>(st, nullptr, B.X, d, 1, th + Lo.W1, d, 1, B.U, d, P, d, d);
  nm_gemm<NM_ENCODER>(st, nullptr, B.MC, 2 * d, 1, th + Lo.W2, d, 1, B.V, d, nq, d, 2 * d);
  k_st_att<<<nq, ST_THREADS, 0, st>>>(g, B.X, B.U, B.V, th + Lo.ba, th + Lo.w0, B.ALPHA, B.MA);
  nm_gemm<NM_ENCODER>(st, nullptr, B.MA, d, 1, th + Lo.Ws, d, 1, B.AS, d, nq, d, d);
  nm_gemm<NM_ENCODER>(st, nullptr, B.MC, 2 * d, 1, th + Lo.Wt, d, 1, B.AT, d, nq, d, d);
  k_st_cells<<<st_grid((long long)nq * d), 256, 0, st>>>(nq, d, B.AS, B.AT, th + Lo.bs, th + Lo.bt, B.HS, B.HT, row, Q);
}

// a batch's loss and gradient G of the loss (flat, the parameters' layout) at th; loss_out a device float
static void st_grad(cudaStream_t st, const StDev& g, const StBuf& B, const NmScratch& ns, const float* th, const StLayout& Lo, int NI, float* G,
                    const float* ones, float* loss_out) {
  const int P = g.P, d = g.d, nq = g.nq;
  float* part = ns.part;
  st_encode(st, g, B, th, Lo, nullptr, B.Q);
  // the catalogue: logits, the softmax gradient, dL/dq and dE
  NmDev nd{};
  nd.P = nq; nd.d = d; nd.NI = NI; nd.S = ns.S; nd.PY = g.PY; nd.LOSS = B.LOSS; nd.re = 1.f;
  const float* E = th + Lo.E;
  nm_gemm<NM_CATALOGUE>(st, part, B.Q, d, 1, E, 1, d, ns.S, NI, nq, NI, d);
  k_nm_softmax<<<nq, 256, 0, st>>>(nd);
  k_nm_mean<<<1, 1024, 0, st>>>(B.LOSS, nq, loss_out);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, NI, 1, E, d, 1, B.DQ, d, nq, d, NI);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, 1, NI, B.Q, d, 1, G + Lo.E, d, NI, d, nq);
  // the cells
  k_st_cells_bwd<<<st_grid((long long)nq * d), 256, 0, st>>>(nq, d, B.DQ, B.HS, B.HT, B.DAS, B.DAT);
  nm_gemm<NM_BACKWARD>(st, part, B.MA, 1, d, B.DAS, d, 1, G + Lo.Ws, d, d, d, nq);
  sg_colsum(st, part, ones, B.DAS, d, G + Lo.bs, nq, d);
  nm_gemm<NM_BACKWARD>(st, part, B.MC, 1, 2 * d, B.DAT, d, 1, G + Lo.Wt, d, d, d, nq);
  sg_colsum(st, part, ones, B.DAT, d, G + Lo.bt, nq, d);
  nm_gemm<NM_BACKWARD>(st, part, B.DAS, d, 1, th + Lo.Ws, 1, d, B.DMA, d, nq, d, d);
  nm_gemm<NM_BACKWARD>(st, part, B.DAT, d, 1, th + Lo.Wt, 1, d, B.DMT, d, nq, d, d);
  // the attention
  k_st_att_bwd<<<nq, ST_THREADS, 0, st>>>(g, B.X, B.U, B.V, th + Lo.ba, th + Lo.w0, B.ALPHA, B.DMA, B.DSIG, B.DW0, B.DXA, B.DV);
  nm_gemm<NM_BACKWARD>(st, part, B.X, 1, d, B.DSIG, d, 1, G + Lo.W1, d, d, d, P);
  sg_colsum(st, part, ones, B.DW0, d, G + Lo.w0, P, d);
  sg_colsum(st, part, ones, B.DV, d, G + Lo.ba, nq, d);
  nm_gemm<NM_BACKWARD>(st, part, B.MC, 1, 2 * d, B.DV, d, 1, G + Lo.W2, d, 2 * d, d, nq);
  nm_gemm<NM_BACKWARD>(st, part, B.DV, d, 1, th + Lo.W2, 1, d, B.DMC, 2 * d, nq, 2 * d, d);
  nm_gemm<NM_BACKWARD>(st, part, B.DSIG, d, 1, th + Lo.W1, 1, d, B.T1, d, P, d, d);
  k_st_dx<<<nq, ST_THREADS, 0, st>>>(g, B.DXA, B.T1, B.DMC, B.DMT, B.DX);
  // the input embeddings: dL/dx rows added to E's rows, positions sorted by (item, position)
  NmDev ne{};
  ne.P = P; ne.d = d; ne.DEMB = B.DX; ne.PS = g.PX; ne.re = 1.f;
  k_nm_keys<<<(P + 255) / 256, 256, 0, st>>>(g.PX, P, ns.keys);
  int end_bit = 33;
  while (end_bit < 64 && ((unsigned long long)NI >> (end_bit - 32)) != 0ull) end_bit++;
  size_t cb = ns.cub_bytes;
  cub::DeviceRadixSort::SortKeys(ns.cub, cb, ns.keys, ns.keys2, P, 0, end_bit, st);
  k_nm_scatter<<<st_grid((long long)P * d), 256, 0, st>>>(ne, ns.keys2, G + Lo.E);
}

static bool st_len_ok(int len) { return len >= 1 && len <= ST_LEN_MAX; }
#define ST_LEN_MSG ": need max_len in 1 .. 512"

// the model buffers of a STAMP handle (NARM's fields): parameters, double(E) and zero biases for bpr_blocks, a device 1.0f
static int st_set_model(g4r_baselines* h, int32_t max_len, const float* params, int64_t n_params, const char* who) {
  if (!params) FAIL(G4R_ERR_INVALID, std::string(who) + ": null parameters");
  if (!st_len_ok(max_len)) FAIL(G4R_ERR_INVALID, std::string(who) + ST_LEN_MSG);
  const StLayout L = st_layout(h->n_items, h->n_keep);
  if (n_params != (int64_t)L.n) FAIL(G4R_ERR_INVALID, std::string(who) + ": need n_params = n_items d + 5 d^2 + 4 d = " + std::to_string(L.n));
  if (!nm_finite(params, L.n)) FAIL(G4R_ERR_INVALID, std::string(who) + ": the parameters must be finite");
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  h->ready = false;
  nm_free_fit(h);
  for (void* p : {(void*)h->dNmTh, (void*)h->dI, (void*)h->dBI, (void*)h->dNmOne}) if (p) cudaFree(p);
  h->dNmTh = nullptr; h->dI = nullptr; h->dBI = nullptr; h->dNmOne = nullptr;
  CK(bl_alloc(&h->dNmTh, L.n)); CK(bl_alloc(&h->dI, (size_t)h->n_items * h->n_keep)); CK(bl_alloc(&h->dBI, h->n_items)); CK(bl_alloc(&h->dNmOne, 1));
  const float one = 1.f;
  CK(cudaMemcpyAsync(h->dNmTh, params, L.n * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(h->dNmOne, &one, sizeof(float), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(h->dBI, 0, (size_t)h->n_items * sizeof(double), st));
  h->nm_len = max_len; h->nm_n = L.n;
  const size_t nE = (size_t)h->n_items * h->n_keep;
  k_nm_to_double<<<(unsigned)((nE + 255) / 256), 256, 0, st>>>(h->dNmTh, nE, h->dI);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_stamp_import(g4r_baselines* h, int32_t max_len, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_STAMP) FAIL(G4R_ERR_STATE, "g4r_bl_stamp_import: the handle is not a STAMP");
  return st_set_model(h, max_len, params, n_params, "g4r_bl_stamp_import");
}

extern "C" int g4r_bl_stamp_export(g4r_baselines* h, float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_STAMP || !h->dNmTh) FAIL(G4R_ERR_STATE, "g4r_bl_stamp_export: no STAMP parameters (g4r_bl_stamp_begin or g4r_bl_stamp_import)");
  if (!params || n_params != (int64_t)h->nm_n) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_export: need n_params floats");
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(params, h->dNmTh, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

extern "C" int g4r_bl_stamp_begin(g4r_baselines* h, int32_t max_len, int32_t batch_size, const int64_t* session_offsets, int64_t n_sessions,
                                  const int32_t* items, int64_t n_entries, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_STAMP) FAIL(G4R_ERR_STATE, "g4r_bl_stamp_begin: the handle is not a STAMP");
  if (!session_offsets || !items || n_sessions < 1 || n_entries < 2 || batch_size < 1)
    FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_begin: null argument, no sessions or batch_size < 1");
  const int NI = h->n_items, dd = h->n_keep;
  if (!st_len_ok(max_len)) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_begin" ST_LEN_MSG);
  if (n_entries > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_begin: more than 2^31 - 1 entries");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_entries)) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_begin: session offsets must rise from 0 to n_entries");
  for (int64_t e = 0; e < n_entries; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_stamp_begin: item index out of range");
  if ((uint64_t)batch_size * (uint64_t)max_len * 2ull * (uint64_t)dd >= 0x80000000ull)
    FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_begin: batch_size * max_len * 2 d must stay below 2^31 (flat indices of a batch)");
  std::vector<int64_t> s0; std::vector<int> sn;
  sg_samples(session_offsets, n_sessions, max_len, s0, sn);
  if (s0.empty()) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_begin: no session of at least 2 events");
  if (s0.size() > (size_t)INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_begin: more than 2^31 - 1 samples");
  const long long Pmax = sg_longest(sn, batch_size);
  const StLayout L = st_layout(NI, dd);
  const size_t act = (size_t)Pmax * st_pos_floats(dd, true) * 4 + (size_t)batch_size * st_qry_floats(dd, true) * 4;
  const size_t need = (size_t)batch_size * NI * 4 + act + (size_t)Pmax * (ST_INTS_POS * 4 + 16) + (size_t)batch_size * ST_INTS_QRY * 4 + NM_PART_CAP * 4 +
                      3 * L.n * 4 + (size_t)n_entries * 4 + s0.size() * 12 + ((size_t)64 << 20);
  int rc = st_set_model(h, max_len, params, n_params, "g4r_bl_stamp_begin");
  if (rc) return rc;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    h->err = "g4r_bl_stamp_begin: the fit needs " + std::to_string(need) + " bytes of device memory (the logits of the largest batch " +
             std::to_string((size_t)batch_size * NI * 4) + ", its activations " + std::to_string(act) + "), " + std::to_string(free_b) + " are free";
    return G4R_ERR_CUDA;
  }
  cudaStream_t st = h->stream;
  h->ready = false;
  NmScratch& s = h->nm_s;
  s = NmScratch{};
  size_t cb = 0;
  CK(cub::DeviceRadixSort::SortKeys(nullptr, cb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)Pmax, 0, 64));
  CK(nm_take(h, &s.part, NM_PART_CAP)); CK(nm_take(h, &s.S, (size_t)batch_size * NI)); CK(nm_take(h, &s.keys, Pmax)); CK(nm_take(h, &s.keys2, Pmax));
  CK(nm_take(h, &s.cub, cb));
  s.cub_bytes = cb;
  CK(nm_take(h, &h->sg_f, (size_t)Pmax * st_pos_floats(dd, true) + (size_t)batch_size * st_qry_floats(dd, true)));
  CK(nm_take(h, &h->sg_i, (size_t)Pmax * ST_INTS_POS + (size_t)batch_size * ST_INTS_QRY));
  CK(nm_take(h, &h->dNmG, L.n)); CK(nm_take(h, &h->dNmM, L.n)); CK(nm_take(h, &h->dNmV, L.n)); CK(nm_take(h, &h->dNmItems, n_entries));
  CK(nm_take(h, &h->dNmLoss, 1));
  CK(cudaMemsetAsync(h->dNmM, 0, L.n * sizeof(float), st)); CK(cudaMemsetAsync(h->dNmV, 0, L.n * sizeof(float), st));
  CK(cudaMemcpyAsync(h->dNmItems, items, n_entries * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  h->sg_start.swap(s0); h->sg_len.swap(sn);
  h->nm_bs = batch_size; h->nm_Pmax = Pmax; h->sg_icap = Pmax; h->nm_step = 0; h->nm_fit = true;
  h->ready = true;
  return G4R_OK;
}

static int st_check_run(g4r_baselines* h, const int32_t* samples, int64_t n, const char* who) {
  if (h->kind != BL_STAMP) FAIL(G4R_ERR_STATE, std::string(who) + ": the handle is not a STAMP");
  if (!h->nm_fit) FAIL(G4R_ERR_STATE, std::string(who) + ": no fit begun (g4r_bl_stamp_begin)");
  if (!samples || n < 1) FAIL(G4R_ERR_INVALID, std::string(who) + ": no samples");
  const int64_t ns = (int64_t)h->sg_start.size();
  for (int64_t q = 0; q < n; q++) if (samples[q] < 0 || samples[q] >= ns) FAIL(G4R_ERR_INDEX, std::string(who) + ": sample index out of range");
  return G4R_OK;
}

// SR-GNN's batch plan of a list of samples (refusing a batch past the scratch), plus each sample's last position qp
static int st_plan(g4r_baselines* h, const int32_t* samples, int64_t n, std::vector<long long>& ps, std::vector<int>& pl, std::vector<int>& po,
                   std::vector<int>& qp, std::vector<std::pair<int64_t, int>>& batches, const char* who) {
  const int rc = sg_plan(h, samples, n, ps, pl, po, batches, who);
  if (rc) return rc;
  qp.resize(n);
  for (int64_t q = 0; q < n; q++) qp[q] = po[q] + pl[q] - 1;
  return G4R_OK;
}

// the StDev and StBuf of a training batch: nb samples at plan slices (device) of P positions, one query each
static void st_train_batch(g4r_baselines* h, StDev& g, StBuf& B, const long long* ps, const int* pl, const int* po, const int* qp, int nb, int P) {
  g = StDev{};
  g.items = h->dNmItems; g.pstart = ps; g.plen = pl; g.poff = po; g.nb = nb; g.P = P;
  g.qs = po; g.qp = qp; g.nq = nb;
  g.E = h->dNmTh; g.d = h->n_keep; g.train = 1;
  g.PX = h->sg_i; g.PY = h->sg_i + h->sg_icap;
  st_carve(B, h->sg_f, h->nm_Pmax, h->nm_bs, h->n_keep, true);
}

extern "C" int g4r_bl_stamp_grads(g4r_baselines* h, const int32_t* samples, int32_t n, float* loss, float* grads) {
  if (!h) return G4R_ERR_INVALID;
  int rc = st_check_run(h, samples, n, "g4r_bl_stamp_grads");
  if (rc) return rc;
  if (n > h->nm_bs || !grads) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_grads: need n <= batch_size and grads");
  std::vector<long long> ps; std::vector<int> pl, po, qp; std::vector<std::pair<int64_t, int>> batches;
  rc = st_plan(h, samples, n, ps, pl, po, qp, batches, "g4r_bl_stamp_grads");
  if (rc) return rc;
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr, *dqp = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  CK(bb.put(&dqp, qp.data(), qp.size(), st));
  StDev g; StBuf B;
  st_train_batch(h, g, B, dps, dpl, dpo, dqp, n, batches[0].second);
  st_grad(st, g, B, h->nm_s, h->dNmTh, st_layout(h->n_items, h->n_keep), h->n_items, h->dNmG, h->dNmOne, h->dNmLoss);
  CK(cudaGetLastError());
  float l = 0.f;
  CK(cudaMemcpyAsync(&l, h->dNmLoss, sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(grads, h->dNmG, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (loss) *loss = l;
  return G4R_OK;
}

extern "C" int g4r_bl_stamp_epoch(g4r_baselines* h, const int32_t* order, int64_t n_order, float learning_rate, float* losses, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  int rc = st_check_run(h, order, n_order, "g4r_bl_stamp_epoch");
  if (rc) return rc;
  if (!(learning_rate > 0.f && std::isfinite(learning_rate))) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_epoch: learning_rate must be finite and > 0");
  std::vector<long long> ps; std::vector<int> pl, po, qp; std::vector<std::pair<int64_t, int>> batches;
  rc = st_plan(h, order, n_order, ps, pl, po, qp, batches, "g4r_bl_stamp_epoch");
  if (rc) return rc;
  if (h->nm_step + (int64_t)batches.size() > 0xffffffffll) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_epoch: more than 2^32 steps since the fit began");
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  const StLayout Lo = st_layout(h->n_items, h->n_keep);
  // the whole epoch's plan goes up once; each batch reads its slice
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr, *dqp = nullptr; float* dloss = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  CK(bb.put(&dqp, qp.data(), qp.size(), st));
  CK(bb.take(&dloss, batches.size()));
  CK(cudaEventRecord(h->ev0, st));
  for (size_t b = 0; b < batches.size(); b++) {
    const int64_t q0 = batches[b].first;
    StDev g; StBuf B;
    st_train_batch(h, g, B, dps + q0, dpl + q0, dpo + q0, dqp + q0, (int)std::min<int64_t>(h->nm_bs, n_order - q0), batches[b].second);
    st_grad(st, g, B, h->nm_s, h->dNmTh, Lo, h->n_items, h->dNmG, h->dNmOne, dloss + b);
    h->nm_step++;
    const double t = (double)h->nm_step;
    const float c1 = (float)(1.0 / (1.0 - std::pow(0.9, t))), c2 = (float)(1.0 / (1.0 - std::pow(0.999, t)));
    k_nm_adam<<<(unsigned)((Lo.n + 255) / 256), 256, 0, st>>>(h->dNmTh, h->dNmG, h->dNmM, h->dNmV, Lo.n, learning_rate, c1, c2);
  }
  const size_t nE = (size_t)h->n_items * h->n_keep;
  k_nm_to_double<<<(unsigned)((nE + 255) / 256), 256, 0, st>>>(h->dNmTh, nE, h->dI);
  CK(cudaGetLastError());
  CK(cudaEventRecord(h->ev1, st));
  if (losses) CK(cudaMemcpyAsync(losses, dloss, batches.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (device_ms) CK(cudaEventElapsedTime(device_ms, h->ev0, h->ev1));
  return G4R_OK;
}

// every counted event's q (the last max_len inputs of its prefix) into qev [n_ev x d] on the device, in NARM's evaluation chunks:
// a piece from a session's start serves every prefix it covers, one query per counted event at the prefix's last position
static int st_encode_events(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* off, int64_t n_sessions, const int32_t* n_history,
                            const std::vector<int64_t>& ev0, float* qev) {
  const int dd = h->n_keep;
  cudaStream_t st = h->stream;
  const StLayout Lo = st_layout(h->n_items, dd);
  BlBufs bb;
  long long* pstart = nullptr; int *plen = nullptr, *poff = nullptr, *qs = nullptr, *qp = nullptr, *row = nullptr, *px = nullptr;
  float* f = nullptr;
  const int* dItems = nullptr;
  CK(bb.take(&pstart, ST_EVAL_POS)); CK(bb.take(&plen, ST_EVAL_POS)); CK(bb.take(&poff, ST_EVAL_POS));
  CK(bb.take(&qs, ST_EVAL_POS)); CK(bb.take(&qp, ST_EVAL_POS)); CK(bb.take(&row, ST_EVAL_POS)); CK(bb.take(&px, ST_EVAL_POS));
  CK(bb.take(&f, (size_t)ST_EVAL_POS * (st_pos_floats(dd, false) + st_qry_floats(dd, false))));
  CK(bb.put(&dItems, items, n_events, st));
  StDev g{};
  g.items = dItems; g.pstart = pstart; g.plen = plen; g.poff = poff; g.qs = qs; g.qp = qp; g.E = h->dNmTh; g.d = dd; g.train = 0; g.PX = px;
  StBuf B;
  st_carve(B, f, ST_EVAL_POS, ST_EVAL_POS, dd, false);
  std::vector<int> qsh;
  auto flush = [&](const std::vector<long long>& ps, const std::vector<int>& pl, const std::vector<int>& po, const std::vector<int>& ev,
                   const std::vector<int>& pair, int P) -> int {
    const int nb = (int)ps.size(), nq = (int)ev.size();
    qsh.resize(nq);
    for (int e = 0, b = 0; e < nq; e++) {                // pairs rise with their pieces: each query's piece start
      while (po[b] + pl[b] <= pair[e]) b++;
      qsh[e] = po[b];
    }
    CK(cudaMemcpyAsync(pstart, ps.data(), nb * sizeof(long long), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(plen, pl.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(poff, po.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(qs, qsh.data(), nq * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(qp, pair.data(), nq * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(row, ev.data(), nq * sizeof(int), cudaMemcpyHostToDevice, st));
    g.nb = nb; g.P = P; g.nq = nq;
    st_encode(st, g, B, h->dNmTh, Lo, row, qev);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));                      // the host arrays are reused by the next chunk
    return G4R_OK;
  };
  return nm_event_chunks(h->nm_len, ST_EVAL_POS, off, n_sessions, n_history, ev0, flush);
}

extern "C" int g4r_bl_stamp_encode(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                                   const int32_t* n_history, float* q, int64_t n_q) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_STAMP || !h->ready) FAIL(G4R_ERR_STATE, "g4r_bl_stamp_encode: no STAMP parameters (g4r_bl_stamp_begin or g4r_bl_stamp_import)");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || n_q < 0 || (n_q > 0 && !q))
    FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_encode: null or out-of-range argument");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_encode: session offsets must rise from 0 to n_events");
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= h->n_items) FAIL(G4R_ERR_INDEX, "g4r_bl_stamp_encode: item index out of range");
  std::vector<int64_t> ev0;
  int rc = bl_counted(h, "g4r_bl_stamp_encode", session_offsets, n_sessions, n_history, ev0);
  if (rc) return rc;
  if (n_q != ev0[n_sessions]) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_encode: n_q must be the number of counted events");
  if (n_q > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_stamp_encode: more than 2^31 - 1 counted events");
  cudaSetDevice(h->device);
  BlBufs bb;
  float* dq = nullptr;
  CK(bb.take(&dq, (size_t)n_q * h->n_keep));
  rc = st_encode_events(h, items, n_events, session_offsets, n_sessions, n_history, ev0, dq);
  if (rc) return rc;
  if (n_q) CK(cudaMemcpyAsync(q, dq, (size_t)n_q * h->n_keep * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// the ranking of a g4r_bl_evaluate call of a STAMP: every counted event's q, then BPR's ranking with I = double(E), bI = 0
static int stamp_rank(g4r_baselines* h, BlCall& c) {
  float* dq = nullptr;
  CK(c.bb.take(&dq, (size_t)c.n_ev * h->n_keep));
  const int rc = st_encode_events(h, c.items, c.n_events, c.off, c.n_sessions, c.n_history, c.ev0, dq);
  if (rc) return rc;
  return bpr_blocks(h, c, dq);
}
