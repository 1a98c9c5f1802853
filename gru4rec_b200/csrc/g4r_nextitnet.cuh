// g4r_nextitnet.cuh -- the NextItNet convolutional baseline on the device (DESIGN §3w): the input embedding, a stack of residual
// blocks of two dilated causal 1-D convolutions (dilation l, then 2 l), each followed by a layer norm and a ReLU, and an output
// item table with a bias, trained with full-catalogue cross-entropy and NARM's dense Adam; and the eval-mode encoder that feeds
// per-event vectors to BPR's ranking.  A convolution is a causal gather of its K taps (k_ni_im2col) and one product with the
// kernel through NARM's k_nm_gemm; its input gradient is the gather's transpose read as a gather-sum (k_ni_col2im), so no
// reduction here uses floating-point atomics and a fit is bitwise reproducible.  Layer norms are SASRec's, the loss NARM's, the
// input-embedding gradient NARM's key sort and scatter, the training plan and the evaluation chunk planner NARM's.  A NextItNet
// handle keeps its model in the handle's NARM fields.  Included at the end of g4r_lib.cu after g4r_sasrec.cuh.
#pragma once

constexpr int NI_D_MAX = 1024, NI_K_MAX = 8, NI_BLOCKS_MAX = 16, NI_DIL_MAX = 256, NI_LEN_MAX = 512;
constexpr int NI_EVAL_PAIRS = 16384;                   // encoder positions (and pieces) per evaluation chunk

// offsets of the parameters in the flat float32 vector: E, per block (C1, c1, g1, n1, C2, c2, g2, n2), W, bW
struct NiLayout {
  size_t E, blk0, blk_n, W, bW, n;
};
static NiLayout ni_layout(int NI, int d, int K, int blocks) {
  NiLayout L;
  const size_t D = d;
  L.E = 0; L.blk0 = (size_t)NI * D; L.blk_n = 2 * (size_t)K * D * D + 6 * D;
  L.W = L.blk0 + (size_t)blocks * L.blk_n; L.bW = L.W + (size_t)NI * D; L.n = L.bW + NI;
  return L;
}
struct NiBlk {
  size_t C1, c1, g1, n1, C2, c2, g2, n2;
};
static NiBlk ni_blk(const NiLayout& L, int b, int d, int K) {
  const size_t D = d, KDD = (size_t)K * D * D;
  size_t o = L.blk0 + (size_t)b * L.blk_n;
  NiBlk k;
  k.C1 = o; o += KDD; k.c1 = o; o += D; k.g1 = o; o += D; k.n1 = o; o += D;
  k.C2 = o; o += KDD; k.c2 = o; o += D; k.g2 = o; o += D; k.n2 = o;
  return k;
}

// one mini-batch (or evaluation chunk) of nb pieces: slot b holds the plen[b] inputs items[pstart[b] ..], its positions are
// poff[b] .. poff[b] + plen[b] - 1, PS[p] = slot * L + t; a training piece's targets follow its inputs
struct NiDev {
  const int* items; const long long* pstart; const int* plen; const int* poff; int nb, P;
  const float* E;
  int d, L, K;                                           // width, max_len (the PS stride), kernel size
  int train;
  int* PX; int* PY; int* PS;
};

// CTA per slot: positions, targets, PS rows and h0 = E[x]
__global__ void __launch_bounds__(256) k_ni_embed(NiDev s, float* H0) {
  const int b = blockIdx.x, n = s.plen[b], p0 = s.poff[b];
  const long long s0 = s.pstart[b];
  for (int x = threadIdx.x; x < n * s.d; x += blockDim.x) {
    const int t = x / s.d, u = x % s.d, p = p0 + t, it = s.items[s0 + t];
    if (u == 0) { s.PX[p] = it; s.PY[p] = s.train ? s.items[s0 + t + 1] : -1; s.PS[p] = b * s.L + t; }
    H0[(size_t)p * s.d + u] = s.E[(size_t)it * s.d + u];
  }
}

// the causal gather of a convolution of dilation l: COL [P x K d], COL[p][k d + i] = X[p - (K - 1 - k) l][i], 0 where that
// position lies before the piece's start
__global__ void k_ni_im2col(NiDev s, const float* X, int l, float* COL) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x, w = (long long)s.K * s.d;
  if (x >= (long long)s.P * w) return;
  const int p = (int)(x / w), r = (int)(x % w), k = r / s.d, i = r % s.d;
  const int back = (s.K - 1 - k) * l, t = s.PS[p] % s.L;
  COL[x] = t >= back ? X[(size_t)(p - back) * s.d + i] : 0.f;
}

// the gather's transpose as a gather-sum: OUT[p][i] = (RES[p][i] +) sum over k in order of DCOL[p + (K - 1 - k) l][k d + i],
// the taps past the piece's end 0.  OUT may be RES.
__global__ void k_ni_col2im(NiDev s, const float* DCOL, int l, const float* RES, float* OUT) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (long long)s.P * s.d) return;
  const int p = (int)(x / s.d), i = (int)(x % s.d), t = s.PS[p] % s.L, n = s.plen[s.PS[p] / s.L];
  const size_t w = (size_t)s.K * s.d;
  float a = 0.f;
  for (int k = 0; k < s.K; k++) {
    const int fwd = (s.K - 1 - k) * l;
    if (t + fwd < n) a = __fadd_rn(a, DCOL[(size_t)(p + fwd) * w + (size_t)k * s.d + i]);
  }
  OUT[x] = RES ? __fadd_rn(RES[x], a) : a;
}

// OUT = (HIN +) relu(Y); OUT may be Y or HIN
__global__ void k_ni_relu(const float* Y, const float* HIN, float* OUT, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float r = fmaxf(Y[i], 0.f);
  OUT[i] = HIN ? __fadd_rn(HIN[i], r) : r;
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
// the per-position float arrays of P positions.  Training keeps every block's activations (blocks + 1 residual streams, the last
// one q); evaluation keeps one block's and one stream, updated in place, and carries no backward buffers.  The gathered taps
// (COL) are recomputed in the backward rather than kept per block.
struct NiBuf {
  long long P = 0; bool keep = false;
  float *H, *U, *A, *V, *Y, *MU1, *RS1, *MU2, *RS2;      // per block (H: per stream)
  float *COL;                                            // one convolution's taps [P x K d]
  float *LOSS, *DH, *T, *DX, *DY, *DYX, *DCOL;           // the backward
  float* at(float* base, int width, int blk) const { return keep ? base + (size_t)blk * P * width : base; }
};
static size_t ni_pos_floats(int d, int K, int blocks, bool train) {
  const size_t D = d, nb = train ? blocks : 1;
  size_t f = (nb + (train ? 1 : 0)) * D + nb * (4 * D + 4) + (size_t)K * D;
  if (train) f += 1 + 5 * D + (size_t)K * D;
  return f;
}
static void ni_carve(NiBuf& B, float* f, long long P, int d, int K, int blocks, bool train) {
  B.P = P; B.keep = train;
  const size_t nb = train ? blocks : 1;
  auto take = [&](float** q, size_t w) { *q = f; f += (size_t)P * w; };
  take(&B.H, (nb + (train ? 1 : 0)) * d);
  take(&B.U, nb * d); take(&B.A, nb * d); take(&B.V, nb * d); take(&B.Y, nb * d);
  take(&B.MU1, nb); take(&B.RS1, nb); take(&B.MU2, nb); take(&B.RS2, nb);
  take(&B.COL, (size_t)K * d);
  if (!train) return;
  take(&B.LOSS, 1); take(&B.DH, d); take(&B.T, d); take(&B.DX, d); take(&B.DY, d); take(&B.DYX, d); take(&B.DCOL, (size_t)K * d);
}

static unsigned ni_grid(long long n) { return (unsigned)((n + 255) / 256); }

// the encoder of a batch or chunk: q = the last stream of B.H [P x d] (part: split scratch; encoder products never split)
static void ni_encode(cudaStream_t st, const NiDev& s, const NiBuf& B, const float* th, const NiLayout& Lo, const std::vector<int>& dil, float* part) {
  const int P = s.P, d = s.d, K = s.K, blocks = (int)dil.size();
  const long long n = (long long)P * d, nc = n * K;
  const unsigned gl = (unsigned)((P + 7) / 8), ge = ni_grid(n), gc = ni_grid(nc);
  k_ni_embed<<<s.nb, 256, 0, st>>>(s, B.at(B.H, d, 0));
  for (int b = 0; b < blocks; b++) {
    const NiBlk k = ni_blk(Lo, b, d, K);
    const int l = dil[b];
    float *hin = B.at(B.H, d, b), *u = B.at(B.U, d, b), *a = B.at(B.A, d, b), *v = B.at(B.V, d, b), *y = B.at(B.Y, d, b), *hout = B.at(B.H, d, b + 1);
    k_ni_im2col<<<gc, 256, 0, st>>>(s, hin, l, B.COL);
    nm_gemm<NM_ENCODER>(st, part, B.COL, (long long)K * d, 1, th + k.C1, d, 1, u, d, P, d, K * d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(u, th + k.c1, n, d);
    k_sa_ln<<<gl, 256, 0, st>>>(u, th + k.g1, th + k.n1, P, d, a, B.at(B.MU1, 1, b), B.at(B.RS1, 1, b));
    k_ni_relu<<<ge, 256, 0, st>>>(a, nullptr, a, n);
    k_ni_im2col<<<gc, 256, 0, st>>>(s, a, 2 * l, B.COL);
    nm_gemm<NM_ENCODER>(st, part, B.COL, (long long)K * d, 1, th + k.C2, d, 1, v, d, P, d, K * d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(v, th + k.c2, n, d);
    k_sa_ln<<<gl, 256, 0, st>>>(v, th + k.g2, th + k.n2, P, d, y, B.at(B.MU2, 1, b), B.at(B.RS2, 1, b));
    k_ni_relu<<<ge, 256, 0, st>>>(y, hin, hout, n);
  }
}

// a batch's loss and gradient G (flat, the parameters' layout) at the handle's parameters; loss_out a device float
static void ni_grad(cudaStream_t st, const NiDev& s, const NiBuf& B, const NmScratch& ns, const float* th, const NiLayout& Lo, const std::vector<int>& dil,
                    int NI, float* G, const float* ones, float* loss_out) {
  const int P = s.P, d = s.d, K = s.K, blocks = (int)dil.size();
  const long long n = (long long)P * d, nc = n * K;
  const unsigned gl = (unsigned)((P + 7) / 8), ge = ni_grid(n), gc = ni_grid(nc);
  float* part = ns.part;
  ni_encode(st, s, B, th, Lo, dil, part);
  const float* Q = B.at(B.H, d, blocks);
  // the catalogue: logits Q W^T + bW, the softmax gradient, dL/dq, dW and dbW
  NmDev nd{};
  nd.P = P; nd.d = d; nd.NI = NI; nd.S = ns.S; nd.PY = s.PY; nd.PX = s.PX; nd.PS = s.PS; nd.LOSS = B.LOSS; nd.re = 1.f;
  const float* W = th + Lo.W;
  nm_gemm<NM_CATALOGUE>(st, part, Q, d, 1, W, 1, d, ns.S, NI, P, NI, d);
  k_sa_bias<false><<<ni_grid((long long)P * NI), 256, 0, st>>>(ns.S, th + Lo.bW, (long long)P * NI, NI);
  k_nm_softmax<<<P, 256, 0, st>>>(nd);
  k_nm_mean<<<1, 1024, 0, st>>>(B.LOSS, P, loss_out);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, NI, 1, W, d, 1, B.DH, d, P, d, NI);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, 1, NI, Q, d, 1, G + Lo.W, d, NI, d, P);
  sa_colsum(st, part, ones, ns.S, G + Lo.bW, P, NI);
  for (int b = blocks - 1; b >= 0; b--) {
    const NiBlk k = ni_blk(Lo, b, d, K);
    const int l = dil[b];
    float *hin = B.at(B.H, d, b), *u = B.at(B.U, d, b), *a = B.at(B.A, d, b), *v = B.at(B.V, d, b), *y = B.at(B.Y, d, b);
    // h' = h + relu(LN2(v)): T = dh' where the ReLU passed, DX = dL/dv
    cudaMemcpyAsync(B.T, B.DH, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    k_sa_relu_bwd<<<ge, 256, 0, st>>>(B.T, y, n);
    k_sa_ln_bwd<<<gl, 256, 0, st>>>(v, B.at(B.MU2, 1, b), B.at(B.RS2, 1, b), th + k.g2, B.T, nullptr, nullptr, nullptr, P, d, B.DX, B.DY, B.DYX);
    sa_colsum(st, part, ones, B.DYX, G + k.g2, P, d);
    sa_colsum(st, part, ones, B.DY, G + k.n2, P, d);
    // v = c2 + taps(a, 2 l) C2: dC2 = COL^T DX, dc2 = 1^T DX, dCOL = DX C2^T and da its gather-sum
    k_ni_im2col<<<gc, 256, 0, st>>>(s, a, 2 * l, B.COL);
    nm_gemm<NM_BACKWARD>(st, part, B.COL, 1, (long long)K * d, B.DX, d, 1, G + k.C2, d, K * d, d, P);
    sa_colsum(st, part, ones, B.DX, G + k.c2, P, d);
    nm_gemm<NM_BACKWARD>(st, part, B.DX, d, 1, th + k.C2, 1, d, B.DCOL, (long long)K * d, P, K * d, d);
    k_ni_col2im<<<ge, 256, 0, st>>>(s, B.DCOL, 2 * l, nullptr, B.T);
    // a = relu(LN1(u))
    k_sa_relu_bwd<<<ge, 256, 0, st>>>(B.T, a, n);
    k_sa_ln_bwd<<<gl, 256, 0, st>>>(u, B.at(B.MU1, 1, b), B.at(B.RS1, 1, b), th + k.g1, B.T, nullptr, nullptr, nullptr, P, d, B.DX, B.DY, B.DYX);
    sa_colsum(st, part, ones, B.DYX, G + k.g1, P, d);
    sa_colsum(st, part, ones, B.DY, G + k.n1, P, d);
    // u = c1 + taps(h, l) C1; dh += the gather-sum of dCOL
    k_ni_im2col<<<gc, 256, 0, st>>>(s, hin, l, B.COL);
    nm_gemm<NM_BACKWARD>(st, part, B.COL, 1, (long long)K * d, B.DX, d, 1, G + k.C1, d, K * d, d, P);
    sa_colsum(st, part, ones, B.DX, G + k.c1, P, d);
    nm_gemm<NM_BACKWARD>(st, part, B.DX, d, 1, th + k.C1, 1, d, B.DCOL, (long long)K * d, P, K * d, d);
    k_ni_col2im<<<ge, 256, 0, st>>>(s, B.DCOL, l, B.DH, B.DH);
  }
  // h0 = E[x]: the input embedding's rows by NARM's sort and scatter (E has no other gradient)
  cudaMemsetAsync(G + Lo.E, 0, (size_t)NI * d * sizeof(float), st);
  nd.DEMB = B.DH;
  k_nm_keys<<<(P + 255) / 256, 256, 0, st>>>(s.PX, P, ns.keys);
  int end_bit = 33;
  while (end_bit < 64 && ((unsigned long long)NI >> (end_bit - 32)) != 0ull) end_bit++;
  size_t cb = ns.cub_bytes;
  cub::DeviceRadixSort::SortKeys(ns.cub, cb, ns.keys, ns.keys2, P, 0, end_bit, st);
  k_nm_scatter<<<ni_grid(n), 256, 0, st>>>(nd, ns.keys2, G + Lo.E);
}

static bool ni_shape_ok(int d, const int32_t* dil, int n_dil, int K, int len) {
  if (d < 1 || d > NI_D_MAX || !dil || n_dil < 1 || n_dil > NI_BLOCKS_MAX || K < 1 || K > NI_K_MAX || len < 1 || len > NI_LEN_MAX) return false;
  for (int b = 0; b < n_dil; b++) if (dil[b] < 1 || dil[b] > NI_DIL_MAX) return false;
  return true;
}
#define NI_SHAPE_MSG ": need 1 .. 16 dilations, each in 1 .. 256, kernel_size in 1 .. 8 and max_len in 1 .. 512"

// dI = double(W) and dBI = double(bW), the item side bpr_blocks ranks against; after every epoch and every import
static cudaError_t ni_refresh(g4r_baselines* h, const NiLayout& L) {
  const size_t nW = (size_t)h->n_items * h->n_keep;
  k_nm_to_double<<<(unsigned)((nW + 255) / 256), 256, 0, h->stream>>>(h->dNmTh + L.W, nW, h->dI);
  k_nm_to_double<<<(unsigned)((h->n_items + 255) / 256), 256, 0, h->stream>>>(h->dNmTh + L.bW, (size_t)h->n_items, h->dBI);
  return cudaGetLastError();
}

// the model buffers of a NextItNet handle (NARM's fields): parameters, double(W) and double(bW) for bpr_blocks, a device 1.0f
static int ni_set_model(g4r_baselines* h, const int32_t* dil, int32_t n_dil, int32_t K, int32_t max_len, const float* params, int64_t n_params,
                        const char* who) {
  if (!params) FAIL(G4R_ERR_INVALID, std::string(who) + ": null parameters");
  if (!ni_shape_ok(h->n_keep, dil, n_dil, K, max_len)) FAIL(G4R_ERR_INVALID, std::string(who) + NI_SHAPE_MSG);
  const NiLayout L = ni_layout(h->n_items, h->n_keep, K, n_dil);
  if (n_params != (int64_t)L.n)
    FAIL(G4R_ERR_INVALID, std::string(who) + ": need n_params = 2 n_items d + n_items + n_dilations (2 kernel_size d^2 + 6 d) = " + std::to_string(L.n));
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
  h->ni_dil.assign(dil, dil + n_dil); h->ni_K = K; h->nm_len = max_len; h->nm_n = L.n;
  CK(ni_refresh(h, L));
  CK(cudaStreamSynchronize(st));
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_nextitnet_import(g4r_baselines* h, const int32_t* dilations, int32_t n_dilations, int32_t kernel_size, int32_t max_len,
                                       const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NEXTITNET) FAIL(G4R_ERR_STATE, "g4r_bl_nextitnet_import: the handle is not a NextItNet");
  return ni_set_model(h, dilations, n_dilations, kernel_size, max_len, params, n_params, "g4r_bl_nextitnet_import");
}

extern "C" int g4r_bl_nextitnet_export(g4r_baselines* h, float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NEXTITNET || !h->dNmTh)
    FAIL(G4R_ERR_STATE, "g4r_bl_nextitnet_export: no NextItNet parameters (g4r_bl_nextitnet_begin or g4r_bl_nextitnet_import)");
  if (!params || n_params != (int64_t)h->nm_n) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_export: need n_params floats");
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(params, h->dNmTh, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

extern "C" int g4r_bl_nextitnet_begin(g4r_baselines* h, const int32_t* dilations, int32_t n_dilations, int32_t kernel_size, int32_t max_len,
                                      int32_t batch_size, const int64_t* piece_offsets, int64_t n_pieces, const int32_t* items, int64_t n_entries,
                                      const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NEXTITNET) FAIL(G4R_ERR_STATE, "g4r_bl_nextitnet_begin: the handle is not a NextItNet");
  if (!piece_offsets || !items || n_pieces < 1 || n_entries < 2 || batch_size < 1)
    FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_begin: null argument, no pieces or batch_size < 1");
  const int NI = h->n_items, dd = h->n_keep;
  if (!ni_shape_ok(dd, dilations, n_dilations, kernel_size, max_len)) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_begin" NI_SHAPE_MSG);
  if (n_entries > INT32_MAX || n_pieces > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_begin: more than 2^31 - 1 entries or pieces");
  if (piece_offsets[0] != 0 || piece_offsets[n_pieces] != n_entries) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_begin: piece offsets must run from 0 to n_entries");
  std::vector<int> lens(n_pieces);
  for (int64_t k = 0; k < n_pieces; k++) {
    const int64_t n = piece_offsets[k + 1] - piece_offsets[k];
    if (n < 2 || n > (int64_t)max_len + 1) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_begin: every piece needs 2 .. max_len + 1 events");
    lens[k] = (int)n - 1;
  }
  for (int64_t e = 0; e < n_entries; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_nextitnet_begin: item index out of range");
  // the largest batch: the batch_size longest pieces
  std::vector<int> srt(lens);
  std::sort(srt.begin(), srt.end(), std::greater<int>());
  long long Pmax = 0;
  for (int64_t k = 0; k < std::min<int64_t>(batch_size, n_pieces); k++) Pmax += srt[k];
  const NiLayout L = ni_layout(NI, dd, kernel_size, n_dilations);
  const size_t act = (size_t)Pmax * ni_pos_floats(dd, kernel_size, n_dilations, true) * 4;
  const size_t need = (size_t)Pmax * ((size_t)NI * 4 + 28) + act + NM_PART_CAP * 4 + 3 * L.n * 4 + (size_t)n_entries * 4 + (size_t)n_pieces * 16 +
                      ((size_t)64 << 20);
  int rc = ni_set_model(h, dilations, n_dilations, kernel_size, max_len, params, n_params, "g4r_bl_nextitnet_begin");
  if (rc) return rc;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    h->err = "g4r_bl_nextitnet_begin: the fit needs " + std::to_string(need) + " bytes of device memory (the logits of the largest batch " +
             std::to_string((size_t)Pmax * NI * 4) + ", its activations " + std::to_string(act) + "), " + std::to_string(free_b) + " are free";
    return G4R_ERR_CUDA;
  }
  cudaStream_t st = h->stream;
  h->ready = false;
  auto take = [&](auto** p, size_t n) { return nm_take(h, p, n); };
  NmScratch& s = h->nm_s;
  s = NmScratch{};
  size_t cb = 0;
  CK(cub::DeviceRadixSort::SortKeys(nullptr, cb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)Pmax, 0, 64));
  CK(take(&s.PX, Pmax)); CK(take(&s.PY, Pmax)); CK(take(&s.PS, Pmax)); CK(take(&s.part, NM_PART_CAP));
  CK(take(&s.pstart, batch_size)); CK(take(&s.plen, batch_size)); CK(take(&s.poff, batch_size));
  CK(take(&s.S, (size_t)Pmax * NI)); CK(take(&s.keys, Pmax)); CK(take(&s.keys2, Pmax)); CK(take(&s.cub, cb));
  s.cub_bytes = cb;
  CK(take(&h->ni_f, (size_t)Pmax * ni_pos_floats(dd, kernel_size, n_dilations, true)));
  CK(nm_take(h, &h->dNmG, L.n)); CK(nm_take(h, &h->dNmM, L.n)); CK(nm_take(h, &h->dNmV, L.n)); CK(nm_take(h, &h->dNmItems, n_entries));
  CK(nm_take(h, &h->dNmLoss, 1));
  CK(cudaMemsetAsync(h->dNmM, 0, L.n * sizeof(float), st)); CK(cudaMemsetAsync(h->dNmV, 0, L.n * sizeof(float), st));
  CK(cudaMemcpyAsync(h->dNmItems, items, n_entries * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  h->nm_off.assign(piece_offsets, piece_offsets + n_pieces + 1);
  h->nm_bs = batch_size; h->nm_Pmax = Pmax; h->nm_step = 0; h->nm_fit = true;
  h->ready = true;
  return G4R_OK;
}

// the NiDev of a handle's parameters (plan pointers and nb / P set by the caller)
static NiDev ni_dev(const g4r_baselines* h, const NiLayout& Lo) {
  NiDev s{};
  s.E = h->dNmTh + Lo.E; s.d = h->n_keep; s.L = h->nm_len; s.K = h->ni_K;
  return s;
}

static NiDev ni_train_dev(g4r_baselines* h, const NiLayout& Lo) {
  NiDev s = ni_dev(h, Lo);
  const NmScratch& ns = h->nm_s;
  s.items = h->dNmItems; s.train = 1;
  s.PX = ns.PX; s.PY = ns.PY; s.PS = ns.PS; s.pstart = ns.pstart; s.plen = ns.plen; s.poff = ns.poff;
  return s;
}

static NiLayout ni_handle_layout(const g4r_baselines* h) { return ni_layout(h->n_items, h->n_keep, h->ni_K, (int)h->ni_dil.size()); }

static int ni_check_run(g4r_baselines* h, const int32_t* pieces, int64_t n, const char* who) {
  if (h->kind != BL_NEXTITNET) FAIL(G4R_ERR_STATE, std::string(who) + ": the handle is not a NextItNet");
  if (!h->nm_fit) FAIL(G4R_ERR_STATE, std::string(who) + ": no fit begun (g4r_bl_nextitnet_begin)");
  if (!pieces || n < 1) FAIL(G4R_ERR_INVALID, std::string(who) + ": no pieces");
  const int64_t np = (int64_t)h->nm_off.size() - 1;
  for (int64_t q = 0; q < n; q++) if (pieces[q] < 0 || pieces[q] >= np) FAIL(G4R_ERR_INDEX, std::string(who) + ": piece index out of range");
  return G4R_OK;
}

extern "C" int g4r_bl_nextitnet_grads(g4r_baselines* h, const int32_t* pieces, int32_t n, float* loss, float* grads) {
  if (!h) return G4R_ERR_INVALID;
  int rc = ni_check_run(h, pieces, n, "g4r_bl_nextitnet_grads");
  if (rc) return rc;
  if (n > h->nm_bs || !grads) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_grads: need n <= batch_size and grads");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = nm_plan(h, pieces, n, ps, pl, po, batches, "g4r_bl_nextitnet_grads");
  if (rc) return rc;
  cudaSetDevice(h->device);
  rc = nm_upload_plan(h, ps, pl, po, 0, n);
  if (rc) return rc;
  const NiLayout Lo = ni_handle_layout(h);
  NiDev s = ni_train_dev(h, Lo);
  s.nb = n; s.P = batches[0].second;
  NiBuf B;
  ni_carve(B, h->ni_f, h->nm_Pmax, h->n_keep, h->ni_K, (int)h->ni_dil.size(), true);
  ni_grad(h->stream, s, B, h->nm_s, h->dNmTh, Lo, h->ni_dil, h->n_items, h->dNmG, h->dNmOne, h->dNmLoss);
  CK(cudaGetLastError());
  float l = 0.f;
  CK(cudaMemcpyAsync(&l, h->dNmLoss, sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(grads, h->dNmG, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (loss) *loss = l;
  return G4R_OK;
}

extern "C" int g4r_bl_nextitnet_epoch(g4r_baselines* h, const int32_t* order, int64_t n_order, float learning_rate, float* losses, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  int rc = ni_check_run(h, order, n_order, "g4r_bl_nextitnet_epoch");
  if (rc) return rc;
  if (!(learning_rate > 0.f && std::isfinite(learning_rate))) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_epoch: learning_rate must be finite and > 0");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = nm_plan(h, order, n_order, ps, pl, po, batches, "g4r_bl_nextitnet_epoch");
  if (rc) return rc;
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  const NiLayout Lo = ni_handle_layout(h);
  NiBuf B;
  ni_carve(B, h->ni_f, h->nm_Pmax, h->n_keep, h->ni_K, (int)h->ni_dil.size(), true);
  // the whole epoch's plan goes up once; each batch reads its slice
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr; float* dloss = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  CK(bb.take(&dloss, batches.size()));
  CK(cudaEventRecord(h->ev0, st));
  for (size_t b = 0; b < batches.size(); b++) {
    const int64_t q0 = batches[b].first;
    NiDev s = ni_train_dev(h, Lo);
    s.pstart = dps + q0; s.plen = dpl + q0; s.poff = dpo + q0; s.nb = (int)std::min<int64_t>(h->nm_bs, n_order - q0); s.P = batches[b].second;
    ni_grad(st, s, B, h->nm_s, h->dNmTh, Lo, h->ni_dil, h->n_items, h->dNmG, h->dNmOne, dloss + b);
    h->nm_step++;
    const double t = (double)h->nm_step;
    const float c1 = (float)(1.0 / (1.0 - std::pow(0.9, t))), c2 = (float)(1.0 / (1.0 - std::pow(0.999, t)));
    k_nm_adam<<<(unsigned)((Lo.n + 255) / 256), 256, 0, st>>>(h->dNmTh, h->dNmG, h->dNmM, h->dNmV, Lo.n, learning_rate, c1, c2);
  }
  CK(ni_refresh(h, Lo));
  CK(cudaEventRecord(h->ev1, st));
  if (losses) CK(cudaMemcpyAsync(losses, dloss, batches.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (device_ms) CK(cudaEventElapsedTime(device_ms, h->ev0, h->ev1));
  return G4R_OK;
}

// every counted event's q (the last max_len inputs of its prefix) into qev [n_ev x d] on the device
static int ni_encode_events(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* off, int64_t n_sessions, const int32_t* n_history,
                            const std::vector<int64_t>& ev0, float* qev) {
  const int dd = h->n_keep, K = h->ni_K;
  cudaStream_t st = h->stream;
  const NiLayout Lo = ni_handle_layout(h);
  BlBufs bb;
  int *PX = nullptr, *PY = nullptr, *PS = nullptr, *dEv = nullptr, *dPair = nullptr, *plen = nullptr, *poff = nullptr;
  long long* pstart = nullptr;
  float *f = nullptr, *part = nullptr;
  const int* dItems = nullptr;
  CK(bb.take(&PX, NI_EVAL_PAIRS)); CK(bb.take(&PY, NI_EVAL_PAIRS)); CK(bb.take(&PS, NI_EVAL_PAIRS));
  CK(bb.take(&dEv, NI_EVAL_PAIRS)); CK(bb.take(&dPair, NI_EVAL_PAIRS));
  CK(bb.take(&pstart, NI_EVAL_PAIRS)); CK(bb.take(&plen, NI_EVAL_PAIRS)); CK(bb.take(&poff, NI_EVAL_PAIRS));
  CK(bb.take(&f, (size_t)NI_EVAL_PAIRS * ni_pos_floats(dd, K, (int)h->ni_dil.size(), false)));
  CK(bb.put(&dItems, items, n_events, st));
  NiBuf B;
  ni_carve(B, f, NI_EVAL_PAIRS, dd, K, (int)h->ni_dil.size(), false);
  NiDev s = ni_dev(h, Lo);
  s.items = dItems; s.train = 0; s.PX = PX; s.PY = PY; s.PS = PS; s.pstart = pstart; s.plen = plen; s.poff = poff;
  auto flush = [&](const std::vector<long long>& ps, const std::vector<int>& pl, const std::vector<int>& po, const std::vector<int>& ev,
                   const std::vector<int>& pair, int P) -> int {
    const int nb = (int)ps.size();
    CK(cudaMemcpyAsync(pstart, ps.data(), nb * sizeof(long long), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(plen, pl.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(poff, po.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dEv, ev.data(), ev.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dPair, pair.data(), pair.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    s.nb = nb; s.P = P;
    ni_encode(st, s, B, h->dNmTh, Lo, h->ni_dil, part);
    const int ne = (int)ev.size();
    k_nm_pick<<<(unsigned)(((long long)ne * dd + 255) / 256), 256, 0, st>>>(B.H, dEv, dPair, ne, dd, qev);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));                      // the host arrays are reused by the next chunk
    return G4R_OK;
  };
  return nm_event_chunks(h->nm_len, NI_EVAL_PAIRS, off, n_sessions, n_history, ev0, flush);
}

extern "C" int g4r_bl_nextitnet_encode(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                                       const int32_t* n_history, float* q, int64_t n_q) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NEXTITNET || !h->ready)
    FAIL(G4R_ERR_STATE, "g4r_bl_nextitnet_encode: no NextItNet parameters (g4r_bl_nextitnet_begin or g4r_bl_nextitnet_import)");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || n_q < 0 || (n_q > 0 && !q))
    FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_encode: null or out-of-range argument");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_encode: session offsets must rise from 0 to n_events");
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= h->n_items) FAIL(G4R_ERR_INDEX, "g4r_bl_nextitnet_encode: item index out of range");
  std::vector<int64_t> ev0;
  int rc = bl_counted(h, "g4r_bl_nextitnet_encode", session_offsets, n_sessions, n_history, ev0);
  if (rc) return rc;
  if (n_q != ev0[n_sessions]) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_encode: n_q must be the number of counted events");
  if (n_q > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_nextitnet_encode: more than 2^31 - 1 counted events");
  cudaSetDevice(h->device);
  BlBufs bb;
  float* dq = nullptr;
  CK(bb.take(&dq, (size_t)n_q * h->n_keep));
  rc = ni_encode_events(h, items, n_events, session_offsets, n_sessions, n_history, ev0, dq);
  if (rc) return rc;
  if (n_q) CK(cudaMemcpyAsync(q, dq, (size_t)n_q * h->n_keep * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// the ranking of a g4r_bl_evaluate call of a NextItNet: every counted event's q, then BPR's ranking with I = double(W),
// bI = double(bW)
static int nextitnet_rank(g4r_baselines* h, BlCall& c) {
  float* dq = nullptr;
  CK(c.bb.take(&dq, (size_t)c.n_ev * h->n_keep));
  const int rc = ni_encode_events(h, c.items, c.n_events, c.off, c.n_sessions, c.n_history, c.ev0, dq);
  if (rc) return rc;
  return bpr_blocks(h, c, dq);
}
