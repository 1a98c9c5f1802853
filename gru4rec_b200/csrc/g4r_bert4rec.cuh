// g4r_bert4rec.cuh -- the BERT4Rec bidirectional baseline on the device (DESIGN §3x): learned positions over an item table with a
// mask row, an embedding layer norm, a stack of post-LN Transformer blocks (bidirectional multi-head attention and a position-wise
// GELU FFN), a GELU / layer-norm head and an output bias, trained by the cloze objective (full-catalogue cross-entropy over the
// masked positions only) with NARM's dense Adam; and the eval-mode encoder that feeds per-event vectors (a window of the prefix
// followed by the mask token) to BPR's ranking.  Every product runs through NARM's k_nm_gemm, the catalogue loss through
// k_nm_softmax, the input-embedding gradient (the mask row included) through k_nm_keys / k_nm_scatter; layer norms, residual
// branches and dropout are SASRec's kernels.  Every reduction here runs in a fixed order (no floating-point atomics), so a fit is
// bitwise reproducible.  A BERT4Rec handle keeps its model and fit in the handle's NARM fields and its n_blocks / n_heads in
// SASRec's.  Included at the end of g4r_lib.cu after g4r_nextitnet.cuh.
#pragma once

constexpr int B4_D_MAX = 1024, B4_BLOCKS_MAX = 8, B4_LEN_MAX = 512;
constexpr int B4_ATT_THREADS = 128;                    // attention CTA: more keys than this, or a wider head, loops per thread
constexpr int B4_EVAL_POS = 16384;                     // encoder positions per evaluation chunk
constexpr unsigned B4_STREAM_H0 = 220u, B4_STREAM_ATT = 221u, B4_STREAM_FFN = 222u;   // dropout streams

// offsets of the parameters in the flat float32 vector: E (n_items + 1 rows, the last the mask token), Pe, g0, c0, per block (Wq,
// bq, Wk, bk, Wv, bv, Wo, bo, g1, c1, W1 [d x 4d], b1 [4d], W2 [4d x d], b2, g2, c2), Wp, bp, gp, cp, bO [n_items]
struct B4Layout {
  size_t E, Pe, g0, c0, blk0, blk_n, Wp, bp, gp, cp, bO, n;
};
static B4Layout b4_layout(int NI, int d, int n_blocks, int len) {
  B4Layout L;
  const size_t D = d;
  L.E = 0; L.Pe = ((size_t)NI + 1) * D; L.g0 = L.Pe + (size_t)len * D; L.c0 = L.g0 + D; L.blk0 = L.c0 + D; L.blk_n = 12 * D * D + 13 * D;
  L.Wp = L.blk0 + (size_t)n_blocks * L.blk_n; L.bp = L.Wp + D * D; L.gp = L.bp + D; L.cp = L.gp + D; L.bO = L.cp + D; L.n = L.bO + NI;
  return L;
}
struct B4Blk {
  size_t Wq, bq, Wk, bk, Wv, bv, Wo, bo, g1, c1, W1, b1, W2, b2, g2, c2;
};
static B4Blk b4_blk(const B4Layout& L, int b, int d) {
  const size_t D = d, DD = D * D;
  size_t o = L.blk0 + (size_t)b * L.blk_n;
  B4Blk k;
  k.Wq = o; o += DD; k.bq = o; o += D; k.Wk = o; o += DD; k.bk = o; o += D; k.Wv = o; o += DD; k.bv = o; o += D; k.Wo = o; o += DD;
  k.bo = o; o += D; k.g1 = o; o += D; k.c1 = o; o += D; k.W1 = o; o += 4 * DD; k.b1 = o; o += 4 * D; k.W2 = o; o += 4 * DD; k.b2 = o; o += D;
  k.g2 = o; o += D; k.c2 = o;
  return k;
}

// CTA per slot: positions, targets and PS rows, and X0 = E[x'] + Pe[t], x' the mask token (row NI) at a masked entry in training
// (mk: one byte per stored entry) and at a window's last position in evaluation; PY the original item at a masked entry, else -1
__global__ void __launch_bounds__(256) k_b4_embed(SaDev s, const unsigned char* mk, int NI, float* X0) {
  const int b = blockIdx.x, n = s.plen[b], p0 = s.poff[b];
  const long long s0 = s.pstart[b];
  for (int x = threadIdx.x; x < n * s.d; x += blockDim.x) {
    const int t = x / s.d, u = x % s.d, p = p0 + t;
    const bool masked = s.train ? mk[s0 + t] != 0 : t == n - 1;
    const int it = masked ? NI : s.items[s0 + t];
    if (u == 0) { s.PX[p] = it; s.PY[p] = s.train && masked ? s.items[s0 + t] : -1; s.PS[p] = b * s.L + t; }
    X0[(size_t)p * s.d + u] = __fadd_rn(s.E[(size_t)it * s.d + u], s.Pe[(size_t)t * s.d + u]);
  }
}

// CTA per (query position, head): the softmax over all n keys of the slot (scores and probabilities in shared memory, max and sum
// thread-strided then a fixed tree), A_t = sum_j p_j V_j in key order; the max and sum saved for the backward
__global__ void __launch_bounds__(B4_ATT_THREADS) k_b4_att_fwd(SaDev s, const float* Q, const float* K, const float* V, float* A, float* M, float* LS) {
  __shared__ float sc[B4_LEN_MAX];
  __shared__ float red[32];
  const int p = blockIdx.x, h = blockIdx.y, t = s.PS[p] % s.L, p0 = p - t, n = s.plen[s.PS[p] / s.L], c0 = h * s.dh;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < n; j += blockDim.x) { sc[j] = sa_score(s, Q, K, p, p0 + j, c0); m = fmaxf(m, sc[j]); }
  m = nm_block_reduce(m, red, true);
  float l = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) l = __fadd_rn(l, expf(__fsub_rn(sc[j], m)));
  l = nm_block_reduce(l, red, false);
  for (int j = threadIdx.x; j < n; j += blockDim.x) sc[j] = __fdiv_rn(expf(__fsub_rn(sc[j], m)), l);
  __syncthreads();
  for (int u = threadIdx.x; u < s.dh; u += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j < n; j++) a = __fmaf_rn(sc[j], V[(size_t)(p0 + j) * s.d + c0 + u], a);
    A[(size_t)p * s.d + c0 + u] = a;
  }
  if (threadIdx.x == 0) { M[(size_t)p * s.heads + h] = m; LS[(size_t)p * s.heads + h] = l; }
}

// CTA per (query position, head), the attention backward of the query over all n keys: D_t = dA_t . A_t,
// dS_tj = p_tj (dA_t . V_j - D_t), dQ_t = sh sum_j dS_tj K_j; p_tj recomputed bitwise from the saved max and sum; D_t saved
__global__ void __launch_bounds__(B4_ATT_THREADS) k_b4_att_bwd_q(SaDev s, const float* Q, const float* K, const float* V, const float* A, const float* dA,
                                                                 const float* M, const float* LS, float* dQ, float* DT) {
  __shared__ float ds[B4_LEN_MAX];
  __shared__ float red[32];
  const int p = blockIdx.x, h = blockIdx.y, t = s.PS[p] % s.L, p0 = p - t, n = s.plen[s.PS[p] / s.L], c0 = h * s.dh;
  const float* da = dA + (size_t)p * s.d + c0;
  float D = 0.f;
  for (int u = threadIdx.x; u < s.dh; u += blockDim.x) D = __fmaf_rn(da[u], A[(size_t)p * s.d + c0 + u], D);
  D = nm_block_reduce(D, red, false);
  const float m = M[(size_t)p * s.heads + h], l = LS[(size_t)p * s.heads + h];
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float pj = __fdiv_rn(expf(__fsub_rn(sa_score(s, Q, K, p, p0 + j, c0), m)), l);
    const float* v = V + (size_t)(p0 + j) * s.d + c0;
    float dp = 0.f;
    for (int u = 0; u < s.dh; u++) dp = __fmaf_rn(da[u], v[u], dp);
    ds[j] = __fmul_rn(pj, __fsub_rn(dp, D));
  }
  __syncthreads();
  for (int u = threadIdx.x; u < s.dh; u += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j < n; j++) a = __fmaf_rn(ds[j], K[(size_t)(p0 + j) * s.d + c0 + u], a);
    dQ[(size_t)p * s.d + c0 + u] = __fmul_rn(a, s.sh);
  }
  if (threadIdx.x == 0) DT[(size_t)p * s.heads + h] = D;
}

// CTA per (key position j, head), the attention backward of the key and value over all n queries i of the slot, in order:
// dV_j = sum_i p_ij dA_i, dK_j = sh sum_i dS_ij Q_i
__global__ void __launch_bounds__(B4_ATT_THREADS) k_b4_att_bwd_kv(SaDev s, const float* Q, const float* K, const float* V, const float* dA, const float* M,
                                                                  const float* LS, const float* DT, float* dK, float* dV) {
  __shared__ float pr[B4_LEN_MAX], ds[B4_LEN_MAX];
  const int p = blockIdx.x, h = blockIdx.y, j = s.PS[p] % s.L, p0 = p - j, n = s.plen[s.PS[p] / s.L], c0 = h * s.dh;
  const float* v = V + (size_t)p * s.d + c0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const size_t pi = (size_t)(p0 + i), hi = pi * s.heads + h;
    const float pij = __fdiv_rn(expf(__fsub_rn(sa_score(s, Q, K, pi, p, c0), M[hi])), LS[hi]);
    const float* da = dA + pi * s.d + c0;
    float dp = 0.f;
    for (int u = 0; u < s.dh; u++) dp = __fmaf_rn(da[u], v[u], dp);
    pr[i] = pij; ds[i] = __fmul_rn(pij, __fsub_rn(dp, DT[hi]));
  }
  __syncthreads();
  for (int u = threadIdx.x; u < s.dh; u += blockDim.x) {
    float av = 0.f, ak = 0.f;
    for (int i = 0; i < n; i++) {
      const size_t o = (size_t)(p0 + i) * s.d + c0 + u;
      av = __fmaf_rn(pr[i], dA[o], av); ak = __fmaf_rn(ds[i], Q[o], ak);
    }
    dV[(size_t)p * s.d + c0 + u] = av; dK[(size_t)p * s.d + c0 + u] = __fmul_rn(ak, s.sh);
  }
}

// Z [n / w x w] += b (per column), the pre-activation kept; G = gelu(Z) = Z Phi(Z), Phi by erf
__global__ void k_b4_gelu(float* Z, const float* b, float* G, long long n, int w) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float z = __fadd_rn(Z[i], b[i % w]);
  Z[i] = z;
  G[i] = __fmul_rn(z, __fmul_rn(0.5f, __fadd_rn(1.f, erff(__fmul_rn(z, 0.70710678118654752f)))));
}

// D *= gelu'(Z) = Phi(Z) + Z phi(Z)
__global__ void k_b4_gelu_bwd(float* D, const float* Z, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float z = Z[i];
  const float cdf = __fmul_rn(0.5f, __fadd_rn(1.f, erff(__fmul_rn(z, 0.70710678118654752f))));
  const float pdf = __fmul_rn(0.39894228040143268f, expf(__fmul_rn(-0.5f, __fmul_rn(z, z))));
  D[i] = __fmul_rn(D[i], __fmaf_rn(z, pdf, cdf));
}

// the masked rows: QM [Pm x d] = Q's rows MP[j] in order, MY[j] their targets
__global__ void k_b4_gather(const float* Q, const int* MP, const int* PY, int Pm, int d, float* QM, int* MY) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (long long)Pm * d) return;
  const int j = (int)(x / d), u = (int)(x % d), p = MP[j];
  QM[x] = Q[(size_t)p * d + u];
  if (u == 0) MY[j] = PY[p];
}

// dL/dq of every position: DQM's row MI[p] at a masked position, 0 elsewhere
__global__ void k_b4_unpick(const float* DQM, const int* MI, int P, int d, float* DQ) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (long long)P * d) return;
  const int p = (int)(x / d), u = (int)(x % d), j = MI[p];
  DQ[x] = j >= 0 ? DQM[(size_t)j * d + u] : 0.f;
}

// OUT = ((A + B) + C) + D
__global__ void k_b4_sum4(float* OUT, const float* A, const float* B, const float* C, const float* D, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) OUT[i] = __fadd_rn(__fadd_rn(__fadd_rn(A[i], B[i]), C[i]), D[i]);
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
// the per-position float arrays of P positions.  Training keeps every block's activations (blocks + 1 residual streams);
// evaluation keeps one block's, the stream updated in place, and carries no backward buffers.
struct B4Buf {
  long long P = 0; bool keep = false;
  float *H, *Q, *K, *V, *A, *X1, *A1, *Z1, *G1, *X2, *MU1, *RS1, *MU2, *RS2, *M, *LS;   // per block (H: per stream)
  float *X0, *MU0, *RS0, *ZH, *GH, *MUP, *RSP, *QO, *T;                              // embedding, head, a product's scratch
  float *LOSS, *QM, *DQM, *DQ, *DH, *DX, *DY, *DYX, *DG, *W[10], *DT;                // the backward
  float* at(float* base, int width, int blk) const { return keep ? base + (size_t)blk * P * width : base; }
};
static size_t b4_pos_floats(int d, int heads, int blocks, bool train) {
  const size_t D = d, nb = train ? blocks : 1;
  size_t f = (nb + (train ? 1 : 0)) * D + nb * (15 * D + 4 + 2 * (size_t)heads) + 5 * D + 4;
  if (train) f += 1 + 21 * D + heads;
  return f;
}
static void b4_carve(B4Buf& B, float* f, long long P, int d, int heads, int blocks, bool train) {
  B.P = P; B.keep = train;
  const size_t nb = train ? blocks : 1, D = d;
  auto take = [&](float** q, size_t w) { *q = f; f += (size_t)P * w; };
  take(&B.H, (nb + (train ? 1 : 0)) * D);
  take(&B.Q, nb * D); take(&B.K, nb * D); take(&B.V, nb * D); take(&B.A, nb * D); take(&B.X1, nb * D); take(&B.A1, nb * D);
  take(&B.Z1, nb * 4 * D); take(&B.G1, nb * 4 * D); take(&B.X2, nb * D);
  take(&B.MU1, nb); take(&B.RS1, nb); take(&B.MU2, nb); take(&B.RS2, nb); take(&B.M, nb * heads); take(&B.LS, nb * heads);
  take(&B.X0, D); take(&B.ZH, D); take(&B.GH, D); take(&B.QO, D); take(&B.T, D); take(&B.MU0, 1); take(&B.RS0, 1); take(&B.MUP, 1); take(&B.RSP, 1);
  if (!train) return;
  take(&B.LOSS, 1); take(&B.QM, D); take(&B.DQM, D); take(&B.DQ, D); take(&B.DH, D); take(&B.DX, D); take(&B.DY, D); take(&B.DYX, D);
  take(&B.DG, 4 * D);
  for (int k = 0; k < 10; k++) take(&B.W[k], D);
  take(&B.DT, heads);
}

// the encoder of a batch or chunk: QO [P x d], the head's output at every position (part: split scratch; encoder products never
// split)
static void b4_encode(cudaStream_t st, const SaDev& s, const B4Buf& B, const unsigned char* mk, int NI, const float* th, const B4Layout& Lo, int blocks,
                      float* part) {
  const int P = s.P, d = s.d;
  const long long n = (long long)P * d, n4 = 4 * n;
  const unsigned gl = (unsigned)((P + 7) / 8), ge = sa_grid(n), g4 = sa_grid(n4);
  k_b4_embed<<<s.nb, 256, 0, st>>>(s, mk, NI, B.X0);
  k_sa_ln<<<gl, 256, 0, st>>>(B.X0, th + Lo.g0, th + Lo.c0, P, d, B.T, B.MU0, B.RS0);
  k_sa_mask<<<ge, 256, 0, st>>>(s, B.T, B4_STREAM_H0, 0, B.at(B.H, d, 0), nullptr, 1.f);
  for (int b = 0; b < blocks; b++) {
    const B4Blk k = b4_blk(Lo, b, d);
    float *hin = B.at(B.H, d, b), *q = B.at(B.Q, d, b), *kk = B.at(B.K, d, b), *v = B.at(B.V, d, b), *a = B.at(B.A, d, b);
    float *x1 = B.at(B.X1, d, b), *a1 = B.at(B.A1, d, b), *z1 = B.at(B.Z1, 4 * d, b), *g1 = B.at(B.G1, 4 * d, b), *x2 = B.at(B.X2, d, b);
    float* hout = B.at(B.H, d, b + 1);
    nm_gemm<NM_ENCODER>(st, part, hin, d, 1, th + k.Wq, d, 1, q, d, P, d, d);
    nm_gemm<NM_ENCODER>(st, part, hin, d, 1, th + k.Wk, d, 1, kk, d, P, d, d);
    nm_gemm<NM_ENCODER>(st, part, hin, d, 1, th + k.Wv, d, 1, v, d, P, d, d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(q, th + k.bq, n, d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(kk, th + k.bk, n, d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(v, th + k.bv, n, d);
    k_b4_att_fwd<<<dim3((unsigned)P, (unsigned)s.heads), B4_ATT_THREADS, 0, st>>>(s, q, kk, v, a, B.at(B.M, s.heads, b), B.at(B.LS, s.heads, b));
    nm_gemm<NM_ENCODER>(st, part, a, d, 1, th + k.Wo, d, 1, B.T, d, P, d, d);
    k_sa_resid<<<ge, 256, 0, st>>>(s, x1, hin, B.T, th + k.bo, B4_STREAM_ATT, b + 1);
    k_sa_ln<<<gl, 256, 0, st>>>(x1, th + k.g1, th + k.c1, P, d, a1, B.at(B.MU1, 1, b), B.at(B.RS1, 1, b));
    nm_gemm<NM_ENCODER>(st, part, a1, d, 1, th + k.W1, 4 * d, 1, z1, 4 * d, P, 4 * d, d);
    k_b4_gelu<<<g4, 256, 0, st>>>(z1, th + k.b1, g1, n4, 4 * d);
    nm_gemm<NM_ENCODER>(st, part, g1, 4 * d, 1, th + k.W2, d, 1, B.T, d, P, d, 4 * d);
    k_sa_resid<<<ge, 256, 0, st>>>(s, x2, a1, B.T, th + k.b2, B4_STREAM_FFN, b + 1);
    k_sa_ln<<<gl, 256, 0, st>>>(x2, th + k.g2, th + k.c2, P, d, hout, B.at(B.MU2, 1, b), B.at(B.RS2, 1, b));
  }
  nm_gemm<NM_ENCODER>(st, part, B.at(B.H, d, blocks), d, 1, th + Lo.Wp, d, 1, B.ZH, d, P, d, d);
  k_b4_gelu<<<ge, 256, 0, st>>>(B.ZH, th + Lo.bp, B.GH, n, d);
  k_sa_ln<<<gl, 256, 0, st>>>(B.GH, th + Lo.gp, th + Lo.cp, P, d, B.QO, B.MUP, B.RSP);
}

// the gradient of a product Y = X W (+ b), X [P x din], W [din x dout], given dY: G.W = X^T dY, G.b = column sums of dY, dX = dY W^T
static void b4_linear_bwd(cudaStream_t st, float* part, const float* ones, const float* X, const float* W, const float* dY, float* gW, float* gb,
                          float* dX, int P, int din, int dout) {
  nm_gemm<NM_BACKWARD>(st, part, X, 1, din, dY, dout, 1, gW, dout, din, dout, P);
  sa_colsum(st, part, ones, dY, gb, P, dout);
  nm_gemm<NM_BACKWARD>(st, part, dY, dout, 1, W, 1, dout, dX, din, P, din, dout);
}

// the masked rows of a batch: MP [Pm] their positions in order, MI [P] each position's row in MP (-1: not masked), MY [Pm]
struct B4Rows {
  const int* MP; const int* MI; int* MY; int Pm;
};

// a batch's loss and gradient G (flat, the parameters' layout) at the handle's parameters; loss_out a device float
static void b4_grad(cudaStream_t st, const SaDev& s, const B4Buf& B, const NmScratch& ns, const B4Rows& r, const unsigned char* mk, const float* th,
                    const B4Layout& Lo, int blocks, int NI, float* G, const float* ones, float* loss_out) {
  const int P = s.P, d = s.d, Pm = r.Pm, hs = s.heads;
  const long long n = (long long)P * d, n4 = 4 * n;
  const unsigned gl = (unsigned)((P + 7) / 8), ge = sa_grid(n);
  float* part = ns.part;
  b4_encode(st, s, B, mk, NI, th, Lo, blocks, part);
  // the catalogue over the masked rows only: logits QM E^T + bO, the softmax gradient, dL/dq, dE (rows < NI) and dbO
  k_b4_gather<<<sa_grid((long long)Pm * d), 256, 0, st>>>(B.QO, r.MP, s.PY, Pm, d, B.QM, r.MY);
  NmDev nd{};
  nd.P = Pm; nd.d = d; nd.NI = NI; nd.S = ns.S; nd.PY = r.MY; nd.PX = s.PX; nd.PS = s.PS; nd.LOSS = B.LOSS; nd.re = 1.f;
  const float* E = th + Lo.E;
  nm_gemm<NM_CATALOGUE>(st, part, B.QM, d, 1, E, 1, d, ns.S, NI, Pm, NI, d);
  k_sa_bias<false><<<sa_grid((long long)Pm * NI), 256, 0, st>>>(ns.S, th + Lo.bO, (long long)Pm * NI, NI);
  k_nm_softmax<<<Pm, 256, 0, st>>>(nd);
  k_nm_mean<<<1, 1024, 0, st>>>(B.LOSS, Pm, loss_out);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, NI, 1, E, d, 1, B.DQM, d, Pm, d, NI);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, 1, NI, B.QM, d, 1, G + Lo.E, d, NI, d, Pm);
  sa_colsum(st, part, ones, ns.S, G + Lo.bO, Pm, NI);
  k_b4_unpick<<<ge, 256, 0, st>>>(B.DQM, r.MI, P, d, B.DQ);
  // the head: q = LNp(gelu(h Wp + bp))
  k_sa_ln_bwd<<<gl, 256, 0, st>>>(B.GH, B.MUP, B.RSP, th + Lo.gp, B.DQ, nullptr, nullptr, nullptr, P, d, B.DX, B.DY, B.DYX);
  sa_colsum(st, part, ones, B.DYX, G + Lo.gp, P, d);
  sa_colsum(st, part, ones, B.DY, G + Lo.cp, P, d);
  k_b4_gelu_bwd<<<ge, 256, 0, st>>>(B.DX, B.ZH, n);
  b4_linear_bwd(st, part, ones, B.at(B.H, d, blocks), th + Lo.Wp, B.DX, G + Lo.Wp, G + Lo.bp, B.DH, P, d, d);
  float* const* T = B.W;
  for (int b = blocks - 1; b >= 0; b--) {
    const B4Blk k = b4_blk(Lo, b, d);
    float *hin = B.at(B.H, d, b), *q = B.at(B.Q, d, b), *kk = B.at(B.K, d, b), *v = B.at(B.V, d, b), *a = B.at(B.A, d, b);
    float *x1 = B.at(B.X1, d, b), *a1 = B.at(B.A1, d, b), *z1 = B.at(B.Z1, 4 * d, b), *g1 = B.at(B.G1, 4 * d, b), *x2 = B.at(B.X2, d, b);
    // h' = LN2(x2), x2 = a1 + mask (gelu(a1 W1 + b1) W2 + b2): T0 = dL/dx2
    k_sa_ln_bwd<<<gl, 256, 0, st>>>(x2, B.at(B.MU2, 1, b), B.at(B.RS2, 1, b), th + k.g2, B.DH, nullptr, nullptr, nullptr, P, d, T[0], B.DY, B.DYX);
    sa_colsum(st, part, ones, B.DYX, G + k.g2, P, d);
    sa_colsum(st, part, ones, B.DY, G + k.c2, P, d);
    k_sa_mask<<<ge, 256, 0, st>>>(s, T[0], B4_STREAM_FFN, b + 1, T[1], nullptr, 1.f);
    b4_linear_bwd(st, part, ones, g1, th + k.W2, T[1], G + k.W2, G + k.b2, B.DG, P, 4 * d, d);
    k_b4_gelu_bwd<<<sa_grid(n4), 256, 0, st>>>(B.DG, z1, n4);
    b4_linear_bwd(st, part, ones, a1, th + k.W1, B.DG, G + k.W1, G + k.b1, T[2], P, d, 4 * d);
    // a1 = LN1(x1) feeds the FFN and the residual: T3 = dL/dx1, x1 = hin + mask (A Wo + bo)
    k_sa_ln_bwd<<<gl, 256, 0, st>>>(x1, B.at(B.MU1, 1, b), B.at(B.RS1, 1, b), th + k.g1, T[2], T[0], nullptr, nullptr, P, d, T[3], B.DY, B.DYX);
    sa_colsum(st, part, ones, B.DYX, G + k.g1, P, d);
    sa_colsum(st, part, ones, B.DY, G + k.c1, P, d);
    k_sa_mask<<<ge, 256, 0, st>>>(s, T[3], B4_STREAM_ATT, b + 1, T[1], nullptr, 1.f);
    b4_linear_bwd(st, part, ones, a, th + k.Wo, T[1], G + k.Wo, G + k.bo, T[4], P, d, d);
    const dim3 ga((unsigned)P, (unsigned)hs);
    k_b4_att_bwd_q<<<ga, B4_ATT_THREADS, 0, st>>>(s, q, kk, v, a, T[4], B.at(B.M, hs, b), B.at(B.LS, hs, b), T[5], B.DT);
    k_b4_att_bwd_kv<<<ga, B4_ATT_THREADS, 0, st>>>(s, q, kk, v, T[4], B.at(B.M, hs, b), B.at(B.LS, hs, b), B.DT, T[6], T[7]);
    b4_linear_bwd(st, part, ones, hin, th + k.Wq, T[5], G + k.Wq, G + k.bq, T[8], P, d, d);
    b4_linear_bwd(st, part, ones, hin, th + k.Wk, T[6], G + k.Wk, G + k.bk, T[9], P, d, d);
    b4_linear_bwd(st, part, ones, hin, th + k.Wv, T[7], G + k.Wv, G + k.bv, T[5], P, d, d);
    k_b4_sum4<<<ge, 256, 0, st>>>(B.DH, T[3], T[8], T[9], T[5], n);
  }
  // h0 = mask LN0(E[x'] + Pe[t]): DX = dL/dX0, Pe's gradient and the input-embedding rows (the mask row's only gradient)
  k_sa_mask<<<ge, 256, 0, st>>>(s, B.DH, B4_STREAM_H0, 0, T[0], nullptr, 1.f);
  k_sa_ln_bwd<<<gl, 256, 0, st>>>(B.X0, B.MU0, B.RS0, th + Lo.g0, T[0], nullptr, nullptr, nullptr, P, d, B.DX, B.DY, B.DYX);
  sa_colsum(st, part, ones, B.DYX, G + Lo.g0, P, d);
  sa_colsum(st, part, ones, B.DY, G + Lo.c0, P, d);
  k_sa_pe_grad<<<sa_grid((long long)s.L * d), 256, 0, st>>>(s, B.DX, G + Lo.Pe);
  cudaMemsetAsync(G + Lo.E + (size_t)NI * d, 0, (size_t)d * sizeof(float), st);
  nd.P = P; nd.DEMB = B.DX;
  k_nm_keys<<<(P + 255) / 256, 256, 0, st>>>(s.PX, P, ns.keys);
  int end_bit = 33;                                      // the keys' item field covers the mask row NI
  while (end_bit < 64 && ((unsigned long long)(NI + 1) >> (end_bit - 32)) != 0ull) end_bit++;
  size_t cb = ns.cub_bytes;
  cub::DeviceRadixSort::SortKeys(ns.cub, cb, ns.keys, ns.keys2, P, 0, end_bit, st);
  k_nm_scatter<<<ge, 256, 0, st>>>(nd, ns.keys2, G + Lo.E);
}

static bool b4_shape_ok(int d, int blocks, int heads, int len) {
  return d >= 1 && d <= B4_D_MAX && blocks >= 1 && blocks <= B4_BLOCKS_MAX && heads >= 1 && heads <= d && d % heads == 0 && len >= 2 &&
         len <= B4_LEN_MAX;
}
#define B4_SHAPE_MSG ": need n_blocks in 1 .. 8, n_heads dividing the embedding and max_len in 2 .. 512"

// dI = double(E[0 .. n_items)) and dBI = double(bO), the item side bpr_blocks ranks against; after every epoch and every import
static cudaError_t b4_refresh(g4r_baselines* h, const B4Layout& L) {
  const size_t nE = (size_t)h->n_items * h->n_keep;
  k_nm_to_double<<<(unsigned)((nE + 255) / 256), 256, 0, h->stream>>>(h->dNmTh + L.E, nE, h->dI);
  k_nm_to_double<<<(unsigned)((h->n_items + 255) / 256), 256, 0, h->stream>>>(h->dNmTh + L.bO, (size_t)h->n_items, h->dBI);
  return cudaGetLastError();
}

static B4Layout b4_handle_layout(const g4r_baselines* h) { return b4_layout(h->n_items, h->n_keep, h->sa_blocks, h->nm_len); }

// the model buffers of a BERT4Rec handle (NARM's fields): parameters, double(E) and double(bO) for bpr_blocks, a device 1.0f
static int b4_set_model(g4r_baselines* h, int32_t blocks, int32_t heads, int32_t max_len, const float* params, int64_t n_params, const char* who) {
  if (!params) FAIL(G4R_ERR_INVALID, std::string(who) + ": null parameters");
  if (!b4_shape_ok(h->n_keep, blocks, heads, max_len)) FAIL(G4R_ERR_INVALID, std::string(who) + B4_SHAPE_MSG);
  const B4Layout L = b4_layout(h->n_items, h->n_keep, blocks, max_len);
  if (n_params != (int64_t)L.n)
    FAIL(G4R_ERR_INVALID, std::string(who) + ": need n_params = (n_items + 1) d + max_len d + 2 d + n_blocks (12 d^2 + 13 d) + d^2 + 3 d + n_items = " +
                              std::to_string(L.n));
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
  h->sa_blocks = blocks; h->sa_heads = heads; h->nm_len = max_len; h->nm_n = L.n;
  CK(b4_refresh(h, L));
  CK(cudaStreamSynchronize(st));
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_bert4rec_import(g4r_baselines* h, int32_t n_blocks, int32_t n_heads, int32_t max_len, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BERT4REC) FAIL(G4R_ERR_STATE, "g4r_bl_bert4rec_import: the handle is not a BERT4Rec");
  return b4_set_model(h, n_blocks, n_heads, max_len, params, n_params, "g4r_bl_bert4rec_import");
}

extern "C" int g4r_bl_bert4rec_export(g4r_baselines* h, float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BERT4REC || !h->dNmTh)
    FAIL(G4R_ERR_STATE, "g4r_bl_bert4rec_export: no BERT4Rec parameters (g4r_bl_bert4rec_begin or g4r_bl_bert4rec_import)");
  if (!params || n_params != (int64_t)h->nm_n) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_export: need n_params floats");
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(params, h->dNmTh, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// The device stores each piece followed by one unused entry (piece k's entries start at piece_offsets[k] + k), so that NARM's
// planner, which counts a piece's inputs as its events minus one, plans a piece of inputs only unchanged; the mask bytes follow the
// same layout.
extern "C" int g4r_bl_bert4rec_begin(g4r_baselines* h, int32_t n_blocks, int32_t n_heads, int32_t max_len, int32_t batch_size, const int64_t* piece_offsets,
                                     int64_t n_pieces, const int32_t* items, int64_t n_entries, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BERT4REC) FAIL(G4R_ERR_STATE, "g4r_bl_bert4rec_begin: the handle is not a BERT4Rec");
  if (!piece_offsets || !items || n_pieces < 1 || n_entries < 2 || batch_size < 1)
    FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_begin: null argument, no pieces or batch_size < 1");
  const int NI = h->n_items, dd = h->n_keep;
  if (!b4_shape_ok(dd, n_blocks, n_heads, max_len)) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_begin" B4_SHAPE_MSG);
  if (n_entries + n_pieces > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_begin: more than 2^31 - 1 entries and pieces");
  if (piece_offsets[0] != 0 || piece_offsets[n_pieces] != n_entries) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_begin: piece offsets must run from 0 to n_entries");
  std::vector<int> lens(n_pieces);
  for (int64_t k = 0; k < n_pieces; k++) {
    const int64_t n = piece_offsets[k + 1] - piece_offsets[k];
    if (n < 2 || n > (int64_t)max_len) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_begin: every piece needs 2 .. max_len events");
    lens[k] = (int)n;
  }
  for (int64_t e = 0; e < n_entries; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_bert4rec_begin: item index out of range");
  if ((uint64_t)(n_blocks + 1) * (uint64_t)batch_size * (uint64_t)max_len * (uint64_t)dd >= 0x100000000ull)
    FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_begin: (n_blocks + 1) * batch_size * max_len * d must stay below 2^32 (dropout indices)");
  // the largest batch: the batch_size longest pieces
  std::vector<int> srt(lens);
  std::sort(srt.begin(), srt.end(), std::greater<int>());
  long long Pmax = 0;
  for (int64_t k = 0; k < std::min<int64_t>(batch_size, n_pieces); k++) Pmax += srt[k];
  const B4Layout L = b4_layout(NI, dd, n_blocks, max_len);
  const size_t stored = (size_t)(n_entries + n_pieces);
  const size_t act = (size_t)Pmax * b4_pos_floats(dd, n_heads, n_blocks, true) * 4;
  const size_t need = (size_t)Pmax * ((size_t)NI * 4 + 40) + act + NM_PART_CAP * 4 + 3 * L.n * 4 + stored * 5 + (size_t)n_pieces * 16 +
                      ((size_t)64 << 20);
  int rc = b4_set_model(h, n_blocks, n_heads, max_len, params, n_params, "g4r_bl_bert4rec_begin");
  if (rc) return rc;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    h->err = "g4r_bl_bert4rec_begin: the fit needs " + std::to_string(need) + " bytes of device memory (the logits of the largest batch " +
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
  CK(take(&h->b4_f, (size_t)Pmax * b4_pos_floats(dd, n_heads, n_blocks, true)));
  CK(take(&h->b4_my, Pmax)); CK(take(&h->b4_mk, stored));
  CK(nm_take(h, &h->dNmG, L.n)); CK(nm_take(h, &h->dNmM, L.n)); CK(nm_take(h, &h->dNmV, L.n)); CK(nm_take(h, &h->dNmItems, stored));
  CK(nm_take(h, &h->dNmLoss, 1));
  CK(cudaMemsetAsync(h->dNmM, 0, L.n * sizeof(float), st)); CK(cudaMemsetAsync(h->dNmV, 0, L.n * sizeof(float), st));
  h->nm_off.resize(n_pieces + 1);
  std::vector<int> padded(stored, 0);
  for (int64_t k = 0; k <= n_pieces; k++) h->nm_off[k] = piece_offsets[k] + k;
  for (int64_t k = 0; k < n_pieces; k++) std::copy(items + piece_offsets[k], items + piece_offsets[k + 1], padded.begin() + h->nm_off[k]);
  CK(cudaMemcpyAsync(h->dNmItems, padded.data(), stored * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  h->nm_bs = batch_size; h->nm_Pmax = Pmax; h->nm_step = 0; h->nm_fit = true;
  h->ready = true;
  return G4R_OK;
}

static SaDev b4_dev(const g4r_baselines* h, const B4Layout& Lo) {
  SaDev s{};
  s.E = h->dNmTh + Lo.E; s.Pe = h->dNmTh + Lo.Pe;
  s.d = h->n_keep; s.L = h->nm_len; s.heads = h->sa_heads; s.dh = h->n_keep / h->sa_heads;
  s.sd = 1.f; s.sh = (float)(1.0 / std::sqrt((double)s.dh));
  s.retain = 1.f; s.bsL = (unsigned)h->nm_bs * (unsigned)h->nm_len;
  return s;
}

static SaDev b4_train_dev(g4r_baselines* h, const B4Layout& Lo, unsigned seed, unsigned gstep, float dropout) {
  SaDev s = b4_dev(h, Lo);
  const NmScratch& ns = h->nm_s;
  s.items = h->dNmItems; s.train = 1; s.seed = seed; s.gstep = gstep; s.retain = dropout > 0.f ? 1.f - dropout : 1.f;
  s.PX = ns.PX; s.PY = ns.PY; s.PS = ns.PS; s.pstart = ns.pstart; s.plen = ns.plen; s.poff = ns.poff;
  return s;
}

// the checks of an epoch or grads call, and the masked rows of its batches: per batch (first position in MP / MI, Pm); MP holds the
// positions of the batch's masked entries in order, MI per position its row in MP or -1.  mk_dev: the mask bytes in the device's
// layout.
static int b4_check_run(g4r_baselines* h, const int32_t* pieces, int64_t n, const uint8_t* masks, int64_t n_masks, float dropout, const char* who,
                        std::vector<long long>& ps, std::vector<int>& pl, std::vector<int>& po, std::vector<std::pair<int64_t, int>>& batches,
                        std::vector<int>& MP, std::vector<int>& MI, std::vector<std::pair<int64_t, int>>& rows, std::vector<uint8_t>& mk_dev) {
  if (h->kind != BL_BERT4REC) FAIL(G4R_ERR_STATE, std::string(who) + ": the handle is not a BERT4Rec");
  if (!h->nm_fit) FAIL(G4R_ERR_STATE, std::string(who) + ": no fit begun (g4r_bl_bert4rec_begin)");
  if (!pieces || n < 1) FAIL(G4R_ERR_INVALID, std::string(who) + ": no pieces");
  if (!(dropout >= 0.f && dropout < 1.f)) FAIL(G4R_ERR_INVALID, std::string(who) + ": dropout must be in [0, 1)");
  const int64_t np = (int64_t)h->nm_off.size() - 1, n_entries = h->nm_off[np] - np;
  for (int64_t q = 0; q < n; q++) if (pieces[q] < 0 || pieces[q] >= np) FAIL(G4R_ERR_INDEX, std::string(who) + ": piece index out of range");
  if (!masks || n_masks != n_entries) FAIL(G4R_ERR_INVALID, std::string(who) + ": need one mask byte per stored entry (n_masks = n_entries)");
  for (int64_t e = 0; e < n_masks; e++) if (masks[e] > 1) FAIL(G4R_ERR_INVALID, std::string(who) + ": mask bytes must be 0 or 1");
  for (int64_t q = 0; q < n; q++) {
    const int k = pieces[q];
    const int64_t e0 = h->nm_off[k] - k, e1 = h->nm_off[k + 1] - (k + 1);
    bool any = false;
    for (int64_t e = e0; e < e1; e++) any = any || masks[e];
    if (!any) FAIL(G4R_ERR_INVALID, std::string(who) + ": every piece used needs at least one masked entry");
  }
  int rc = nm_plan(h, pieces, n, ps, pl, po, batches, who);
  if (rc) return rc;
  mk_dev.assign((size_t)(n_entries + np), 0);
  for (int64_t k = 0; k < np; k++)
    for (int64_t e = h->nm_off[k] - k; e < h->nm_off[k + 1] - (k + 1); e++) mk_dev[e + k] = masks[e];
  for (const auto& bt : batches) {
    const int64_t m0 = (int64_t)MP.size();
    for (int64_t q = bt.first; q < std::min<int64_t>(n, bt.first + h->nm_bs); q++)
      for (int t = 0; t < pl[q]; t++) {
        if (mk_dev[ps[q] + t]) { MI.push_back((int)(MP.size() - m0)); MP.push_back(po[q] + t); }
        else MI.push_back(-1);
      }
    rows.push_back({m0, (int)(MP.size() - m0)});
  }
  return G4R_OK;
}

extern "C" int g4r_bl_bert4rec_grads(g4r_baselines* h, const int32_t* pieces, int32_t n, const uint8_t* masks, int64_t n_masks, uint32_t seed, int64_t step,
                                     float dropout, float* loss, float* grads) {
  if (!h) return G4R_ERR_INVALID;
  std::vector<long long> ps; std::vector<int> pl, po, MP, MI; std::vector<std::pair<int64_t, int>> batches, rows; std::vector<uint8_t> mk;
  if (h->kind == BL_BERT4REC && h->nm_fit && (n > h->nm_bs || !grads || step < 0 || step > 0xffffffffll))
    FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_grads: need n <= batch_size, grads and step in 0 .. 2^32 - 1");
  int rc = b4_check_run(h, pieces, n, masks, n_masks, dropout, "g4r_bl_bert4rec_grads", ps, pl, po, batches, MP, MI, rows, mk);
  if (rc) return rc;
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  rc = nm_upload_plan(h, ps, pl, po, 0, n);
  if (rc) return rc;
  BlBufs bb;
  const int *dMP = nullptr, *dMI = nullptr;
  CK(bb.put(&dMP, MP.data(), MP.size(), st)); CK(bb.put(&dMI, MI.data(), MI.size(), st));
  CK(cudaMemcpyAsync(h->b4_mk, mk.data(), mk.size(), cudaMemcpyHostToDevice, st));
  const B4Layout Lo = b4_handle_layout(h);
  SaDev s = b4_train_dev(h, Lo, seed, (unsigned)step, dropout);
  s.nb = n; s.P = batches[0].second;
  B4Buf B;
  b4_carve(B, h->b4_f, h->nm_Pmax, h->n_keep, h->sa_heads, h->sa_blocks, true);
  const B4Rows r{dMP, dMI, h->b4_my, rows[0].second};
  b4_grad(st, s, B, h->nm_s, r, h->b4_mk, h->dNmTh, Lo, h->sa_blocks, h->n_items, h->dNmG, h->dNmOne, h->dNmLoss);
  CK(cudaGetLastError());
  float l = 0.f;
  CK(cudaMemcpyAsync(&l, h->dNmLoss, sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(grads, h->dNmG, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (loss) *loss = l;
  return G4R_OK;
}

extern "C" int g4r_bl_bert4rec_epoch(g4r_baselines* h, const int32_t* order, int64_t n_order, const uint8_t* masks, int64_t n_masks, uint32_t seed,
                                     float learning_rate, float dropout, float* losses, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind == BL_BERT4REC && h->nm_fit && !(learning_rate > 0.f && std::isfinite(learning_rate)))
    FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_epoch: learning_rate must be finite and > 0");
  std::vector<long long> ps; std::vector<int> pl, po, MP, MI; std::vector<std::pair<int64_t, int>> batches, rows; std::vector<uint8_t> mk;
  int rc = b4_check_run(h, order, n_order, masks, n_masks, dropout, "g4r_bl_bert4rec_epoch", ps, pl, po, batches, MP, MI, rows, mk);
  if (rc) return rc;
  if (h->nm_step + (int64_t)batches.size() > 0xffffffffll) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_epoch: more than 2^32 steps since the fit began");
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  const B4Layout Lo = b4_handle_layout(h);
  B4Buf B;
  b4_carve(B, h->b4_f, h->nm_Pmax, h->n_keep, h->sa_heads, h->sa_blocks, true);
  // the whole epoch's plan, masked rows and mask bytes go up once; each batch reads its slice
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr, *dMP = nullptr, *dMI = nullptr; float* dloss = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  CK(bb.put(&dMP, MP.data(), MP.size(), st)); CK(bb.put(&dMI, MI.data(), MI.size(), st));
  CK(cudaMemcpyAsync(h->b4_mk, mk.data(), mk.size(), cudaMemcpyHostToDevice, st));
  CK(bb.take(&dloss, batches.size()));
  CK(cudaEventRecord(h->ev0, st));
  int64_t mi0 = 0;
  for (size_t b = 0; b < batches.size(); b++) {
    const int64_t q0 = batches[b].first;
    SaDev s = b4_train_dev(h, Lo, seed, (unsigned)h->nm_step, dropout);
    s.pstart = dps + q0; s.plen = dpl + q0; s.poff = dpo + q0; s.nb = (int)std::min<int64_t>(h->nm_bs, n_order - q0); s.P = batches[b].second;
    const B4Rows r{dMP + rows[b].first, dMI + mi0, h->b4_my, rows[b].second};
    mi0 += s.P;
    b4_grad(st, s, B, h->nm_s, r, h->b4_mk, h->dNmTh, Lo, h->sa_blocks, h->n_items, h->dNmG, h->dNmOne, dloss + b);
    h->nm_step++;
    const double t = (double)h->nm_step;
    const float c1 = (float)(1.0 / (1.0 - std::pow(0.9, t))), c2 = (float)(1.0 / (1.0 - std::pow(0.999, t)));
    k_nm_adam<<<(unsigned)((Lo.n + 255) / 256), 256, 0, st>>>(h->dNmTh, h->dNmG, h->dNmM, h->dNmV, Lo.n, learning_rate, c1, c2);
  }
  CK(b4_refresh(h, Lo));
  CK(cudaEventRecord(h->ev1, st));
  if (losses) CK(cudaMemcpyAsync(losses, dloss, batches.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (device_ms) CK(cudaEventElapsedTime(device_ms, h->ev0, h->ev1));
  return G4R_OK;
}

// every counted event's q into qev [n_ev x d] on the device (eval mode: no dropout).  Each event is its own window, the last
// min(p, max_len - 1) inputs of its prefix followed by the mask token, q the head's output at the mask; windows share no work, so
// they are planned per event in chunks of at most B4_EVAL_POS positions.
static int b4_encode_events(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* off, int64_t n_sessions, const int32_t* n_history,
                            const std::vector<int64_t>& ev0, float* qev) {
  const int dd = h->n_keep, len = h->nm_len;
  cudaStream_t st = h->stream;
  const B4Layout Lo = b4_handle_layout(h);
  BlBufs bb;
  int *PX = nullptr, *PY = nullptr, *PS = nullptr, *dEv = nullptr, *dPair = nullptr, *plen = nullptr, *poff = nullptr;
  long long* pstart = nullptr;
  float* f = nullptr;
  const int* dItems = nullptr;
  CK(bb.take(&PX, B4_EVAL_POS)); CK(bb.take(&PY, B4_EVAL_POS)); CK(bb.take(&PS, B4_EVAL_POS));
  CK(bb.take(&dEv, B4_EVAL_POS)); CK(bb.take(&dPair, B4_EVAL_POS));
  CK(bb.take(&pstart, B4_EVAL_POS)); CK(bb.take(&plen, B4_EVAL_POS)); CK(bb.take(&poff, B4_EVAL_POS));
  CK(bb.take(&f, (size_t)B4_EVAL_POS * b4_pos_floats(dd, h->sa_heads, h->sa_blocks, false)));
  CK(bb.put(&dItems, items, n_events, st));
  B4Buf B;
  b4_carve(B, f, B4_EVAL_POS, dd, h->sa_heads, h->sa_blocks, false);
  SaDev s = b4_dev(h, Lo);
  s.items = dItems; s.train = 0; s.PX = PX; s.PY = PY; s.PS = PS; s.pstart = pstart; s.plen = plen; s.poff = poff;
  std::vector<long long> ps; std::vector<int> pl, po, ev, pair;
  int P = 0;
  auto flush = [&]() -> int {
    if (ps.empty()) return G4R_OK;
    const int nb = (int)ps.size();
    CK(cudaMemcpyAsync(pstart, ps.data(), nb * sizeof(long long), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(plen, pl.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(poff, po.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dEv, ev.data(), ev.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dPair, pair.data(), pair.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    s.nb = nb; s.P = P;
    b4_encode(st, s, B, nullptr, h->n_items, h->dNmTh, Lo, h->sa_blocks, nullptr);
    k_nm_pick<<<(unsigned)(((long long)nb * dd + 255) / 256), 256, 0, st>>>(B.QO, dEv, dPair, nb, dd, qev);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));                      // the host arrays are reused by the next chunk
    ps.clear(); pl.clear(); po.clear(); ev.clear(); pair.clear(); P = 0;
    return G4R_OK;
  };
  for (int64_t sI = 0; sI < n_sessions; sI++) {
    const int64_t st0 = off[sI], en = off[sI + 1];
    const int64_t i0 = std::max<int64_t>(n_history ? n_history[sI] : 0, 1) - 1;   // input index of the first counted event
    for (int64_t i = i0; i <= en - st0 - 2; i++) {
      const int m = (int)std::min<int64_t>(i + 1, len - 1), n = m + 1;
      if (P + n > B4_EVAL_POS) { const int rc = flush(); if (rc) return rc; }
      ev.push_back((int)(ev0[sI] + i - i0)); pair.push_back(P + m);
      ps.push_back(st0 + i + 1 - m); pl.push_back(n); po.push_back(P); P += n;
    }
  }
  return flush();
}

extern "C" int g4r_bl_bert4rec_encode(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                                      const int32_t* n_history, float* q, int64_t n_q) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_BERT4REC || !h->ready)
    FAIL(G4R_ERR_STATE, "g4r_bl_bert4rec_encode: no BERT4Rec parameters (g4r_bl_bert4rec_begin or g4r_bl_bert4rec_import)");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || n_q < 0 || (n_q > 0 && !q))
    FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_encode: null or out-of-range argument");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_encode: session offsets must rise from 0 to n_events");
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= h->n_items) FAIL(G4R_ERR_INDEX, "g4r_bl_bert4rec_encode: item index out of range");
  std::vector<int64_t> ev0;
  int rc = bl_counted(h, "g4r_bl_bert4rec_encode", session_offsets, n_sessions, n_history, ev0);
  if (rc) return rc;
  if (n_q != ev0[n_sessions]) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_encode: n_q must be the number of counted events");
  if (n_q > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_bert4rec_encode: more than 2^31 - 1 counted events");
  cudaSetDevice(h->device);
  BlBufs bb;
  float* dq = nullptr;
  CK(bb.take(&dq, (size_t)n_q * h->n_keep));
  rc = b4_encode_events(h, items, n_events, session_offsets, n_sessions, n_history, ev0, dq);
  if (rc) return rc;
  if (n_q) CK(cudaMemcpyAsync(q, dq, (size_t)n_q * h->n_keep * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// the ranking of a g4r_bl_evaluate call of a BERT4Rec: every counted event's q, then BPR's ranking with I = double(E[0 ..
// n_items)), bI = double(bO)
static int bert4rec_rank(g4r_baselines* h, BlCall& c) {
  float* dq = nullptr;
  CK(c.bb.take(&dq, (size_t)c.n_ev * h->n_keep));
  const int rc = b4_encode_events(h, c.items, c.n_events, c.off, c.n_sessions, c.n_history, c.ev0, dq);
  if (rc) return rc;
  return bpr_blocks(h, c, dq);
}
