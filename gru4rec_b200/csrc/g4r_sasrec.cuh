// g4r_sasrec.cuh -- the SASRec self-attentive baseline on the device (DESIGN §3t): learned positions over the tied item table, a
// stack of pre-LN Transformer blocks (causal multi-head attention and a position-wise ReLU FFN), a final layer norm and
// full-catalogue cross-entropy, trained with NARM's dense Adam; and the eval-mode encoder that feeds per-event vectors to BPR's
// ranking.  Every product runs through NARM's k_nm_gemm, the catalogue loss through k_nm_softmax, the input-embedding gradient
// through k_nm_keys / k_nm_scatter; every reduction here runs in a fixed order (no floating-point atomics), so a fit is bitwise
// reproducible and independent of grid sizes.  The training plan (pieces, batches, scratch bound) and the evaluation's chunk
// planner are NARM's; a SASRec handle keeps its model in the handle's NARM fields.  Included at the end of g4r_lib.cu after
// g4r_narm.cuh.
#pragma once

constexpr int SA_D_MAX = 1024, SA_BLOCKS_MAX = 8, SA_LEN_MAX = 512;
constexpr int SA_ATT_THREADS = 128;                    // attention CTA: more keys than this, or a wider head, loops per thread
constexpr int SA_EVAL_PAIRS = 16384;                   // encoder positions (and pieces) per evaluation chunk
constexpr unsigned SA_STREAM_H0 = 210u, SA_STREAM_ATT = 211u, SA_STREAM_FFN = 212u;   // dropout streams
constexpr float SA_LN_EPS = 1e-8f;

// offsets of the parameters in the flat float32 vector: E, Pe, per block (g1, c1, Wq, bq, Wk, bk, Wv, bv, Wo, bo, g2, c2, W1, b1,
// W2, b2), gf, cf
struct SaLayout {
  size_t E, Pe, blk0, blk_n, gf, cf, n;
};
static SaLayout sa_layout(int NI, int d, int n_blocks, int len) {
  SaLayout L;
  const size_t D = d;
  L.E = 0; L.Pe = (size_t)NI * D; L.blk0 = L.Pe + (size_t)len * D; L.blk_n = 6 * D * D + 10 * D;
  L.gf = L.blk0 + (size_t)n_blocks * L.blk_n; L.cf = L.gf + D; L.n = L.cf + D;
  return L;
}
struct SaBlk {
  size_t g1, c1, Wq, bq, Wk, bk, Wv, bv, Wo, bo, g2, c2, W1, b1, W2, b2;
};
static SaBlk sa_blk(const SaLayout& L, int b, int d) {
  const size_t D = d, DD = D * D;
  size_t o = L.blk0 + (size_t)b * L.blk_n;
  SaBlk k;
  k.g1 = o; o += D; k.c1 = o; o += D; k.Wq = o; o += DD; k.bq = o; o += D; k.Wk = o; o += DD; k.bk = o; o += D; k.Wv = o; o += DD;
  k.bv = o; o += D; k.Wo = o; o += DD; k.bo = o; o += D; k.g2 = o; o += D; k.c2 = o; o += D; k.W1 = o; o += DD; k.b1 = o; o += D;
  k.W2 = o; o += DD; k.b2 = o;
  return k;
}

// one mini-batch (or evaluation chunk) of nb pieces: slot b holds the plen[b] inputs items[pstart[b] ..], its positions are
// poff[b] .. poff[b] + plen[b] - 1, PS[p] = slot * L + t; a training piece's targets follow its inputs
struct SaDev {
  const int* items; const long long* pstart; const int* plen; const int* poff; int nb, P;
  const float* E; const float* Pe;
  int d, L, heads, dh;                                   // width, max_len (the mask and PS stride), heads, head width
  float sd, sh;                                          // float32 nearest sqrt(d) and 1 / sqrt(dh)
  unsigned seed, gstep, bsL; float retain;               // dropout: seed, global step, batch_size * max_len, retain (1: off)
  int train;
  int* PX; int* PY; int* PS;
};

// the dropout factor of unit u at position row ps of mask block blk (0: h0, b + 1: block b's residual branches)
__device__ __forceinline__ float sa_mask(const SaDev& s, unsigned stream, int blk, int ps, int u) {
  return s.retain < 1.f ? drop_scale(s.seed, s.gstep, stream, ((unsigned)blk * s.bsL + (unsigned)ps) * (unsigned)s.d + (unsigned)u, s.retain) : 1.f;
}

__device__ __forceinline__ float sa_warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// CTA per slot: positions, targets, mask rows and h0 = mask * (E[x] sd + Pe[t])
__global__ void __launch_bounds__(256) k_sa_embed(SaDev s, float* H0) {
  const int b = blockIdx.x, n = s.plen[b], p0 = s.poff[b];
  const long long s0 = s.pstart[b];
  for (int x = threadIdx.x; x < n * s.d; x += blockDim.x) {
    const int t = x / s.d, u = x % s.d, p = p0 + t, it = s.items[s0 + t];
    if (u == 0) { s.PX[p] = it; s.PY[p] = s.train ? s.items[s0 + t + 1] : -1; s.PS[p] = b * s.L + t; }
    const float h = __fadd_rn(__fmul_rn(s.E[(size_t)it * s.d + u], s.sd), s.Pe[(size_t)t * s.d + u]);
    H0[(size_t)p * s.d + u] = __fmul_rn(h, sa_mask(s, SA_STREAM_H0, 0, b * s.L + t, u));
  }
}

// warp per position: Y = g (x - mu) rs + c, mu the mean, rs = 1 / sqrt(mean of (x - mu)^2 + eps); mu and rs saved
__global__ void __launch_bounds__(256) k_sa_ln(const float* X, const float* g, const float* c, int P, int d, float* Y, float* MU, float* RS) {
  const int p = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= P) return;
  const float* x = X + (size_t)p * d;
  float s = 0.f;
  for (int u = lane; u < d; u += 32) s = __fadd_rn(s, x[u]);
  const float mu = __fdiv_rn(sa_warp_sum(s), (float)d);
  float v = 0.f;
  for (int u = lane; u < d; u += 32) { const float e = __fsub_rn(x[u], mu); v = __fmaf_rn(e, e, v); }
  const float rs = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fdiv_rn(sa_warp_sum(v), (float)d), SA_LN_EPS)));
  for (int u = lane; u < d; u += 32) Y[(size_t)p * d + u] = __fadd_rn(__fmul_rn(g[u], __fmul_rn(__fsub_rn(x[u], mu), rs)), c[u]);
  if (lane == 0) { MU[p] = mu; RS[p] = rs; }
}

// warp per position, the layer norm's backward: dy = dy1 (+ dy2) (+ dy3), xh = (x - mu) rs, e = dy g;
// DX = (dres +) rs ((e - mean e) - xh mean(e xh)); DY = dy and DYX = dy xh for the gain and bias gradients
__global__ void __launch_bounds__(256) k_sa_ln_bwd(const float* X, const float* MU, const float* RS, const float* g, const float* dy1, const float* dy2,
                                                   const float* dy3, const float* dres, int P, int d, float* DX, float* DY, float* DYX) {
  const int p = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= P) return;
  const size_t r = (size_t)p * d;
  const float mu = MU[p], rs = RS[p];
  auto dy = [&](int u) {
    float a = dy1[r + u];
    if (dy2) a = __fadd_rn(a, dy2[r + u]);
    if (dy3) a = __fadd_rn(a, dy3[r + u]);
    return a;
  };
  float s1 = 0.f, s2 = 0.f;
  for (int u = lane; u < d; u += 32) {
    const float xh = __fmul_rn(__fsub_rn(X[r + u], mu), rs), e = __fmul_rn(dy(u), g[u]);
    s1 = __fadd_rn(s1, e); s2 = __fmaf_rn(e, xh, s2);
  }
  const float m1 = __fdiv_rn(sa_warp_sum(s1), (float)d), m2 = __fdiv_rn(sa_warp_sum(s2), (float)d);
  for (int u = lane; u < d; u += 32) {
    const float xh = __fmul_rn(__fsub_rn(X[r + u], mu), rs), y = dy(u), e = __fmul_rn(y, g[u]);
    const float dx = __fmul_rn(rs, __fsub_rn(__fsub_rn(e, m1), __fmul_rn(xh, m2)));
    DX[r + u] = dres ? __fadd_rn(dres[r + u], dx) : dx;
    DY[r + u] = y; DYX[r + u] = __fmul_rn(y, xh);
  }
}

// X [n / d x d] += b (per column), with relu when RELU
template <bool RELU>
__global__ void k_sa_bias(float* X, const float* b, long long n, int d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = __fadd_rn(X[i], b[i % d]);
  X[i] = RELU ? fmaxf(v, 0.f) : v;
}

// a residual branch: OUT = HIN + mask * (T + b)
__global__ void k_sa_resid(SaDev s, float* OUT, const float* HIN, const float* T, const float* b, unsigned stream, int blk) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)s.P * s.d) return;
  const int p = (int)(i / s.d), u = (int)(i % s.d);
  OUT[i] = __fadd_rn(HIN[i], __fmul_rn(__fadd_rn(T[i], b[u]), sa_mask(s, stream, blk, s.PS[p], u)));
}

// OUT = IN * mask; OUT2 (may be null) = OUT * scale2
__global__ void k_sa_mask(SaDev s, const float* IN, unsigned stream, int blk, float* OUT, float* OUT2, float scale2) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)s.P * s.d) return;
  const int p = (int)(i / s.d), u = (int)(i % s.d);
  const float v = __fmul_rn(IN[i], sa_mask(s, stream, blk, s.PS[p], u));
  OUT[i] = v;
  if (OUT2) OUT2[i] = __fmul_rn(v, scale2);
}

// X = X where F > 0, else 0 (F the ReLU's output)
__global__ void k_sa_relu_bwd(float* X, const float* F, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(F[i] > 0.f)) X[i] = 0.f;
}

// the score of query position pq and key position pk in head columns c0 .. c0 + dh: sh * (Q . K), the dot in column order
__device__ __forceinline__ float sa_score(const SaDev& s, const float* Q, const float* K, size_t pq, size_t pk, int c0) {
  const float* q = Q + pq * s.d + c0;
  const float* k = K + pk * s.d + c0;
  float a = 0.f;
  for (int u = 0; u < s.dh; u++) a = __fmaf_rn(q[u], k[u], a);
  return __fmul_rn(a, s.sh);
}

// CTA per (query position, head): the causal softmax over the piece's keys 0 .. t (scores and probabilities in shared memory,
// max and sum thread-strided then a fixed tree), A_t = sum_j p_j V_j in key order; the max and sum saved for the backward
__global__ void __launch_bounds__(SA_ATT_THREADS) k_sa_att_fwd(SaDev s, const float* Q, const float* K, const float* V, float* A, float* M, float* LS) {
  __shared__ float sc[SA_LEN_MAX];
  __shared__ float red[32];
  const int p = blockIdx.x, h = blockIdx.y, t = s.PS[p] % s.L, p0 = p - t, c0 = h * s.dh;
  float m = -INFINITY;
  for (int j = threadIdx.x; j <= t; j += blockDim.x) { sc[j] = sa_score(s, Q, K, p, p0 + j, c0); m = fmaxf(m, sc[j]); }
  m = nm_block_reduce(m, red, true);
  float l = 0.f;
  for (int j = threadIdx.x; j <= t; j += blockDim.x) l = __fadd_rn(l, expf(__fsub_rn(sc[j], m)));
  l = nm_block_reduce(l, red, false);
  for (int j = threadIdx.x; j <= t; j += blockDim.x) sc[j] = __fdiv_rn(expf(__fsub_rn(sc[j], m)), l);
  __syncthreads();
  for (int u = threadIdx.x; u < s.dh; u += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j <= t; j++) a = __fmaf_rn(sc[j], V[(size_t)(p0 + j) * s.d + c0 + u], a);
    A[(size_t)p * s.d + c0 + u] = a;
  }
  if (threadIdx.x == 0) { M[(size_t)p * s.heads + h] = m; LS[(size_t)p * s.heads + h] = l; }
}

// CTA per (query position, head), the attention backward of the query: D_t = dA_t . A_t, dS_tj = p_tj (dA_t . V_j - D_t),
// dQ_t = sh sum_j dS_tj K_j; D_t saved for k_sa_att_bwd_kv
__global__ void __launch_bounds__(SA_ATT_THREADS) k_sa_att_bwd_q(SaDev s, const float* Q, const float* K, const float* V, const float* A, const float* dA,
                                                                 const float* M, const float* LS, float* dQ, float* DT) {
  __shared__ float ds[SA_LEN_MAX];
  __shared__ float red[32];
  const int p = blockIdx.x, h = blockIdx.y, t = s.PS[p] % s.L, p0 = p - t, c0 = h * s.dh;
  const float* da = dA + (size_t)p * s.d + c0;
  float D = 0.f;
  for (int u = threadIdx.x; u < s.dh; u += blockDim.x) D = __fmaf_rn(da[u], A[(size_t)p * s.d + c0 + u], D);
  D = nm_block_reduce(D, red, false);
  const float m = M[(size_t)p * s.heads + h], l = LS[(size_t)p * s.heads + h];
  for (int j = threadIdx.x; j <= t; j += blockDim.x) {
    const float pj = __fdiv_rn(expf(__fsub_rn(sa_score(s, Q, K, p, p0 + j, c0), m)), l);
    const float* v = V + (size_t)(p0 + j) * s.d + c0;
    float dp = 0.f;
    for (int u = 0; u < s.dh; u++) dp = __fmaf_rn(da[u], v[u], dp);
    ds[j] = __fmul_rn(pj, __fsub_rn(dp, D));
  }
  __syncthreads();
  for (int u = threadIdx.x; u < s.dh; u += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j <= t; j++) a = __fmaf_rn(ds[j], K[(size_t)(p0 + j) * s.d + c0 + u], a);
    dQ[(size_t)p * s.d + c0 + u] = __fmul_rn(a, s.sh);
  }
  if (threadIdx.x == 0) DT[(size_t)p * s.heads + h] = D;
}

// CTA per (key position j, head), the attention backward of the key and value: over the piece's queries i = j .. n - 1 in order,
// dV_j = sum_i p_ij dA_i, dK_j = sh sum_i dS_ij Q_i
__global__ void __launch_bounds__(SA_ATT_THREADS) k_sa_att_bwd_kv(SaDev s, const float* Q, const float* K, const float* V, const float* dA, const float* M,
                                                                  const float* LS, const float* DT, float* dK, float* dV) {
  __shared__ float pr[SA_LEN_MAX], ds[SA_LEN_MAX];
  const int p = blockIdx.x, h = blockIdx.y, j = s.PS[p] % s.L, p0 = p - j, n = s.plen[s.PS[p] / s.L], c0 = h * s.dh;
  const float* v = V + (size_t)p * s.d + c0;
  for (int i = j + (int)threadIdx.x; i < n; i += blockDim.x) {
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
    for (int i = j; i < n; i++) {
      const size_t o = (size_t)(p0 + i) * s.d + c0 + u;
      av = __fmaf_rn(pr[i], dA[o], av); ak = __fmaf_rn(ds[i], Q[o], ak);
    }
    dV[(size_t)p * s.d + c0 + u] = av; dK[(size_t)p * s.d + c0 + u] = __fmul_rn(ak, s.sh);
  }
}

// thread per (t, unit): gPe[t][u] = the sum over slots in order of D at the slot's position t (0 past every piece)
__global__ void k_sa_pe_grad(SaDev s, const float* D, float* gPe) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= s.L * s.d) return;
  const int t = x / s.d, u = x % s.d;
  float a = 0.f;
  for (int b = 0; b < s.nb; b++) if (s.plen[b] > t) a = __fadd_rn(a, D[(size_t)(s.poff[b] + t) * s.d + u]);
  gPe[x] = a;
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
// the per-position float arrays of P positions.  Training keeps every block's activations (blocks + 1 residual streams, the last
// one the encoder's output); evaluation keeps one block's and reuses them, and carries no backward buffers.
struct SaBuf {
  long long P = 0; bool keep = false; int blocks = 0;
  float *H, *U1, *Q, *K, *V, *A, *AR, *U2, *F1, *MU1, *RS1, *MU2, *RS2, *M, *LS;   // per block
  float *T, *MUF, *RSF, *QO;                                                     // a product's scratch; the final norm and q
  float *LOSS, *DQ, *DH, *DA, *DY, *DYX, *B[8], *DT;                             // the backward
  float* at(float* base, int width, int blk) const { return keep ? base + (size_t)blk * P * width : base; }
};
static size_t sa_pos_floats(int d, int heads, int blocks, bool train) {
  const size_t D = d, nb = train ? blocks : 1;
  size_t f = (nb + (train ? 1 : 0)) * D + nb * (8 * D + 4 + 2 * (size_t)heads) + 2 * D + 2;
  if (train) f += 1 + 13 * D + heads;
  return f;
}
static void sa_carve(SaBuf& B, float* f, long long P, int d, int heads, int blocks, bool train) {
  B.P = P; B.keep = train; B.blocks = blocks;
  const size_t nb = train ? blocks : 1;
  auto take = [&](float** q, size_t w) { *q = f; f += (size_t)P * w; };
  take(&B.H, (nb + (train ? 1 : 0)) * d);
  take(&B.U1, nb * d); take(&B.Q, nb * d); take(&B.K, nb * d); take(&B.V, nb * d); take(&B.A, nb * d); take(&B.AR, nb * d); take(&B.U2, nb * d);
  take(&B.F1, nb * d); take(&B.MU1, nb); take(&B.RS1, nb); take(&B.MU2, nb); take(&B.RS2, nb); take(&B.M, nb * heads); take(&B.LS, nb * heads);
  take(&B.T, d); take(&B.QO, d); take(&B.MUF, 1); take(&B.RSF, 1);
  if (!train) return;
  take(&B.LOSS, 1); take(&B.DQ, d); take(&B.DH, d); take(&B.DA, d); take(&B.DY, d); take(&B.DYX, d);
  for (int k = 0; k < 8; k++) take(&B.B[k], d);
  take(&B.DT, heads);
}

static unsigned sa_grid(long long n) { return (unsigned)((n + 255) / 256); }

// the encoder of a batch or chunk: QO [P x d] (part: split scratch; encoder products never split)
static void sa_encode(cudaStream_t st, const SaDev& s, const SaBuf& B, const float* th, const SaLayout& Lo, int blocks, float* part) {
  const int P = s.P, d = s.d;
  const long long n = (long long)P * d;
  const unsigned gl = (unsigned)((P + 7) / 8), ge = sa_grid(n);
  k_sa_embed<<<s.nb, 256, 0, st>>>(s, B.at(B.H, d, 0));
  for (int b = 0; b < blocks; b++) {
    const SaBlk k = sa_blk(Lo, b, d);
    float *hin = B.at(B.H, d, b), *u1 = B.at(B.U1, d, b), *q = B.at(B.Q, d, b), *kk = B.at(B.K, d, b), *v = B.at(B.V, d, b), *a = B.at(B.A, d, b);
    float *ar = B.at(B.AR, d, b), *u2 = B.at(B.U2, d, b), *f1 = B.at(B.F1, d, b), *hout = B.at(B.H, d, b + 1);
    k_sa_ln<<<gl, 256, 0, st>>>(hin, th + k.g1, th + k.c1, P, d, u1, B.at(B.MU1, 1, b), B.at(B.RS1, 1, b));
    nm_gemm<NM_ENCODER>(st, part, u1, d, 1, th + k.Wq, d, 1, q, d, P, d, d);
    nm_gemm<NM_ENCODER>(st, part, u1, d, 1, th + k.Wk, d, 1, kk, d, P, d, d);
    nm_gemm<NM_ENCODER>(st, part, u1, d, 1, th + k.Wv, d, 1, v, d, P, d, d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(q, th + k.bq, n, d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(kk, th + k.bk, n, d);
    k_sa_bias<false><<<ge, 256, 0, st>>>(v, th + k.bv, n, d);
    k_sa_att_fwd<<<dim3((unsigned)P, (unsigned)s.heads), SA_ATT_THREADS, 0, st>>>(s, q, kk, v, a, B.at(B.M, s.heads, b), B.at(B.LS, s.heads, b));
    nm_gemm<NM_ENCODER>(st, part, a, d, 1, th + k.Wo, d, 1, B.T, d, P, d, d);
    k_sa_resid<<<ge, 256, 0, st>>>(s, ar, hin, B.T, th + k.bo, SA_STREAM_ATT, b + 1);
    k_sa_ln<<<gl, 256, 0, st>>>(ar, th + k.g2, th + k.c2, P, d, u2, B.at(B.MU2, 1, b), B.at(B.RS2, 1, b));
    nm_gemm<NM_ENCODER>(st, part, u2, d, 1, th + k.W1, d, 1, f1, d, P, d, d);
    k_sa_bias<true><<<ge, 256, 0, st>>>(f1, th + k.b1, n, d);
    nm_gemm<NM_ENCODER>(st, part, f1, d, 1, th + k.W2, d, 1, B.T, d, P, d, d);
    k_sa_resid<<<ge, 256, 0, st>>>(s, hout, ar, B.T, th + k.b2, SA_STREAM_FFN, b + 1);
  }
  k_sa_ln<<<gl, 256, 0, st>>>(B.at(B.H, d, blocks), th + Lo.gf, th + Lo.cf, P, d, B.QO, B.MUF, B.RSF);
}

// G[off ..] = the column sums of X [P x d] in position order (bias and gain gradients)
static void sa_colsum(cudaStream_t st, float* part, const float* ones, const float* X, float* G, int P, int d) {
  nm_gemm<NM_BACKWARD>(st, part, ones, 0, 0, X, d, 1, G, d, 1, d, P);
}
// the gradient of a product Y = X W (+ b) given dY: G.W = X^T dY, G.b = column sums of dY, and dX = dY W^T (dX may be null)
static void sa_linear_bwd(cudaStream_t st, float* part, const float* ones, const float* X, const float* W, const float* dY, float* gW, float* gb, float* dX,
                          int P, int d) {
  nm_gemm<NM_BACKWARD>(st, part, X, 1, d, dY, d, 1, gW, d, d, d, P);
  sa_colsum(st, part, ones, dY, gb, P, d);
  if (dX) nm_gemm<NM_BACKWARD>(st, part, dY, d, 1, W, 1, d, dX, d, P, d, d);
}

// a batch's loss and gradient G (flat, the parameters' layout) at the handle's parameters; loss_out a device float
static void sa_grad(cudaStream_t st, const SaDev& s, const SaBuf& B, const NmScratch& ns, const float* th, const SaLayout& Lo, int blocks, int NI,
                    float* G, const float* ones, float* loss_out) {
  const int P = s.P, d = s.d;
  const long long n = (long long)P * d;
  const unsigned gl = (unsigned)((P + 7) / 8), ge = sa_grid(n);
  float* part = ns.part;
  sa_encode(st, s, B, th, Lo, blocks, part);
  // the catalogue: logits, the softmax gradient, dL/dq and dE
  NmDev nd{};
  nd.P = P; nd.d = d; nd.NI = NI; nd.S = ns.S; nd.PY = s.PY; nd.PX = s.PX; nd.PS = s.PS; nd.LOSS = B.LOSS; nd.re = 1.f;
  const float* E = th + Lo.E;
  nm_gemm<NM_CATALOGUE>(st, part, B.QO, d, 1, E, 1, d, ns.S, NI, P, NI, d);
  k_nm_softmax<<<P, 256, 0, st>>>(nd);
  k_nm_mean<<<1, 1024, 0, st>>>(B.LOSS, P, loss_out);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, NI, 1, E, d, 1, B.DQ, d, P, d, NI);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, 1, NI, B.QO, d, 1, G + Lo.E, d, NI, d, P);
  // the final norm
  k_sa_ln_bwd<<<gl, 256, 0, st>>>(B.at(B.H, d, blocks), B.MUF, B.RSF, th + Lo.gf, B.DQ, nullptr, nullptr, nullptr, P, d, B.DH, B.DY, B.DYX);
  sa_colsum(st, part, ones, B.DYX, G + Lo.gf, P, d);
  sa_colsum(st, part, ones, B.DY, G + Lo.cf, P, d);
  float* const* T = B.B;
  for (int b = blocks - 1; b >= 0; b--) {
    const SaBlk k = sa_blk(Lo, b, d);
    const int hs = s.heads;
    float *hin = B.at(B.H, d, b), *u1 = B.at(B.U1, d, b), *q = B.at(B.Q, d, b), *kk = B.at(B.K, d, b), *v = B.at(B.V, d, b), *a = B.at(B.A, d, b);
    float *ar = B.at(B.AR, d, b), *u2 = B.at(B.U2, d, b), *f1 = B.at(B.F1, d, b);
    // the FFN: h' = ar + mask (relu(u2 W1 + b1) W2 + b2)
    k_sa_mask<<<ge, 256, 0, st>>>(s, B.DH, SA_STREAM_FFN, b + 1, T[0], nullptr, 1.f);
    sa_linear_bwd(st, part, ones, f1, th + k.W2, T[0], G + k.W2, G + k.b2, T[1], P, d);
    k_sa_relu_bwd<<<ge, 256, 0, st>>>(T[1], f1, n);
    sa_linear_bwd(st, part, ones, u2, th + k.W1, T[1], G + k.W1, G + k.b1, T[2], P, d);
    k_sa_ln_bwd<<<gl, 256, 0, st>>>(ar, B.at(B.MU2, 1, b), B.at(B.RS2, 1, b), th + k.g2, T[2], nullptr, nullptr, B.DH, P, d, B.DA, B.DY, B.DYX);
    sa_colsum(st, part, ones, B.DYX, G + k.g2, P, d);
    sa_colsum(st, part, ones, B.DY, G + k.c2, P, d);
    // the attention: ar = hin + mask (A Wo + bo)
    k_sa_mask<<<ge, 256, 0, st>>>(s, B.DA, SA_STREAM_ATT, b + 1, T[0], nullptr, 1.f);
    sa_linear_bwd(st, part, ones, a, th + k.Wo, T[0], G + k.Wo, G + k.bo, T[1], P, d);
    const dim3 ga((unsigned)P, (unsigned)hs);
    k_sa_att_bwd_q<<<ga, SA_ATT_THREADS, 0, st>>>(s, q, kk, v, a, T[1], B.at(B.M, hs, b), B.at(B.LS, hs, b), T[2], B.DT);
    k_sa_att_bwd_kv<<<ga, SA_ATT_THREADS, 0, st>>>(s, q, kk, v, T[1], B.at(B.M, hs, b), B.at(B.LS, hs, b), B.DT, T[3], T[4]);
    sa_linear_bwd(st, part, ones, u1, th + k.Wq, T[2], G + k.Wq, G + k.bq, T[5], P, d);
    sa_linear_bwd(st, part, ones, u1, th + k.Wk, T[3], G + k.Wk, G + k.bk, T[6], P, d);
    sa_linear_bwd(st, part, ones, u1, th + k.Wv, T[4], G + k.Wv, G + k.bv, T[7], P, d);
    k_sa_ln_bwd<<<gl, 256, 0, st>>>(hin, B.at(B.MU1, 1, b), B.at(B.RS1, 1, b), th + k.g1, T[5], T[6], T[7], B.DA, P, d, B.DH, B.DY, B.DYX);
    sa_colsum(st, part, ones, B.DYX, G + k.g1, P, d);
    sa_colsum(st, part, ones, B.DY, G + k.c1, P, d);
  }
  // h0 = mask (E[x] sd + Pe[t]): T0 = dh0 mask for Pe, T1 = T0 sd the input-embedding rows
  k_sa_mask<<<ge, 256, 0, st>>>(s, B.DH, SA_STREAM_H0, 0, T[0], T[1], s.sd);
  k_sa_pe_grad<<<sa_grid((long long)s.L * d), 256, 0, st>>>(s, T[0], G + Lo.Pe);
  nd.DEMB = T[1];
  k_nm_keys<<<(P + 255) / 256, 256, 0, st>>>(s.PX, P, ns.keys);
  int end_bit = 33;
  while (end_bit < 64 && ((unsigned long long)NI >> (end_bit - 32)) != 0ull) end_bit++;
  size_t cb = ns.cub_bytes;
  cub::DeviceRadixSort::SortKeys(ns.cub, cb, ns.keys, ns.keys2, P, 0, end_bit, st);
  k_nm_scatter<<<sa_grid(n), 256, 0, st>>>(nd, ns.keys2, G + Lo.E);
}

static bool sa_shape_ok(int d, int blocks, int heads, int len) {
  return blocks >= 1 && blocks <= SA_BLOCKS_MAX && heads >= 1 && heads <= d && d % heads == 0 && len >= 1 && len <= SA_LEN_MAX;
}
#define SA_SHAPE_MSG ": need n_blocks in 1 .. 8, n_heads dividing the embedding and max_len in 1 .. 512"

// the model buffers of a SASRec handle (NARM's fields): parameters, double(E) and zero biases for bpr_blocks, a device 1.0f
static int sa_set_model(g4r_baselines* h, int32_t blocks, int32_t heads, int32_t max_len, const float* params, int64_t n_params, const char* who) {
  if (!params) FAIL(G4R_ERR_INVALID, std::string(who) + ": null parameters");
  if (!sa_shape_ok(h->n_keep, blocks, heads, max_len)) FAIL(G4R_ERR_INVALID, std::string(who) + SA_SHAPE_MSG);
  const SaLayout L = sa_layout(h->n_items, h->n_keep, blocks, max_len);
  if (n_params != (int64_t)L.n)
    FAIL(G4R_ERR_INVALID, std::string(who) + ": need n_params = n_items d + max_len d + n_blocks (6 d^2 + 10 d) + 2 d = " + std::to_string(L.n));
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
  h->sa_blocks = blocks; h->sa_heads = heads; h->nm_len = max_len; h->nm_n = L.n;
  const size_t nE = (size_t)h->n_items * h->n_keep;
  k_nm_to_double<<<(unsigned)((nE + 255) / 256), 256, 0, st>>>(h->dNmTh, nE, h->dI);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_sasrec_import(g4r_baselines* h, int32_t n_blocks, int32_t n_heads, int32_t max_len, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SASREC) FAIL(G4R_ERR_STATE, "g4r_bl_sasrec_import: the handle is not a SASRec");
  return sa_set_model(h, n_blocks, n_heads, max_len, params, n_params, "g4r_bl_sasrec_import");
}

extern "C" int g4r_bl_sasrec_export(g4r_baselines* h, float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SASREC || !h->dNmTh) FAIL(G4R_ERR_STATE, "g4r_bl_sasrec_export: no SASRec parameters (g4r_bl_sasrec_begin or g4r_bl_sasrec_import)");
  if (!params || n_params != (int64_t)h->nm_n) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_export: need n_params floats");
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(params, h->dNmTh, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

extern "C" int g4r_bl_sasrec_begin(g4r_baselines* h, int32_t n_blocks, int32_t n_heads, int32_t max_len, int32_t batch_size, const int64_t* piece_offsets,
                                   int64_t n_pieces, const int32_t* items, int64_t n_entries, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SASREC) FAIL(G4R_ERR_STATE, "g4r_bl_sasrec_begin: the handle is not a SASRec");
  if (!piece_offsets || !items || n_pieces < 1 || n_entries < 2 || batch_size < 1)
    FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_begin: null argument, no pieces or batch_size < 1");
  const int NI = h->n_items, dd = h->n_keep;
  if (!sa_shape_ok(dd, n_blocks, n_heads, max_len)) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_begin" SA_SHAPE_MSG);
  if (n_entries > INT32_MAX || n_pieces > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_begin: more than 2^31 - 1 entries or pieces");
  if (piece_offsets[0] != 0 || piece_offsets[n_pieces] != n_entries) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_begin: piece offsets must run from 0 to n_entries");
  std::vector<int> lens(n_pieces);
  for (int64_t k = 0; k < n_pieces; k++) {
    const int64_t n = piece_offsets[k + 1] - piece_offsets[k];
    if (n < 2 || n > (int64_t)max_len + 1) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_begin: every piece needs 2 .. max_len + 1 events");
    lens[k] = (int)n - 1;
  }
  for (int64_t e = 0; e < n_entries; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_sasrec_begin: item index out of range");
  if ((uint64_t)(n_blocks + 1) * (uint64_t)batch_size * (uint64_t)max_len * (uint64_t)dd >= 0x100000000ull)
    FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_begin: (n_blocks + 1) * batch_size * max_len * d must stay below 2^32 (dropout indices)");
  // the largest batch: the batch_size longest pieces
  std::vector<int> srt(lens);
  std::sort(srt.begin(), srt.end(), std::greater<int>());
  long long Pmax = 0;
  for (int64_t k = 0; k < std::min<int64_t>(batch_size, n_pieces); k++) Pmax += srt[k];
  const SaLayout L = sa_layout(NI, dd, n_blocks, max_len);
  const size_t act = (size_t)Pmax * sa_pos_floats(dd, n_heads, n_blocks, true) * 4;
  const size_t need = (size_t)Pmax * ((size_t)NI * 4 + 28) + act + NM_PART_CAP * 4 + 3 * L.n * 4 + (size_t)n_entries * 4 + (size_t)n_pieces * 16 +
                      ((size_t)64 << 20);
  int rc = sa_set_model(h, n_blocks, n_heads, max_len, params, n_params, "g4r_bl_sasrec_begin");
  if (rc) return rc;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    h->err = "g4r_bl_sasrec_begin: the fit needs " + std::to_string(need) + " bytes of device memory (the logits of the largest batch " +
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
  CK(take(&h->sa_f, (size_t)Pmax * sa_pos_floats(dd, n_heads, n_blocks, true)));
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

// the SaDev of a handle's parameters (plan pointers and nb / P set by the caller)
static SaDev sa_dev(const g4r_baselines* h, const SaLayout& Lo) {
  SaDev s{};
  s.E = h->dNmTh + Lo.E; s.Pe = h->dNmTh + Lo.Pe;
  s.d = h->n_keep; s.L = h->nm_len; s.heads = h->sa_heads; s.dh = h->n_keep / h->sa_heads;
  s.sd = (float)std::sqrt((double)h->n_keep); s.sh = (float)(1.0 / std::sqrt((double)s.dh));
  s.retain = 1.f; s.bsL = (unsigned)h->nm_bs * (unsigned)h->nm_len;
  return s;
}

static SaDev sa_train_dev(g4r_baselines* h, const SaLayout& Lo, unsigned seed, unsigned gstep, float dropout) {
  SaDev s = sa_dev(h, Lo);
  const NmScratch& ns = h->nm_s;
  s.items = h->dNmItems; s.train = 1; s.seed = seed; s.gstep = gstep; s.retain = dropout > 0.f ? 1.f - dropout : 1.f;
  s.PX = ns.PX; s.PY = ns.PY; s.PS = ns.PS; s.pstart = ns.pstart; s.plen = ns.plen; s.poff = ns.poff;
  return s;
}

static int sa_check_run(g4r_baselines* h, const int32_t* pieces, int64_t n, float dropout, const char* who) {
  if (h->kind != BL_SASREC) FAIL(G4R_ERR_STATE, std::string(who) + ": the handle is not a SASRec");
  if (!h->nm_fit) FAIL(G4R_ERR_STATE, std::string(who) + ": no fit begun (g4r_bl_sasrec_begin)");
  if (!pieces || n < 1) FAIL(G4R_ERR_INVALID, std::string(who) + ": no pieces");
  if (!(dropout >= 0.f && dropout < 1.f)) FAIL(G4R_ERR_INVALID, std::string(who) + ": dropout must be in [0, 1)");
  const int64_t np = (int64_t)h->nm_off.size() - 1;
  for (int64_t q = 0; q < n; q++) if (pieces[q] < 0 || pieces[q] >= np) FAIL(G4R_ERR_INDEX, std::string(who) + ": piece index out of range");
  return G4R_OK;
}

extern "C" int g4r_bl_sasrec_grads(g4r_baselines* h, const int32_t* pieces, int32_t n, uint32_t seed, int64_t step, float dropout, float* loss,
                                   float* grads) {
  if (!h) return G4R_ERR_INVALID;
  int rc = sa_check_run(h, pieces, n, dropout, "g4r_bl_sasrec_grads");
  if (rc) return rc;
  if (n > h->nm_bs || !grads || step < 0 || step > 0xffffffffll) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_grads: need n <= batch_size, grads and step in 0 .. 2^32 - 1");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = nm_plan(h, pieces, n, ps, pl, po, batches, "g4r_bl_sasrec_grads");
  if (rc) return rc;
  cudaSetDevice(h->device);
  rc = nm_upload_plan(h, ps, pl, po, 0, n);
  if (rc) return rc;
  const SaLayout Lo = sa_layout(h->n_items, h->n_keep, h->sa_blocks, h->nm_len);
  SaDev s = sa_train_dev(h, Lo, seed, (unsigned)step, dropout);
  s.nb = n; s.P = batches[0].second;
  SaBuf B;
  sa_carve(B, h->sa_f, h->nm_Pmax, h->n_keep, h->sa_heads, h->sa_blocks, true);
  sa_grad(h->stream, s, B, h->nm_s, h->dNmTh, Lo, h->sa_blocks, h->n_items, h->dNmG, h->dNmOne, h->dNmLoss);
  CK(cudaGetLastError());
  float l = 0.f;
  CK(cudaMemcpyAsync(&l, h->dNmLoss, sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(grads, h->dNmG, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (loss) *loss = l;
  return G4R_OK;
}

extern "C" int g4r_bl_sasrec_epoch(g4r_baselines* h, const int32_t* order, int64_t n_order, uint32_t seed, float learning_rate, float dropout,
                                   float* losses, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  int rc = sa_check_run(h, order, n_order, dropout, "g4r_bl_sasrec_epoch");
  if (rc) return rc;
  if (!(learning_rate > 0.f && std::isfinite(learning_rate))) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_epoch: learning_rate must be finite and > 0");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = nm_plan(h, order, n_order, ps, pl, po, batches, "g4r_bl_sasrec_epoch");
  if (rc) return rc;
  if (h->nm_step + (int64_t)batches.size() > 0xffffffffll) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_epoch: more than 2^32 steps since the fit began");
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  const SaLayout Lo = sa_layout(h->n_items, h->n_keep, h->sa_blocks, h->nm_len);
  SaBuf B;
  sa_carve(B, h->sa_f, h->nm_Pmax, h->n_keep, h->sa_heads, h->sa_blocks, true);
  // the whole epoch's plan goes up once; each batch reads its slice
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr; float* dloss = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  CK(bb.take(&dloss, batches.size()));
  CK(cudaEventRecord(h->ev0, st));
  for (size_t b = 0; b < batches.size(); b++) {
    const int64_t q0 = batches[b].first;
    SaDev s = sa_train_dev(h, Lo, seed, (unsigned)h->nm_step, dropout);
    s.pstart = dps + q0; s.plen = dpl + q0; s.poff = dpo + q0; s.nb = (int)std::min<int64_t>(h->nm_bs, n_order - q0); s.P = batches[b].second;
    sa_grad(st, s, B, h->nm_s, h->dNmTh, Lo, h->sa_blocks, h->n_items, h->dNmG, h->dNmOne, dloss + b);
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

// every counted event's q (eval mode: no dropout; the last max_len inputs of its prefix) into qev [n_ev x d] on the device
static int sa_encode_events(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* off, int64_t n_sessions, const int32_t* n_history,
                            const std::vector<int64_t>& ev0, float* qev) {
  const int dd = h->n_keep;
  cudaStream_t st = h->stream;
  const SaLayout Lo = sa_layout(h->n_items, dd, h->sa_blocks, h->nm_len);
  BlBufs bb;
  int *PX = nullptr, *PY = nullptr, *PS = nullptr, *dEv = nullptr, *dPair = nullptr, *plen = nullptr, *poff = nullptr;
  long long* pstart = nullptr;
  float* f = nullptr;
  const int* dItems = nullptr;
  CK(bb.take(&PX, SA_EVAL_PAIRS)); CK(bb.take(&PY, SA_EVAL_PAIRS)); CK(bb.take(&PS, SA_EVAL_PAIRS));
  CK(bb.take(&dEv, SA_EVAL_PAIRS)); CK(bb.take(&dPair, SA_EVAL_PAIRS));
  CK(bb.take(&pstart, SA_EVAL_PAIRS)); CK(bb.take(&plen, SA_EVAL_PAIRS)); CK(bb.take(&poff, SA_EVAL_PAIRS));
  CK(bb.take(&f, (size_t)SA_EVAL_PAIRS * sa_pos_floats(dd, h->sa_heads, h->sa_blocks, false)));
  CK(bb.put(&dItems, items, n_events, st));
  SaBuf B;
  sa_carve(B, f, SA_EVAL_PAIRS, dd, h->sa_heads, h->sa_blocks, false);
  SaDev s = sa_dev(h, Lo);
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
    sa_encode(st, s, B, h->dNmTh, Lo, h->sa_blocks, nullptr);
    const int ne = (int)ev.size();
    k_nm_pick<<<(unsigned)(((long long)ne * dd + 255) / 256), 256, 0, st>>>(B.QO, dEv, dPair, ne, dd, qev);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));                      // the host arrays are reused by the next chunk
    return G4R_OK;
  };
  return nm_event_chunks(h->nm_len, SA_EVAL_PAIRS, off, n_sessions, n_history, ev0, flush);
}

extern "C" int g4r_bl_sasrec_encode(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                                    const int32_t* n_history, float* q, int64_t n_q) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SASREC || !h->ready) FAIL(G4R_ERR_STATE, "g4r_bl_sasrec_encode: no SASRec parameters (g4r_bl_sasrec_begin or g4r_bl_sasrec_import)");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || n_q < 0 || (n_q > 0 && !q))
    FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_encode: null or out-of-range argument");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_encode: session offsets must rise from 0 to n_events");
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= h->n_items) FAIL(G4R_ERR_INDEX, "g4r_bl_sasrec_encode: item index out of range");
  std::vector<int64_t> ev0;
  int rc = bl_counted(h, "g4r_bl_sasrec_encode", session_offsets, n_sessions, n_history, ev0);
  if (rc) return rc;
  if (n_q != ev0[n_sessions]) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_encode: n_q must be the number of counted events");
  if (n_q > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_sasrec_encode: more than 2^31 - 1 counted events");
  cudaSetDevice(h->device);
  BlBufs bb;
  float* dq = nullptr;
  CK(bb.take(&dq, (size_t)n_q * h->n_keep));
  rc = sa_encode_events(h, items, n_events, session_offsets, n_sessions, n_history, ev0, dq);
  if (rc) return rc;
  if (n_q) CK(cudaMemcpyAsync(q, dq, (size_t)n_q * h->n_keep * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// the ranking of a g4r_bl_evaluate call of a SASRec: every counted event's q, then BPR's ranking with I = double(E), bI = 0
static int sasrec_rank(g4r_baselines* h, BlCall& c) {
  float* dq = nullptr;
  CK(c.bb.take(&dq, (size_t)c.n_ev * h->n_keep));
  const int rc = sa_encode_events(h, c.items, c.n_events, c.off, c.n_sessions, c.n_history, c.ev0, dq);
  if (rc) return rc;
  return bpr_blocks(h, c, dq);
}
