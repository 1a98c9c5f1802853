// g4r_narm.cuh -- the NARM neural session baseline on the device (DESIGN §3s): a GRU encoder with NARM's item-level attention,
// a bilinear decoder against the item table and full-catalogue cross-entropy, trained with dense Adam; and the eval-mode encoder
// that feeds per-event vectors to BPR's ranking.  Every reduction runs in a fixed order (no floating-point atomics), so a fit is
// bitwise reproducible and independent of grid sizes.  Included at the end of g4r_lib.cu after g4r_bpr.cuh (BprEvalDev,
// bpr_blocks) and g4r_kernels.cuh (drop_scale).
#pragma once

constexpr int NM_BM = 64, NM_BN = 64, NM_BK = 16;       // product tile: rows x columns x k per shared-memory stage
constexpr int NM_KCHUNK = 512;                          // k per split of a product with few output tiles
constexpr int NM_SPLIT_TILES = 264;                     // products with fewer output tiles than this split k
constexpr size_t NM_PART_CAP = (size_t)16 << 20;        // floats of split partials
constexpr int NM_EVAL_PAIRS = 32768;                    // encoder positions per evaluation chunk
constexpr unsigned NM_STREAM_EMB = 200u, NM_STREAM_CT = 201u;   // dropout streams: embeddings, c
constexpr int NM_H_MAX = 1024, NM_LEN_MAX = 512;

// offsets of the parameters in the flat float32 vector: E, Wx, Wrz, Wh, Bh, A1, A2, v, B
struct NmLayout {
  size_t E, Wx, Wrz, Wh, Bh, A1, A2, v, B, n;
};
static NmLayout nm_layout(int NI, int d, int H) {
  NmLayout L;
  L.E = 0; L.Wx = L.E + (size_t)NI * d; L.Wrz = L.Wx + (size_t)d * 3 * H; L.Wh = L.Wrz + (size_t)H * 2 * H; L.Bh = L.Wh + (size_t)H * H;
  L.A1 = L.Bh + 3 * (size_t)H; L.A2 = L.A1 + (size_t)H * H; L.v = L.A2 + (size_t)H * H; L.B = L.v + H; L.n = L.B + (size_t)d * 2 * H;
  return L;
}

// ---------------------------------------------------------------------------------------------------------------------------
// one fp32 product C[m, n] = sum over k in order of A(m, k) * B(k, n), A(m, k) = A[m lam + k lak], B(k, n) = B[k lbk + n lbn].
// Each output is one thread's sequential fmaf chain over its k range; with gridDim.z > 1 the ranges go to part[z] and
// k_nm_gsum adds them in z order.  The split depends only on the shape, so the result does too.  blockIdx.x is the output tile
// (column tiles fastest), so the number of row tiles is not bounded by gridDim.y.  ROLE only names the instance (profiles
// tell the catalogue products apart): NM_ENCODER products never split k, so an event's q does not depend on how many other
// positions share its evaluation chunk.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int NM_ENCODER = 0, NM_CATALOGUE = 1, NM_BACKWARD = 2;

template <int ROLE>
__global__ void __launch_bounds__(256) k_nm_gemm(const float* A, long long lam, long long lak, const float* B, long long lbk, long long lbn,
                                                 float* C, long long ldc, int M, int N, int K, int kchunk, float* part) {
  __shared__ float sA[NM_BK][NM_BM + 1];
  __shared__ float sB[NM_BK][NM_BN + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n_tiles = (N + NM_BN - 1) / NM_BN;
  const int m0 = (int)(blockIdx.x / n_tiles) * NM_BM, n0 = (int)(blockIdx.x % n_tiles) * NM_BN;
  const int k_beg = blockIdx.z * kchunk, k_end = min(K, k_beg + kchunk);
  float acc[4][4];
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) acc[r][c] = 0.f;
  for (int k0 = k_beg; k0 < k_end; k0 += NM_BK) {
    __syncthreads();
    for (int x = tid; x < NM_BK * NM_BM; x += 256) {   // consecutive threads walk the operand's unit-stride index
      int kk = lak == 1 ? x % NM_BK : x / NM_BM, r = lak == 1 ? x / NM_BK : x % NM_BM;
      const int m = m0 + r;
      sA[kk][r] = (m < M && k0 + kk < k_end) ? A[m * lam + (k0 + kk) * lak] : 0.f;
      kk = lbk == 1 ? x % NM_BK : x / NM_BN; r = lbk == 1 ? x / NM_BK : x % NM_BN;
      const int n = n0 + r;
      sB[kk][r] = (n < N && k0 + kk < k_end) ? B[(k0 + kk) * lbk + n * lbn] : 0.f;
    }
    __syncthreads();
    const int kn = min(NM_BK, k_end - k0);
    for (int kk = 0; kk < kn; kk++) {
      float a[4], b[4];
      for (int r = 0; r < 4; r++) a[r] = sA[kk][ty + 16 * r];
      for (int c = 0; c < 4; c++) b[c] = sB[kk][tx + 16 * c];
      for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) acc[r][c] = __fmaf_rn(a[r], b[c], acc[r][c]);
    }
  }
  for (int r = 0; r < 4; r++) {
    const int m = m0 + ty + 16 * r;
    if (m >= M) continue;
    for (int c = 0; c < 4; c++) {
      const int n = n0 + tx + 16 * c;
      if (n >= N) continue;
      if (gridDim.z == 1) C[m * ldc + n] = acc[r][c];
      else part[((size_t)blockIdx.z * M + m) * N + n] = acc[r][c];
    }
  }
}

template <int ROLE>
__global__ void k_nm_gsum(const float* part, int splits, int M, int N, float* C, long long ldc) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * N) return;
  float s = part[i];
  for (int z = 1; z < splits; z++) s = __fadd_rn(s, part[(size_t)z * M * N + i]);
  C[(i / N) * ldc + i % N] = s;
}

template <int ROLE>
static void nm_gemm(cudaStream_t st, float* part, const float* A, long long lam, long long lak, const float* B, long long lbk, long long lbn,
                    float* C, long long ldc, int M, int N, int K) {
  if (M <= 0 || N <= 0) return;
  const long long tiles = (long long)((M + NM_BM - 1) / NM_BM) * ((N + NM_BN - 1) / NM_BN);
  int splits = 1;
  if (ROLE != NM_ENCODER && tiles < NM_SPLIT_TILES)
    splits = (int)std::max<long long>(1, std::min<long long>({64ll, ((long long)K + NM_KCHUNK - 1) / NM_KCHUNK, (long long)(NM_PART_CAP / ((size_t)M * N))}));
  int kchunk = (K + splits - 1) / splits;
  kchunk = std::max(NM_BK, (kchunk + NM_BK - 1) / NM_BK * NM_BK);
  splits = std::max(1, (K + kchunk - 1) / kchunk);
  const dim3 grid((unsigned)tiles, 1, (unsigned)splits);
  k_nm_gemm<ROLE><<<grid, 256, 0, st>>>(A, lam, lak, B, lbk, lbn, C, ldc, M, N, K, kchunk, part);
  if (splits > 1) k_nm_gsum<ROLE><<<(unsigned)(((long long)M * N + 255) / 256), 256, 0, st>>>(part, splits, M, N, C, ldc);
}

// ---------------------------------------------------------------------------------------------------------------------------
// the encoder, one mini-batch (or evaluation chunk) of nb pieces: slot b holds the plen[b] inputs items[pstart[b] ..], its
// positions are pairs poff[b] .. poff[b] + plen[b] - 1; a training piece's targets follow its inputs
// ---------------------------------------------------------------------------------------------------------------------------
struct NmDev {
  const int* items; const long long* pstart; const int* plen; const int* poff; int nb, P;
  const float* E; const float* Wx; const float* Wrz; const float* Wh; const float* Bh; const float* A1; const float* A2; const float* v;
  const float* B;
  int NI, d, H, L;                                       // items, d_e, hidden, max_len (the mask and attention row stride)
  unsigned seed, gstep; float re, rc;                    // dropout: seed, global step, retain of the embeddings and of c (1: off)
  int train;
  int* PX; int* PY; int* PS;                             // per position: input, target (-1: none), mask row (slot * L + t)
  float *EMB, *VEC, *HH, *R, *Z, *HT, *HP, *HR, *A1H, *A2H, *AL, *C, *Q;
  float *S, *LOSS, *DQ, *DC, *DA, *G1, *G2, *DV, *DHA, *T1, *T2, *DVEC, *DEMB;
};

__device__ __forceinline__ float nm_sig(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }
__device__ __forceinline__ float nm_mask(const NmDev& d, unsigned stream, int row, int dim, int u, float retain) {
  return retain < 1.f ? drop_scale(d.seed, d.gstep, stream, (unsigned)row * (unsigned)dim + (unsigned)u, retain) : 1.f;
}

// CTA per slot: positions, targets, mask rows and the (dropped-out) input embeddings
__global__ void __launch_bounds__(256) k_nm_gather(NmDev d) {
  const int b = blockIdx.x, n = d.plen[b], p0 = d.poff[b];
  const long long s0 = d.pstart[b];
  for (int x = threadIdx.x; x < n * d.d; x += blockDim.x) {
    const int t = x / d.d, u = x % d.d, p = p0 + t, it = d.items[s0 + t];
    if (u == 0) { d.PX[p] = it; d.PY[p] = d.train ? d.items[s0 + t + 1] : -1; d.PS[p] = b * d.L + t; }
    d.EMB[(size_t)p * d.d + u] = d.E[(size_t)it * d.d + u] * nm_mask(d, NM_STREAM_EMB, b * d.L + t, d.d, u, d.re);
  }
}

// CTA per slot: the GRU over its positions from a zero state; VEC = EMB Wx (without Bh) is precomputed
__global__ void __launch_bounds__(256) k_nm_gru_fwd(NmDev d) {
  extern __shared__ float sm[];
  const int H = d.H, b = blockIdx.x, n = d.plen[b], p0 = d.poff[b];
  float* hp = sm;                                        // [H] h of the previous position
  float* hr = sm + H;                                    // [H] hp * r
  for (int k = threadIdx.x; k < H; k += blockDim.x) hp[k] = 0.f;
  __syncthreads();
  for (int t = 0; t < n; t++) {
    const size_t p = (size_t)(p0 + t);
    const float* vec = d.VEC + p * 3 * H;
    for (int c = threadIdx.x; c < 2 * H; c += blockDim.x) {
      float a = __fadd_rn(vec[H + c], d.Bh[H + c]);
      for (int k = 0; k < H; k++) a = __fmaf_rn(hp[k], d.Wrz[(size_t)k * 2 * H + c], a);
      const float g = nm_sig(a);
      if (c < H) { d.R[p * H + c] = g; hr[c] = hp[c] * g; d.HR[p * H + c] = hp[c] * g; d.HP[p * H + c] = hp[c]; }
      else d.Z[p * H + c - H] = g;
    }
    __syncthreads();
    float hn[NM_H_MAX / 256 + 1];
    for (int c = threadIdx.x, q = 0; c < H; c += blockDim.x, q++) {
      float a = __fadd_rn(vec[c], d.Bh[c]);
      for (int k = 0; k < H; k++) a = __fmaf_rn(hr[k], d.Wh[(size_t)k * H + c], a);
      const float ht = tanhf(a), z = d.Z[p * H + c];
      hn[q] = __fadd_rn(__fmul_rn(__fsub_rn(1.f, z), hp[c]), __fmul_rn(z, ht));
      d.HT[p * H + c] = ht; d.HH[p * H + c] = hn[q];
    }
    __syncthreads();
    for (int c = threadIdx.x, q = 0; c < H; c += blockDim.x, q++) hp[c] = hn[q];
    __syncthreads();
  }
}

// CTA per slot: alpha[t][j] = sum_k v[k] sig(A1H[t][k] + A2H[j][k]) for j <= t, s_t = sum_j alpha[t][j] h_j, c = [h_t ; s_t] (dropped out)
__global__ void __launch_bounds__(256) k_nm_att_fwd(NmDev d) {
  const int H = d.H, b = blockIdx.x, n = d.plen[b], p0 = d.poff[b];
  for (int x = threadIdx.x; x < n * n; x += blockDim.x) {
    const int t = x / n, j = x % n;
    if (j > t) continue;
    const float* a1 = d.A1H + (size_t)(p0 + t) * H;
    const float* a2 = d.A2H + (size_t)(p0 + j) * H;
    float a = 0.f;
    for (int k = 0; k < H; k++) a = __fmaf_rn(d.v[k], nm_sig(__fadd_rn(a1[k], a2[k])), a);
    d.AL[(size_t)(p0 + t) * d.L + j] = a;
  }
  __syncthreads();
  for (int x = threadIdx.x; x < n * H; x += blockDim.x) {
    const int t = x / H, k = x % H;
    const size_t p = (size_t)(p0 + t);
    float s = 0.f;
    for (int j = 0; j <= t; j++) s = __fmaf_rn(d.AL[p * d.L + j], d.HH[(size_t)(p0 + j) * H + k], s);
    d.C[p * 2 * H + k] = d.HH[p * H + k] * nm_mask(d, NM_STREAM_CT, b * d.L + t, 2 * H, k, d.rc);
    d.C[p * 2 * H + H + k] = s * nm_mask(d, NM_STREAM_CT, b * d.L + t, 2 * H, H + k, d.rc);
  }
}

// the encoder of a batch: Q [P x d] (part: split scratch)
static void nm_encode(cudaStream_t st, const NmDev& d, float* part) {
  const int H = d.H, P = d.P, dd = d.d;
  k_nm_gather<<<d.nb, 256, 0, st>>>(d);
  nm_gemm<NM_ENCODER>(st, part, d.EMB, dd, 1, d.Wx, 3 * H, 1, d.VEC, 3 * H, P, 3 * H, dd);
  k_nm_gru_fwd<<<d.nb, 256, 2 * H * sizeof(float), st>>>(d);
  nm_gemm<NM_ENCODER>(st, part, d.HH, H, 1, d.A1, 1, H, d.A1H, H, P, H, H);
  nm_gemm<NM_ENCODER>(st, part, d.HH, H, 1, d.A2, 1, H, d.A2H, H, P, H, H);
  k_nm_att_fwd<<<d.nb, 256, 0, st>>>(d);
  nm_gemm<NM_ENCODER>(st, part, d.C, 2 * H, 1, d.B, 1, 2 * H, d.Q, dd, P, dd, 2 * H);
}

// ---------------------------------------------------------------------------------------------------------------------------
// the loss and the backward pass
// ---------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float nm_block_reduce(float v, float* red, bool is_max) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) { const float u = __shfl_xor_sync(0xffffffffu, v, o); v = is_max ? fmaxf(v, u) : __fadd_rn(v, u); }
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = red[0];
  for (int q = 1; q < (int)(blockDim.x >> 5); q++) r = is_max ? fmaxf(r, red[q]) : __fadd_rn(r, red[q]);
  return r;
}

// CTA per position: m = max S, l = sum exp(S - m) (thread-strided then a fixed tree), loss = log l + m - S[y]; S becomes
// dL/dS = (exp(S - m) / l - [i == y]) / P in place
__global__ void __launch_bounds__(256) k_nm_softmax(NmDev d) {
  __shared__ float red[32];
  const int p = blockIdx.x, NI = d.NI, y = d.PY[p];
  float* s = d.S + (size_t)p * NI;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < NI; i += blockDim.x) m = fmaxf(m, s[i]);
  m = nm_block_reduce(m, red, true);
  float l = 0.f;
  for (int i = threadIdx.x; i < NI; i += blockDim.x) l = __fadd_rn(l, expf(__fsub_rn(s[i], m)));
  l = nm_block_reduce(l, red, false);
  const float sy = s[y];
  __syncthreads();
  for (int i = threadIdx.x; i < NI; i += blockDim.x) {
    const float pr = __fdiv_rn(expf(__fsub_rn(s[i], m)), l);
    s[i] = __fdiv_rn(i == y ? __fsub_rn(pr, 1.f) : pr, (float)d.P);
  }
  if (threadIdx.x == 0) d.LOSS[p] = __fsub_rn(__fadd_rn(logf(l), m), sy);
}

// the mean loss of the batch in a fixed order (one block), in float64
__global__ void __launch_bounds__(1024) k_nm_mean(const float* v, int n, float* out) {
  __shared__ double red[32];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  double s = 0.0;
  for (int i = tid; i < n; i += 1024) s += (double)v[i];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red[w] = s;
  __syncthreads();
  if (tid == 0) {
    double a = 0.0;
    for (int q = 0; q < 32; q++) a += red[q];
    *out = (float)(a / n);
  }
}

// CTA per slot, the attention backward.  dc = DC * mask; ds_t = dc[H:], dh_t gets dc[:H].  DA[t][j] = ds_t . h_j;
// g_tj = DA[t][j] v sig'(.), G1_t = sum_j g_tj, G2_j = sum_(t >= j) g_tj, DV_t = sum_j DA[t][j] sig(.);
// DHA_j = dc_j[:H] + sum_(t >= j) alpha[t][j] ds_t
__global__ void __launch_bounds__(256) k_nm_att_bwd(NmDev d) {
  const int H = d.H, b = blockIdx.x, n = d.plen[b], p0 = d.poff[b];
  auto dc = [&](int t, int k) { return d.DC[(size_t)(p0 + t) * 2 * H + k] * nm_mask(d, NM_STREAM_CT, b * d.L + t, 2 * H, k, d.rc); };
  for (int x = threadIdx.x; x < n * n; x += blockDim.x) {
    const int t = x / n, j = x % n;
    if (j > t) continue;
    float a = 0.f;
    for (int k = 0; k < H; k++) a = __fmaf_rn(dc(t, H + k), d.HH[(size_t)(p0 + j) * H + k], a);
    d.DA[(size_t)(p0 + t) * d.L + j] = a;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < H; k += blockDim.x) {
    const float vk = d.v[k];
    for (int t = 0; t < n; t++) {
      const size_t pt = (size_t)(p0 + t);
      const float a1 = d.A1H[pt * H + k];
      float g1 = 0.f, dv = 0.f;
      for (int j = 0; j <= t; j++) {
        const float u = nm_sig(__fadd_rn(a1, d.A2H[(size_t)(p0 + j) * H + k])), da = d.DA[pt * d.L + j];
        g1 = __fadd_rn(g1, __fmul_rn(__fmul_rn(da, vk), __fmul_rn(u, __fsub_rn(1.f, u))));
        dv = __fmaf_rn(da, u, dv);
      }
      d.G1[pt * H + k] = g1; d.DV[pt * H + k] = dv;
    }
    for (int j = 0; j < n; j++) {
      const size_t pj = (size_t)(p0 + j);
      const float a2 = d.A2H[pj * H + k];
      float g2 = 0.f, dh = dc(j, k);
      for (int t = j; t < n; t++) {
        const size_t pt = (size_t)(p0 + t);
        const float u = nm_sig(__fadd_rn(d.A1H[pt * H + k], a2)), da = d.DA[pt * d.L + j];
        g2 = __fadd_rn(g2, __fmul_rn(__fmul_rn(da, vk), __fmul_rn(u, __fsub_rn(1.f, u))));
        dh = __fmaf_rn(d.AL[pt * d.L + j], dc(t, H + k), dh);
      }
      d.G2[pj * H + k] = g2; d.DHA[pj * H + k] = dh;
    }
  }
}

// CTA per slot, the GRU backward in reverse: dh = DHA + T1 + T2 + the recurrent part; DVEC = [d a_h, d pre(r), d pre(z)]
__global__ void __launch_bounds__(256) k_nm_gru_bwd(NmDev d) {
  extern __shared__ float sm[];
  const int H = d.H, b = blockIdx.x, n = d.plen[b], p0 = d.poff[b];
  float* dhn = sm;                                       // [H] dL/dh_(t-1) handed to the step before
  float* dah = sm + H;                                   // [H]
  float* drz = sm + 2 * H;                               // [2H]
  for (int k = threadIdx.x; k < H; k += blockDim.x) dhn[k] = 0.f;
  __syncthreads();
  for (int t = n - 1; t >= 0; t--) {
    const size_t p = (size_t)(p0 + t);
    float dz[NM_H_MAX / 256 + 1], dhp[NM_H_MAX / 256 + 1];
    for (int k = threadIdx.x, q = 0; k < H; k += blockDim.x, q++) {
      const float dh = __fadd_rn(__fadd_rn(__fadd_rn(d.DHA[p * H + k], d.T1[p * H + k]), d.T2[p * H + k]), dhn[k]);
      const float z = d.Z[p * H + k], ht = d.HT[p * H + k], hp = d.HP[p * H + k];
      dz[q] = __fmul_rn(dh, __fsub_rn(ht, hp));
      dhp[q] = __fmul_rn(dh, __fsub_rn(1.f, z));
      dah[k] = __fmul_rn(__fmul_rn(dh, z), __fsub_rn(1.f, __fmul_rn(ht, ht)));
    }
    __syncthreads();
    for (int k = threadIdx.x, q = 0; k < H; k += blockDim.x, q++) {
      float dhr = 0.f;
      for (int c = 0; c < H; c++) dhr = __fmaf_rn(dah[c], d.Wh[(size_t)k * H + c], dhr);
      const float r = d.R[p * H + k], z = d.Z[p * H + k], hp = d.HP[p * H + k];
      drz[k] = __fmul_rn(__fmul_rn(dhr, hp), __fmul_rn(r, __fsub_rn(1.f, r)));
      drz[H + k] = __fmul_rn(dz[q], __fmul_rn(z, __fsub_rn(1.f, z)));
      dhp[q] = __fadd_rn(dhp[q], __fmul_rn(dhr, r));
      d.DVEC[p * 3 * H + k] = dah[k];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < 2 * H; c += blockDim.x) d.DVEC[p * 3 * H + H + c] = drz[c];
    for (int k = threadIdx.x, q = 0; k < H; k += blockDim.x, q++) {
      float a = dhp[q];
      for (int c = 0; c < 2 * H; c++) a = __fmaf_rn(drz[c], d.Wrz[(size_t)k * 2 * H + c], a);
      dhp[q] = a;
    }
    __syncthreads();
    for (int k = threadIdx.x, q = 0; k < H; k += blockDim.x, q++) dhn[k] = dhp[q];
    __syncthreads();
  }
}

// the input-embedding gradient: positions sorted by (input item, position); the thread of a run's head and unit u adds the
// run's DEMB * mask in position order to gE[item][u]
__global__ void k_nm_keys(const int* PX, int P, unsigned long long* keys) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < P) keys[p] = ((unsigned long long)(unsigned)PX[p] << 32) | (unsigned)p;
}
__global__ void k_nm_scatter(NmDev d, const unsigned long long* srt, float* gE) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (long long)d.P * d.d) return;
  const int q = (int)(x / d.d), u = (int)(x % d.d);
  const unsigned it = (unsigned)(srt[q] >> 32);
  if (q > 0 && (unsigned)(srt[q - 1] >> 32) == it) return;
  float a = 0.f;
  for (int r = q; r < d.P && (unsigned)(srt[r] >> 32) == it; r++) {
    const int p = (int)(srt[r] & 0xffffffffu);
    a = __fadd_rn(a, d.DEMB[(size_t)p * d.d + u] * nm_mask(d, NM_STREAM_EMB, d.PS[p], d.d, u, d.re));
  }
  gE[(size_t)it * d.d + u] = __fadd_rn(gE[(size_t)it * d.d + u], a);
}

// dense Adam (Kingma & Ba) over the flat parameters; c1 = 1 / (1 - b1^t), c2 = 1 / (1 - b2^t)
__global__ void k_nm_adam(float* th, const float* g, float* m, float* v, size_t n, float lr, float c1, float c2) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  const float mi = __fadd_rn(__fmul_rn(0.9f, m[i]), __fmul_rn(0.1f, gi));
  const float vi = __fadd_rn(__fmul_rn(0.999f, v[i]), __fmul_rn(0.001f, __fmul_rn(gi, gi)));
  m[i] = mi; v[i] = vi;
  th[i] = __fsub_rn(th[i], __fdiv_rn(__fmul_rn(lr, __fmul_rn(mi, c1)), __fadd_rn(__fsqrt_rn(__fmul_rn(vi, c2)), 1e-8f)));
}

__global__ void k_nm_to_double(const float* E, size_t n, double* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (double)E[i];
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
// per-position scratch in floats, the logits S excluded (nm_carve's arrays)
static size_t nm_pair_floats(int d, int H, int L) { return (size_t)4 * d + 24 * (size_t)H + 2 * (size_t)L + 1; }

// evaluation: Q rows of the chunk's positions to their counted events
__global__ void k_nm_pick(const float* Q, const int* ev, const int* pair, int ne, int dd, float* qev) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (long long)ne * dd) return;
  const int e = (int)(x / dd), u = (int)(x % dd);
  qev[(size_t)ev[e] * dd + u] = Q[(size_t)pair[e] * dd + u];
}

// the scratch of P positions and nb slots, carved from the handle's allocations; S only when the loss is needed
template <class Take>
static cudaError_t nm_scratch(Take take, NmScratch& s, long long P, long long nb, int d, int H, int L, int NI, bool loss) {
  cudaError_t e;
  if ((e = take(&s.PX, P)) || (e = take(&s.PY, P)) || (e = take(&s.PS, P))) return e;
  if ((e = take(&s.f, (size_t)P * nm_pair_floats(d, H, L)))) return e;
  if ((e = take(&s.part, NM_PART_CAP))) return e;
  if ((e = take(&s.pstart, nb)) || (e = take(&s.plen, nb)) || (e = take(&s.poff, nb))) return e;
  if (loss) {
    if ((e = take(&s.S, (size_t)P * NI)) || (e = take(&s.keys, P)) || (e = take(&s.keys2, P))) return e;
    size_t cb = 0;
    if ((e = cub::DeviceRadixSort::SortKeys(nullptr, cb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)P, 0, 64))) return e;
    if ((e = take(&s.cub, cb))) return e;
    s.cub_bytes = cb;
  }
  return cudaSuccess;
}

static void nm_bind(NmDev& d, const NmScratch& s, const float* th, const NmLayout& L, int NI, int dd, int H, int len) {
  d.E = th + L.E; d.Wx = th + L.Wx; d.Wrz = th + L.Wrz; d.Wh = th + L.Wh; d.Bh = th + L.Bh; d.A1 = th + L.A1; d.A2 = th + L.A2;
  d.v = th + L.v; d.B = th + L.B;
  d.NI = NI; d.d = dd; d.H = H; d.L = len;
  d.PX = s.PX; d.PY = s.PY; d.PS = s.PS; d.S = s.S;
  d.pstart = s.pstart; d.plen = s.plen; d.poff = s.poff;
}

// a batch's loss and gradient G (flat, the parameters' layout) at the handle's parameters; loss_out a device float
static void nm_grad(cudaStream_t st, NmDev d, const NmScratch& s, const NmLayout& L, float* G, const float* ones, float* loss_out) {
  const int H = d.H, P = d.P, dd = d.d, NI = d.NI;
  float* part = s.part;
  nm_encode(st, d, part);
  // the catalogue products: logits, the softmax gradient, dL/dq and dE
  nm_gemm<NM_CATALOGUE>(st, part, d.Q, dd, 1, d.E, 1, dd, d.S, NI, P, NI, dd);
  k_nm_softmax<<<P, 256, 0, st>>>(d);
  k_nm_mean<<<1, 1024, 0, st>>>(d.LOSS, P, loss_out);
  nm_gemm<NM_CATALOGUE>(st, part, d.S, NI, 1, d.E, dd, 1, d.DQ, dd, P, dd, NI);
  nm_gemm<NM_CATALOGUE>(st, part, d.S, 1, NI, d.Q, dd, 1, G + L.E, dd, NI, dd, P);
  // the decoder
  nm_gemm<NM_BACKWARD>(st, part, d.DQ, 1, dd, d.C, 2 * H, 1, G + L.B, 2 * H, dd, 2 * H, P);
  nm_gemm<NM_BACKWARD>(st, part, d.DQ, dd, 1, d.B, 2 * H, 1, d.DC, 2 * H, P, 2 * H, dd);
  // the attention
  k_nm_att_bwd<<<d.nb, 256, 0, st>>>(d);
  nm_gemm<NM_BACKWARD>(st, part, d.G1, H, 1, d.A1, H, 1, d.T1, H, P, H, H);
  nm_gemm<NM_BACKWARD>(st, part, d.G2, H, 1, d.A2, H, 1, d.T2, H, P, H, H);
  nm_gemm<NM_BACKWARD>(st, part, d.G1, 1, H, d.HH, H, 1, G + L.A1, H, H, H, P);
  nm_gemm<NM_BACKWARD>(st, part, d.G2, 1, H, d.HH, H, 1, G + L.A2, H, H, H, P);
  nm_gemm<NM_BACKWARD>(st, part, ones, 0, 0, d.DV, H, 1, G + L.v, H, 1, H, P);
  // the GRU
  k_nm_gru_bwd<<<d.nb, 256, 4 * H * sizeof(float), st>>>(d);
  nm_gemm<NM_BACKWARD>(st, part, d.HR, 1, H, d.DVEC, 3 * H, 1, G + L.Wh, H, H, H, P);
  nm_gemm<NM_BACKWARD>(st, part, d.HP, 1, H, d.DVEC + H, 3 * H, 1, G + L.Wrz, 2 * H, H, 2 * H, P);
  nm_gemm<NM_BACKWARD>(st, part, d.EMB, 1, dd, d.DVEC, 3 * H, 1, G + L.Wx, 3 * H, dd, 3 * H, P);
  nm_gemm<NM_BACKWARD>(st, part, ones, 0, 0, d.DVEC, 3 * H, 1, G + L.Bh, 3 * H, 1, 3 * H, P);
  nm_gemm<NM_BACKWARD>(st, part, d.DVEC, 3 * H, 1, d.Wx, 1, 3 * H, d.DEMB, dd, P, dd, 3 * H);
  // the input embeddings
  k_nm_keys<<<(P + 255) / 256, 256, 0, st>>>(d.PX, P, s.keys);
  int end_bit = 33;
  while (end_bit < 64 && ((unsigned long long)NI >> (end_bit - 32)) != 0ull) end_bit++;
  size_t cb = s.cub_bytes;
  cub::DeviceRadixSort::SortKeys(s.cub, cb, s.keys, s.keys2, P, 0, end_bit, st);
  k_nm_scatter<<<(unsigned)(((long long)P * dd + 255) / 256), 256, 0, st>>>(d, s.keys2, G + L.E);
}

// the per-position arrays of d from s.f, rows of P positions
static void nm_carve(NmDev& d, float* f, long long Pmax, int dd, int H, int L) {
  auto take = [&](float** q, size_t w) { *q = f; f += (size_t)Pmax * w; };
  take(&d.EMB, dd); take(&d.VEC, 3 * H); take(&d.HH, H); take(&d.R, H); take(&d.Z, H); take(&d.HT, H); take(&d.HP, H); take(&d.HR, H);
  take(&d.A1H, H); take(&d.A2H, H); take(&d.AL, L); take(&d.DA, L); take(&d.C, 2 * H); take(&d.Q, dd); take(&d.LOSS, 1); take(&d.DQ, dd);
  take(&d.DC, 2 * H); take(&d.G1, H); take(&d.G2, H); take(&d.DV, H); take(&d.DHA, H); take(&d.T1, H); take(&d.T2, H); take(&d.DVEC, 3 * H);
  take(&d.DEMB, dd);
}

static void nm_free_fit(g4r_baselines* h) {
  for (void* p : h->nm_mem) cudaFree(p);
  h->nm_mem.clear();
  h->nm_fit = false;
}

template <class T>
static cudaError_t nm_take(g4r_baselines* h, T** p, size_t n) {
  cudaError_t e = bl_alloc(p, n);
  if (e == cudaSuccess) h->nm_mem.push_back(*p); else *p = nullptr;
  return e;
}

static bool nm_finite(const float* v, size_t n) {
  for (size_t i = 0; i < n; i++) if (!std::isfinite(v[i])) return false;
  return true;
}

// the model buffers of a NARM handle: parameters, double(E) and zero biases for bpr_blocks, a device 1.0f
static int nm_set_model(g4r_baselines* h, int32_t hidden, int32_t max_len, const float* params, int64_t n_params, const char* who) {
  if (!params) FAIL(G4R_ERR_INVALID, std::string(who) + ": null parameters");
  if (hidden < 1 || hidden > NM_H_MAX || max_len < 2 || max_len > NM_LEN_MAX)
    FAIL(G4R_ERR_INVALID, std::string(who) + ": need hidden in 1 .. 1024 and max_len in 2 .. 512");
  const NmLayout L = nm_layout(h->n_items, h->n_keep, hidden);
  if (n_params != (int64_t)L.n) FAIL(G4R_ERR_INVALID, std::string(who) + ": need n_params = n_items d + 5 d H + 5 H^2 + 4 H = " + std::to_string(L.n));
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
  h->nm_H = hidden; h->nm_len = max_len; h->nm_n = L.n;
  const size_t nE = (size_t)h->n_items * h->n_keep;
  k_nm_to_double<<<(unsigned)((nE + 255) / 256), 256, 0, st>>>(h->dNmTh, nE, h->dI);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_narm_import(g4r_baselines* h, int32_t hidden, int32_t max_len, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NARM) FAIL(G4R_ERR_STATE, "g4r_bl_narm_import: the handle is not a NARM");
  return nm_set_model(h, hidden, max_len, params, n_params, "g4r_bl_narm_import");
}

extern "C" int g4r_bl_narm_export(g4r_baselines* h, float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NARM || !h->dNmTh) FAIL(G4R_ERR_STATE, "g4r_bl_narm_export: no NARM parameters (g4r_bl_narm_begin or g4r_bl_narm_import)");
  if (!params || n_params != (int64_t)h->nm_n) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_export: need n_params floats");
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(params, h->dNmTh, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

extern "C" int g4r_bl_narm_begin(g4r_baselines* h, int32_t hidden, int32_t max_len, int32_t batch_size, const int64_t* piece_offsets,
                                 int64_t n_pieces, const int32_t* items, int64_t n_entries, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NARM) FAIL(G4R_ERR_STATE, "g4r_bl_narm_begin: the handle is not a NARM");
  if (!piece_offsets || !items || n_pieces < 1 || n_entries < 2 || batch_size < 1)
    FAIL(G4R_ERR_INVALID, "g4r_bl_narm_begin: null argument, no pieces or batch_size < 1");
  if (hidden < 1 || hidden > NM_H_MAX || max_len < 2 || max_len > NM_LEN_MAX)
    FAIL(G4R_ERR_INVALID, "g4r_bl_narm_begin: need hidden in 1 .. 1024 and max_len in 2 .. 512");
  if (n_entries > INT32_MAX || n_pieces > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_begin: more than 2^31 - 1 entries or pieces");
  if (piece_offsets[0] != 0 || piece_offsets[n_pieces] != n_entries) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_begin: piece offsets must run from 0 to n_entries");
  std::vector<int> lens(n_pieces);
  for (int64_t k = 0; k < n_pieces; k++) {
    const int64_t n = piece_offsets[k + 1] - piece_offsets[k];
    if (n < 2 || n > max_len) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_begin: every piece needs 2 .. max_len events");
    lens[k] = (int)n - 1;
  }
  const int NI = h->n_items, dd = h->n_keep;
  for (int64_t e = 0; e < n_entries; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_narm_begin: item index out of range");
  if ((uint64_t)batch_size * max_len * std::max(dd, 2 * hidden) >= 0xffffffffull)
    FAIL(G4R_ERR_INVALID, "g4r_bl_narm_begin: batch_size * max_len * max(d_e, 2 hidden) must stay below 2^32 (dropout indices)");
  // the largest batch: the batch_size longest pieces
  std::vector<int> srt(lens);
  std::sort(srt.begin(), srt.end(), std::greater<int>());
  long long Pmax = 0;
  for (int64_t k = 0; k < std::min<int64_t>(batch_size, n_pieces); k++) Pmax += srt[k];
  const NmLayout L = nm_layout(NI, dd, hidden);
  const size_t need = (size_t)Pmax * ((size_t)NI * 4 + nm_pair_floats(dd, hidden, max_len) * 4 + 28) + NM_PART_CAP * 4 + 3 * L.n * 4 +
                      (size_t)n_entries * 4 + (size_t)n_pieces * 16 + ((size_t)64 << 20);
  int rc = nm_set_model(h, hidden, max_len, params, n_params, "g4r_bl_narm_begin");
  if (rc) return rc;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    h->err = "g4r_bl_narm_begin: the fit needs " + std::to_string(need) + " bytes of device memory (the logits of the largest batch alone " +
             std::to_string((size_t)Pmax * NI * 4) + "), " + std::to_string(free_b) + " are free";
    return G4R_ERR_CUDA;
  }
  cudaStream_t st = h->stream;
  h->ready = false;
  auto take = [&](auto** p, size_t n) { return nm_take(h, p, n); };
  NmScratch& s = h->nm_s;
  s = NmScratch{};
  CK(nm_scratch(take, s, Pmax, batch_size, dd, hidden, max_len, NI, true));
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

// the batches of a list of pieces: per entry its start, inputs and position offset within its batch; per batch (first entry, P).
// The scratch holds the positions of the batch_size longest distinct pieces (nm_Pmax); a batch that repeats a long piece can
// exceed it, and is refused here, before any device write.
static int nm_plan(g4r_baselines* h, const int32_t* pieces, int64_t n, std::vector<long long>& ps, std::vector<int>& pl,
                   std::vector<int>& po, std::vector<std::pair<int64_t, int>>& batches, const char* who) {
  ps.resize(n); pl.resize(n); po.resize(n);
  for (int64_t b0 = 0; b0 < n; b0 += h->nm_bs) {
    long long P = 0;
    for (int64_t q = b0; q < std::min<int64_t>(n, b0 + h->nm_bs); q++) {
      const int k = pieces[q];
      ps[q] = h->nm_off[k]; pl[q] = (int)(h->nm_off[k + 1] - h->nm_off[k]) - 1; po[q] = (int)P; P += pl[q];
    }
    if (P > h->nm_Pmax)
      FAIL(G4R_ERR_INVALID, std::string(who) + ": a batch holds " + std::to_string(P) + " positions, more than the " + std::to_string(h->nm_Pmax) +
                                " of the batch_size longest distinct pieces the fit was begun with (a piece repeated in a batch?)");
    batches.push_back({b0, (int)P});
  }
  return G4R_OK;
}

static NmDev nm_train_dev(g4r_baselines* h, unsigned seed, unsigned gstep, float p_emb, float p_ct) {
  NmDev d{};
  const NmLayout L = nm_layout(h->n_items, h->n_keep, h->nm_H);
  nm_bind(d, h->nm_s, h->dNmTh, L, h->n_items, h->n_keep, h->nm_H, h->nm_len);
  nm_carve(d, h->nm_s.f, h->nm_Pmax, h->n_keep, h->nm_H, h->nm_len);
  d.items = h->dNmItems; d.train = 1; d.seed = seed; d.gstep = gstep;
  d.re = p_emb > 0.f ? 1.f - p_emb : 1.f; d.rc = p_ct > 0.f ? 1.f - p_ct : 1.f;
  return d;
}

static int nm_check_run(g4r_baselines* h, const int32_t* pieces, int64_t n, float p_emb, float p_ct, const char* who) {
  if (h->kind != BL_NARM) FAIL(G4R_ERR_STATE, std::string(who) + ": the handle is not a NARM");
  if (!h->nm_fit) FAIL(G4R_ERR_STATE, std::string(who) + ": no fit begun (g4r_bl_narm_begin)");
  if (!pieces || n < 1) FAIL(G4R_ERR_INVALID, std::string(who) + ": no pieces");
  if (!(p_emb >= 0.f && p_emb < 1.f && p_ct >= 0.f && p_ct < 1.f)) FAIL(G4R_ERR_INVALID, std::string(who) + ": dropout must be in [0, 1)");
  const int64_t np = (int64_t)h->nm_off.size() - 1;
  for (int64_t q = 0; q < n; q++) if (pieces[q] < 0 || pieces[q] >= np) FAIL(G4R_ERR_INDEX, std::string(who) + ": piece index out of range");
  return G4R_OK;
}

static int nm_upload_plan(g4r_baselines* h, const std::vector<long long>& ps, const std::vector<int>& pl, const std::vector<int>& po, int64_t q0, int nb) {
  NmScratch& s = h->nm_s;
  CK(cudaMemcpyAsync(s.pstart, ps.data() + q0, nb * sizeof(long long), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(s.plen, pl.data() + q0, nb * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(s.poff, po.data() + q0, nb * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  return G4R_OK;
}

extern "C" int g4r_bl_narm_grads(g4r_baselines* h, const int32_t* pieces, int32_t n, uint32_t seed, int64_t step, float dropout_emb,
                                 float dropout_ct, float* loss, float* grads) {
  if (!h) return G4R_ERR_INVALID;
  int rc = nm_check_run(h, pieces, n, dropout_emb, dropout_ct, "g4r_bl_narm_grads");
  if (rc) return rc;
  if (n > h->nm_bs || !grads || step < 0 || step > 0xffffffffll) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_grads: need n <= batch_size, grads and step in 0 .. 2^32 - 1");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = nm_plan(h, pieces, n, ps, pl, po, batches, "g4r_bl_narm_grads");
  if (rc) return rc;
  cudaSetDevice(h->device);
  rc = nm_upload_plan(h, ps, pl, po, 0, n);
  if (rc) return rc;
  NmDev d = nm_train_dev(h, seed, (unsigned)step, dropout_emb, dropout_ct);
  d.nb = n; d.P = batches[0].second;
  nm_grad(h->stream, d, h->nm_s, nm_layout(h->n_items, h->n_keep, h->nm_H), h->dNmG, h->dNmOne, h->dNmLoss);
  CK(cudaGetLastError());
  float l = 0.f;
  CK(cudaMemcpyAsync(&l, h->dNmLoss, sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(grads, h->dNmG, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (loss) *loss = l;
  return G4R_OK;
}

extern "C" int g4r_bl_narm_epoch(g4r_baselines* h, const int32_t* order, int64_t n_order, uint32_t seed, float learning_rate, float dropout_emb,
                                 float dropout_ct, float* losses, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  int rc = nm_check_run(h, order, n_order, dropout_emb, dropout_ct, "g4r_bl_narm_epoch");
  if (rc) return rc;
  if (!(learning_rate > 0.f && std::isfinite(learning_rate))) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_epoch: learning_rate must be finite and > 0");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = nm_plan(h, order, n_order, ps, pl, po, batches, "g4r_bl_narm_epoch");
  if (rc) return rc;
  if (h->nm_step + (int64_t)batches.size() > 0xffffffffll) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_epoch: more than 2^32 steps since the fit began");
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  NmScratch& s = h->nm_s;
  const NmLayout L = nm_layout(h->n_items, h->n_keep, h->nm_H);
  // the whole epoch's plan goes up once; each batch reads its slice
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr; float* dloss = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  CK(bb.take(&dloss, batches.size()));
  CK(cudaEventRecord(h->ev0, st));
  for (size_t b = 0; b < batches.size(); b++) {
    const int64_t q0 = batches[b].first;
    const int nb = (int)std::min<int64_t>(h->nm_bs, n_order - q0);
    NmDev d = nm_train_dev(h, seed, (unsigned)h->nm_step, dropout_emb, dropout_ct);
    d.pstart = dps + q0; d.plen = dpl + q0; d.poff = dpo + q0; d.nb = nb; d.P = batches[b].second;
    nm_grad(st, d, s, L, h->dNmG, h->dNmOne, dloss + b);
    h->nm_step++;
    const double t = (double)h->nm_step;
    const float c1 = (float)(1.0 / (1.0 - std::pow(0.9, t))), c2 = (float)(1.0 / (1.0 - std::pow(0.999, t)));
    k_nm_adam<<<(unsigned)((L.n + 255) / 256), 256, 0, st>>>(h->dNmTh, h->dNmG, h->dNmM, h->dNmV, L.n, learning_rate, c1, c2);
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

// the encoder pieces of an evaluation's counted events, in chunks of at most cap positions and cap pieces: per session one piece
// from its start covers the prefixes of <= len inputs, and each longer prefix takes a window of its last len inputs.  The encoder
// hook flush(ps, pl, po, ev, pair, P) encodes one chunk: per piece its start, inputs and position offset, per counted event of
// the chunk its index and position, and the chunk's positions.  NARM and SASRec share it.
template <class Flush>
static int nm_event_chunks(int len, int cap, const int64_t* off, int64_t n_sessions, const int32_t* n_history, const std::vector<int64_t>& ev0,
                           Flush flush) {
  std::vector<long long> ps; std::vector<int> pl, po, ev, pair;
  int P = 0;
  auto emit = [&]() -> int {
    if (ps.empty()) return G4R_OK;
    const int rc = flush(ps, pl, po, ev, pair, P);
    ps.clear(); pl.clear(); po.clear(); ev.clear(); pair.clear(); P = 0;
    return rc;
  };
  auto piece = [&](long long start, int n) -> int {
    if (P + n > cap || (int)ps.size() >= cap) { const int rc = emit(); if (rc) return rc; }
    ps.push_back(start); pl.push_back(n); po.push_back(P); P += n;
    return G4R_OK;
  };
  for (int64_t sI = 0; sI < n_sessions; sI++) {
    const int64_t st0 = off[sI], en = off[sI + 1];
    const int64_t i0 = std::max<int64_t>(n_history ? n_history[sI] : 0, 1) - 1;   // input index of the first counted event
    const int64_t last = en - st0 - 2;                                            // input index of the last counted event
    if (last < i0) continue;
    if (i0 < len) {                                      // one piece from the session start covers the prefixes of <= len inputs
      const int n = (int)std::min<int64_t>(last + 1, len);
      int rc = piece(st0, n);
      if (rc) return rc;
      for (int64_t i = i0; i < n; i++) { ev.push_back((int)(ev0[sI] + i - i0)); pair.push_back(po.back() + (int)i); }
    }
    for (int64_t i = std::max<int64_t>(i0, len); i <= last; i++) {   // longer prefixes: a window of the last len inputs each
      int rc = piece(st0 + i - len + 1, len);
      if (rc) return rc;
      ev.push_back((int)(ev0[sI] + i - i0)); pair.push_back(po.back() + len - 1);
    }
  }
  return emit();
}

// every counted event's q (eval mode: no dropout; the last max_len inputs of its prefix) into qev [n_ev x d] on the device
static int nm_encode_events(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* off, int64_t n_sessions, const int32_t* n_history,
                            const std::vector<int64_t>& ev0, float* qev) {
  const int dd = h->n_keep, H = h->nm_H, len = h->nm_len;
  cudaStream_t st = h->stream;
  BlBufs bb;
  NmScratch s;
  auto take = [&](auto** p, size_t n) { return bb.take(p, n); };
  CK(nm_scratch(take, s, NM_EVAL_PAIRS, NM_EVAL_PAIRS, dd, H, len, h->n_items, false));
  const int* dItems = nullptr;
  CK(bb.put(&dItems, items, n_events, st));
  int *dEv = nullptr, *dPair = nullptr;
  CK(bb.take(&dEv, NM_EVAL_PAIRS)); CK(bb.take(&dPair, NM_EVAL_PAIRS));
  NmDev d{};
  nm_bind(d, s, h->dNmTh, nm_layout(h->n_items, dd, H), h->n_items, dd, H, len);
  nm_carve(d, s.f, NM_EVAL_PAIRS, dd, H, len);
  d.items = dItems; d.train = 0; d.re = 1.f; d.rc = 1.f;
  auto flush = [&](const std::vector<long long>& ps, const std::vector<int>& pl, const std::vector<int>& po, const std::vector<int>& ev,
                   const std::vector<int>& pair, int P) -> int {
    const int nb = (int)ps.size();
    CK(cudaMemcpyAsync(s.pstart, ps.data(), nb * sizeof(long long), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(s.plen, pl.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(s.poff, po.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dEv, ev.data(), ev.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(dPair, pair.data(), pair.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    d.nb = nb; d.P = P;
    nm_encode(st, d, s.part);
    const int ne = (int)ev.size();
    k_nm_pick<<<(unsigned)(((long long)ne * dd + 255) / 256), 256, 0, st>>>(d.Q, dEv, dPair, ne, dd, qev);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));                      // the host arrays are reused by the next chunk
    return G4R_OK;
  };
  return nm_event_chunks(len, NM_EVAL_PAIRS, off, n_sessions, n_history, ev0, flush);
}

extern "C" int g4r_bl_narm_encode(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                                  const int32_t* n_history, float* q, int64_t n_q) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_NARM || !h->ready) FAIL(G4R_ERR_STATE, "g4r_bl_narm_encode: no NARM parameters (g4r_bl_narm_begin or g4r_bl_narm_import)");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || n_q < 0 || (n_q > 0 && !q))
    FAIL(G4R_ERR_INVALID, "g4r_bl_narm_encode: null or out-of-range argument");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_encode: session offsets must rise from 0 to n_events");
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= h->n_items) FAIL(G4R_ERR_INDEX, "g4r_bl_narm_encode: item index out of range");
  std::vector<int64_t> ev0;
  int rc = bl_counted(h, "g4r_bl_narm_encode", session_offsets, n_sessions, n_history, ev0);
  if (rc) return rc;
  if (n_q != ev0[n_sessions]) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_encode: n_q must be the number of counted events");
  if (n_q > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_narm_encode: more than 2^31 - 1 counted events");
  cudaSetDevice(h->device);
  BlBufs bb;
  float* dq = nullptr;
  CK(bb.take(&dq, (size_t)n_q * h->n_keep));
  rc = nm_encode_events(h, items, n_events, session_offsets, n_sessions, n_history, ev0, dq);
  if (rc) return rc;
  if (n_q) CK(cudaMemcpyAsync(q, dq, (size_t)n_q * h->n_keep * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// the ranking of a g4r_bl_evaluate call of a NARM: every counted event's q, then BPR's ranking with I = double(E), bI = 0
static int narm_rank(g4r_baselines* h, BlCall& c) {
  float* dq = nullptr;
  CK(c.bb.take(&dq, (size_t)c.n_ev * h->n_keep));
  const int rc = nm_encode_events(h, c.items, c.n_events, c.off, c.n_sessions, c.n_history, c.ev0, dq);
  if (rc) return rc;
  return bpr_blocks(h, c, dq);
}
