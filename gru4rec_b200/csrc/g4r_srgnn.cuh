// g4r_srgnn.cuh -- the SR-GNN session-graph baseline on the device (DESIGN §3u): per (prefix, next item) sample the directed
// graph of the prefix's distinct items, `step` gated propagation steps over its normalised in- and out-adjacency, the hybrid
// attention readout s_h = W3 [s_g ; s_l] + b3 and full-catalogue cross-entropy, trained with NARM's dense Adam on the gradient
// plus coupled L2; and the eval-mode encoder that feeds per-event vectors to BPR's ranking.  Every dense product runs through
// NARM's k_nm_gemm, the catalogue loss through k_nm_softmax, the node-embedding gradient through k_nm_keys / k_nm_scatter.  The
// graphs are sparse lists (at most n - 1 edges for n inputs), built on the device per sample.  Every reduction runs in a fixed
// order (no floating-point atomics), so a fit is bitwise reproducible.  A handle keeps its model in the handle's NARM fields.
// Included at the end of g4r_lib.cu after g4r_sasrec.cuh.
#pragma once

constexpr int SG_D_MAX = 1024, SG_STEP_MAX = 8, SG_LEN_MAX = 512;
constexpr int SG_THREADS = 256;                        // graph, readout and node CTAs (one per sample)
constexpr int SG_EVAL_POS = 16384;                     // positions (and samples) per evaluation chunk

// offsets of the parameters in the flat float32 vector (DESIGN §3u)
struct SgLayout {
  size_t E, Win, Wout, bin, bout, biah, boah, Wih, bih, Whh, bhh, W1, W2, b1, b2, q, W3, b3, n;
};
static SgLayout sg_layout(int NI, int d) {
  SgLayout L;
  const size_t D = d, DD = D * D;
  L.E = 0; L.Win = (size_t)NI * D; L.Wout = L.Win + DD; L.bin = L.Wout + DD; L.bout = L.bin + D; L.biah = L.bout + D; L.boah = L.biah + D;
  L.Wih = L.boah + D; L.bih = L.Wih + 6 * DD; L.Whh = L.bih + 3 * D; L.bhh = L.Whh + 3 * DD; L.W1 = L.bhh + 3 * D; L.W2 = L.W1 + DD;
  L.b1 = L.W2 + DD; L.b2 = L.b1 + D; L.q = L.b2 + D; L.W3 = L.q + D; L.b3 = L.W3 + 2 * DD; L.n = L.b3 + D;
  return L;
}

// one mini-batch (or evaluation chunk) of nb samples: sample b has the n = slen[b] inputs items[sstart[b] ..] (a training
// sample's target follows them), its positions and its node slots are soff[b] .. soff[b] + n - 1; its K <= n nodes take the
// first K slots, the rest are zero rows without edges.  Per slot (node lists hold global slots, in ascending order):
// in-neighbours INL[INS .. INS + INC), out-neighbours OUL[OUS .. OUS + OUC), positions NPL[NPS .. NPS + NPC)
struct SgDev {
  const int* items; const long long* sstart; const int* slen; const int* soff; int nb, P;
  const float* E;
  int d, train;
  int *ALIAS, *NX, *INS, *INC, *INL, *OUS, *OUC, *OUL, *NPS, *NPC, *NPL;   // per position / slot
  int *NK, *PY;                                                           // per sample: nodes, target (-1: none)
};

// CTA per sample: the nodes (distinct items ascending), alias, the deduplicated edge lists and each node's positions, by rank
// counting in shared memory; H0 = E[node] (0 past the nodes)
__global__ void __launch_bounds__(SG_THREADS) k_sg_graph(SgDev g, float* H0) {
  __shared__ int x[SG_LEN_MAX], al[SG_LEN_MAX], first[SG_LEN_MAX], eu[SG_LEN_MAX], ev[SG_LEN_MAX], ek[SG_LEN_MAX], nx[SG_LEN_MAX];
  const int b = blockIdx.x, n = g.slen[b], o = g.soff[b], tid = threadIdx.x, nt = blockDim.x;
  const long long s0 = g.sstart[b];
  for (int t = tid; t < n; t += nt) x[t] = g.items[s0 + t];
  __syncthreads();
  for (int t = tid; t < n; t += nt) {
    int f = 1;
    for (int j = 0; j < t && f; j++) f = x[j] != x[t];
    first[t] = f;
  }
  __syncthreads();
  for (int t = tid; t < n; t += nt) {
    int a = 0;
    for (int j = 0; j < n; j++) a += first[j] && x[j] < x[t];
    al[t] = a;
    if (first[t]) nx[a] = x[t];
  }
  __syncthreads();
  int K = 0;
  for (int j = 0; j < n; j++) K += first[j];
  const int ne = n - 1;                                  // edge e joins positions e and e + 1; a repeat counts once
  for (int e = tid; e < ne; e += nt) {
    const int u = al[e], v = al[e + 1];
    int uq = 1;
    for (int j = 0; j < e && uq; j++) uq = !(al[j] == u && al[j + 1] == v);
    eu[e] = u; ev[e] = v; ek[e] = uq;
  }
  __syncthreads();
  for (int k = tid; k < n; k += nt) {
    int ci = 0, si = 0, co = 0, so = 0, pc = 0, ps = 0;
    if (k < K) {
      for (int e = 0; e < ne; e++)
        if (ek[e]) { ci += ev[e] == k; si += ev[e] < k; co += eu[e] == k; so += eu[e] < k; }
      for (int t = 0; t < n; t++) { pc += al[t] == k; ps += al[t] < k; }
    }
    g.INS[o + k] = o + si; g.INC[o + k] = ci; g.OUS[o + k] = o + so; g.OUC[o + k] = co; g.NPS[o + k] = o + ps; g.NPC[o + k] = pc;
    g.NX[o + k] = k < K ? nx[k] : 0;
  }
  for (int e = tid; e < ne; e += nt) {
    if (!ek[e]) continue;
    const int u = eu[e], v = ev[e];
    int ii = 0, oi = 0;
    for (int f = 0; f < ne; f++)
      if (ek[f]) { ii += ev[f] < v || (ev[f] == v && eu[f] < u); oi += eu[f] < u || (eu[f] == u && ev[f] < v); }
    g.INL[o + ii] = o + u; g.OUL[o + oi] = o + v;
  }
  for (int t = tid; t < n; t += nt) {
    int i = 0;
    for (int j = 0; j < n; j++) i += al[j] < al[t] || (al[j] == al[t] && j < t);
    g.NPL[o + i] = o + t; g.ALIAS[o + t] = o + al[t];
  }
  for (int z = tid; z < n * g.d; z += nt) {
    const int k = z / g.d, c = z % g.d;
    H0[(size_t)(o + k) * g.d + c] = k < K ? g.E[(size_t)nx[k] * g.d + c] : 0.f;
  }
  if (tid == 0) { g.NK[b] = K; g.PY[b] = g.train ? g.items[s0 + n] : -1; }
}

// thread per (slot v, unit c): A[v] = [a_in ; a_out], a_in = (sum over in-neighbours u ascending of (XI[u] + b_in)) / indeg(v)
// + b_iah, a_out likewise over out-neighbours with XO, b_out, b_oah (a node without such edges: the bias alone)
__global__ void k_sg_agg(SgDev g, const float* XI, const float* XO, const float* bin, const float* bout, const float* biah, const float* boah, float* A) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)g.P * g.d) return;
  const int v = (int)(i / g.d), c = (int)(i % g.d), d = g.d;
  const int ni = g.INC[v], no = g.OUC[v];
  float a = 0.f, b = 0.f;
  for (int j = 0; j < ni; j++) a = __fadd_rn(a, __fadd_rn(XI[(size_t)g.INL[g.INS[v] + j] * d + c], bin[c]));
  for (int j = 0; j < no; j++) b = __fadd_rn(b, __fadd_rn(XO[(size_t)g.OUL[g.OUS[v] + j] * d + c], bout[c]));
  A[(size_t)v * 2 * d + c] = __fadd_rn(ni ? __fdiv_rn(a, (float)ni) : 0.f, biah[c]);
  A[(size_t)v * 2 * d + d + c] = __fadd_rn(no ? __fdiv_rn(b, (float)no) : 0.f, boah[c]);
}

// the transposed aggregation: DXI[u] = sum over out-neighbours v ascending of DA_in[v] / indeg(v), DXO[v] = sum over
// in-neighbours u ascending of DA_out[u] / outdeg(u)
__global__ void k_sg_agg_bwd(SgDev g, const float* DA, float* DXI, float* DXO) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)g.P * g.d) return;
  const int u = (int)(i / g.d), c = (int)(i % g.d), d = g.d;
  float a = 0.f, b = 0.f;
  for (int j = 0; j < g.OUC[u]; j++) {
    const int v = g.OUL[g.OUS[u] + j];
    a = __fadd_rn(a, __fdiv_rn(DA[(size_t)v * 2 * d + c], (float)g.INC[v]));
  }
  for (int j = 0; j < g.INC[u]; j++) {
    const int w = g.INL[g.INS[u] + j];
    b = __fadd_rn(b, __fdiv_rn(DA[(size_t)w * 2 * d + d + c], (float)g.OUC[w]));
  }
  DXI[i] = a; DXO[i] = b;
}

// thread per (slot, unit), the gated update: gi = GI + b_ih, gh = GH + b_hh in (r, z, n) thirds; r, z, n saved with
// ghn = gh_n for the backward; Hn = n + z (H - n)
__global__ void k_sg_gate(int P, int d, const float* GI, const float* GH, const float* bih, const float* bhh, const float* H, float* R, float* Z,
                          float* N, float* GHN, float* Hn) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)P * d) return;
  const size_t p = (size_t)(i / d), c = (size_t)(i % d), o = p * 3 * d;
  const float r = nm_sig(__fadd_rn(__fadd_rn(GI[o + c], bih[c]), __fadd_rn(GH[o + c], bhh[c])));
  const float z = nm_sig(__fadd_rn(__fadd_rn(GI[o + d + c], bih[d + c]), __fadd_rn(GH[o + d + c], bhh[d + c])));
  const float ghn = __fadd_rn(GH[o + 2 * d + c], bhh[2 * d + c]);
  const float nn = tanhf(__fadd_rn(__fadd_rn(GI[o + 2 * d + c], bih[2 * d + c]), __fmul_rn(r, ghn)));
  R[i] = r; Z[i] = z; N[i] = nn; GHN[i] = ghn;
  Hn[i] = __fadd_rn(nn, __fmul_rn(z, __fsub_rn(H[i], nn)));
}

// dL/dH of a state: D0 (+ T1 + T2 + T3), added in that order
__device__ __forceinline__ float sg_dh(long long i, const float* D0, const float* T1, const float* T2, const float* T3) {
  float a = D0[i];
  if (T1) a = __fadd_rn(__fadd_rn(__fadd_rn(a, T1[i]), T2[i]), T3[i]);
  return a;
}

// the gated update's backward, given dL/dHn (sg_dh): DGI = d[gi_r, gi_z, gi_n], DGH = d[gh_r, gh_z, gh_n], DHD = dHn z the
// direct part of dL/dH (in place of D0 is allowed: each thread reads its element first)
__global__ void k_sg_gate_bwd(int P, int d, const float* D0, const float* T1, const float* T2, const float* T3, const float* H, const float* R,
                              const float* Z, const float* N, const float* GHN, float* DGI, float* DGH, float* DHD) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)P * d) return;
  const size_t p = (size_t)(i / d), c = (size_t)(i % d), o = p * 3 * d;
  const float dh = sg_dh(i, D0, T1, T2, T3), r = R[i], z = Z[i], nn = N[i];
  const float dz = __fmul_rn(dh, __fsub_rn(H[i], nn)), dn = __fmul_rn(dh, __fsub_rn(1.f, z));
  const float dpn = __fmul_rn(dn, __fsub_rn(1.f, __fmul_rn(nn, nn)));
  const float dpr = __fmul_rn(__fmul_rn(dpn, GHN[i]), __fmul_rn(r, __fsub_rn(1.f, r)));
  const float dpz = __fmul_rn(dz, __fmul_rn(z, __fsub_rn(1.f, z)));
  DGI[o + c] = dpr; DGI[o + d + c] = dpz; DGI[o + 2 * d + c] = dpn;
  DGH[o + c] = dpr; DGH[o + d + c] = dpz; DGH[o + 2 * d + c] = __fmul_rn(dpn, r);
  DHD[i] = __fmul_rn(dh, z);
}

// OUT = D0 + T1 + T2 + T3 (sg_dh's order): dL/dH0, the node-embedding rows
__global__ void k_sg_dsum(long long n, const float* D0, const float* T1, const float* T2, const float* T3, float* OUT) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) OUT[i] = sg_dh(i, D0, T1, T2, T3);
}

// the readout's rows: HP[p] = H[alias(p)] per position, SL[b] = H[alias(last position of b)] per sample
__global__ void k_sg_rows(SgDev g, const float* H, float* HP, float* SL) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x, np = (long long)g.P * g.d;
  if (i >= np + (long long)g.nb * g.d) return;
  if (i < np) { HP[i] = H[(size_t)g.ALIAS[i / g.d] * g.d + i % g.d]; return; }
  const long long j = i - np;
  const int b = (int)(j / g.d), c = (int)(j % g.d);
  SL[j] = H[(size_t)g.ALIAS[g.soff[b] + g.slen[b] - 1] * g.d + c];
}

// sig(W1 s_l + b1 + W2 h_t + b2) of unit c, from Q1 = s_l W1 and Q2 = h_t W2
__device__ __forceinline__ float sg_att_u(float q1, float b1, float q2, float b2) { return nm_sig(__fadd_rn(__fadd_rn(q1, b1), __fadd_rn(q2, b2))); }

__device__ __forceinline__ float sg_warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// CTA per sample: ALPHA[p] = q . u_p (warp per position, lanes strided over units then a fixed tree), s_g = sum over positions in
// order of ALPHA h_t; CAT[b] = [s_g ; s_l]
__global__ void __launch_bounds__(SG_THREADS) k_sg_readout(SgDev g, const float* HP, const float* SL, const float* Q1, const float* Q2, const float* b1,
                                                           const float* b2, const float* qv, float* ALPHA, float* CAT) {
  const int b = blockIdx.x, n = g.slen[b], o = g.soff[b], d = g.d, lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int t = w; t < n; t += nw) {
    const size_t p = (size_t)(o + t);
    float a = 0.f;
    for (int c = lane; c < d; c += 32) a = __fmaf_rn(qv[c], sg_att_u(Q1[(size_t)b * d + c], b1[c], Q2[p * d + c], b2[c]), a);
    a = sg_warp_sum(a);
    if (lane == 0) ALPHA[p] = a;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < n; t++) s = __fmaf_rn(ALPHA[o + t], HP[(size_t)(o + t) * d + c], s);
    CAT[(size_t)b * 2 * d + c] = s; CAT[(size_t)b * 2 * d + d + c] = SL[(size_t)b * d + c];
  }
}

// CTA per sample, the readout's backward from DCAT = [ds_g ; ds_l]: dalpha_t = ds_g . h_t; DHP[p] = alpha_t ds_g (the s_g part of
// dh_t), DQ2[p] = dalpha_t q u (1 - u), DQV[p] = dalpha_t u (q's gradient rows); DQ1[b] = sum over positions in order of DQ2
__global__ void __launch_bounds__(SG_THREADS) k_sg_readout_bwd(SgDev g, const float* HP, const float* Q1, const float* Q2, const float* b1,
                                                               const float* b2, const float* qv, const float* ALPHA, const float* DCAT, float* DHP,
                                                               float* DQ2, float* DQV, float* DQ1) {
  __shared__ float da[SG_LEN_MAX];
  const int b = blockIdx.x, n = g.slen[b], o = g.soff[b], d = g.d, lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* dsg = DCAT + (size_t)b * 2 * d;
  for (int t = w; t < n; t += nw) {
    float a = 0.f;
    for (int c = lane; c < d; c += 32) a = __fmaf_rn(dsg[c], HP[(size_t)(o + t) * d + c], a);
    a = sg_warp_sum(a);
    if (lane == 0) da[t] = a;
  }
  __syncthreads();
  for (int z = threadIdx.x; z < n * d; z += blockDim.x) {
    const int t = z / d, c = z % d;
    const size_t p = (size_t)(o + t);
    const float u = sg_att_u(Q1[(size_t)b * d + c], b1[c], Q2[p * d + c], b2[c]);
    DQ2[p * d + c] = __fmul_rn(__fmul_rn(da[t], qv[c]), __fmul_rn(u, __fsub_rn(1.f, u)));
    DQV[p * d + c] = __fmul_rn(da[t], u);
    DHP[p * d + c] = __fmul_rn(ALPHA[p], dsg[c]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < n; t++) s = __fadd_rn(s, DQ2[(size_t)(o + t) * d + c]);
    DQ1[(size_t)b * d + c] = s;
  }
}

// CTA per sample: dL/dH of the last state per node slot: over the node's positions in order (DHP + TP), then at the last
// position's node (ds_l + TS); 0 past the nodes
__global__ void __launch_bounds__(SG_THREADS) k_sg_node_bwd(SgDev g, const float* DHP, const float* TP, const float* DCAT, const float* TS, float* DH) {
  const int b = blockIdx.x, n = g.slen[b], o = g.soff[b], d = g.d, K = g.NK[b], last = g.ALIAS[o + n - 1] - o;
  for (int z = threadIdx.x; z < n * d; z += blockDim.x) {
    const int k = z / d, c = z % d;
    float a = 0.f;
    if (k < K) {
      for (int j = 0; j < g.NPC[o + k]; j++) {
        const size_t p = (size_t)g.NPL[g.NPS[o + k] + j];
        a = __fadd_rn(a, __fadd_rn(DHP[p * d + c], TP[p * d + c]));
      }
      if (k == last) a = __fadd_rn(a, __fadd_rn(DCAT[(size_t)b * 2 * d + d + c], TS[(size_t)b * d + c]));
    }
    DH[(size_t)(o + k) * d + c] = a;
  }
}

// X [n / d x d] += b per column
__global__ void k_sg_bias(float* X, const float* b, long long n, int d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) X[i] = __fadd_rn(X[i], b[i % d]);
}

// coupled L2: G += l2 theta over every parameter
__global__ void k_sg_l2(float* G, const float* th, size_t n, float l2) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) G[i] = __fadd_rn(G[i], __fmul_rn(l2, th[i]));
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
// the float arrays of a batch of P positions (= node slots) and nb samples.  Training keeps every step's arrays, stacked with
// row stride P so that a weight gradient over all steps is one product over step P rows; evaluation keeps one step's and two
// alternating states, and carries no backward buffers.
struct SgBuf {
  long long P = 0; int d = 0; bool keep = false;
  float *H, *A, *R, *Z, *N, *GHN;                       // per step (H: steps + 1 states)
  float *XI, *XO, *GH, *GI, *HP, *Q2, *ALPHA;           // per position
  float *SL, *Q1, *CAT, *SH;                            // per sample
  float *DGI, *DGH, *DA, *DXI, *DXO;                    // the backward, per step
  float *DHD, *T1, *T2, *T3, *DH, *DHP, *DQ2, *DQV, *TP; // per position
  float *LOSS, *DSH, *DCAT, *DQ1, *TS;                  // per sample
  float* at(float* base, int w, int k) const { return keep ? base + (size_t)k * P * w : base; }
  float* h(int k) const { return keep ? H + (size_t)k * P * d : H + (size_t)(k & 1) * P * d; }
};
static size_t sg_pos_floats(int d, int steps, bool train) { return train ? (size_t)(17 * steps + 20) * d + 1 : (size_t)18 * d + 1; }
static size_t sg_smp_floats(int d, bool train) { return train ? (size_t)10 * d + 1 : (size_t)5 * d; }
// pcap positions and bcap samples of room; P the batch's positions (the stacked stride)
static void sg_carve(SgBuf& B, float* f, long long pcap, long long bcap, long long P, int d, int steps, bool train) {
  B.P = P; B.d = d; B.keep = train;
  const size_t ns = train ? steps : 1;
  auto take = [&](float** q, size_t w) { *q = f; f += (size_t)pcap * w; };
  auto smp = [&](float** q, size_t w) { *q = f; f += (size_t)bcap * w; };
  take(&B.H, (train ? ns + 1 : 2) * d); take(&B.A, ns * 2 * d); take(&B.R, ns * d); take(&B.Z, ns * d); take(&B.N, ns * d); take(&B.GHN, ns * d);
  take(&B.XI, d); take(&B.XO, d); take(&B.GH, 3 * d); take(&B.GI, 3 * d); take(&B.HP, d); take(&B.Q2, d); take(&B.ALPHA, 1);
  smp(&B.SL, d); smp(&B.Q1, d); smp(&B.CAT, 2 * d); smp(&B.SH, d);
  if (!train) return;
  take(&B.DGI, ns * 3 * d); take(&B.DGH, ns * 3 * d); take(&B.DA, ns * 2 * d); take(&B.DXI, ns * d); take(&B.DXO, ns * d);
  take(&B.DHD, d); take(&B.T1, d); take(&B.T2, d); take(&B.T3, d); take(&B.DH, d); take(&B.DHP, d); take(&B.DQ2, d); take(&B.DQV, d); take(&B.TP, d);
  smp(&B.LOSS, 1); smp(&B.DSH, d); smp(&B.DCAT, 2 * d); smp(&B.DQ1, d); smp(&B.TS, d);
}
constexpr int SG_INTS_POS = 11, SG_INTS_SMP = 2;
static void sg_carve_ints(SgDev& g, int* f, long long pcap) {
  int** pos[SG_INTS_POS] = {&g.ALIAS, &g.NX, &g.INS, &g.INC, &g.INL, &g.OUS, &g.OUC, &g.OUL, &g.NPS, &g.NPC, &g.NPL};
  for (int k = 0; k < SG_INTS_POS; k++) { *pos[k] = f; f += pcap; }
  g.NK = f; f += pcap; g.PY = f;                          // per sample (pcap >= the samples)
}

static unsigned sg_grid(long long n) { return (unsigned)((n + 255) / 256); }

// the encoder of a batch or chunk: SH [nb x d] (encoder products never split k)
static void sg_encode(cudaStream_t st, const SgDev& g, const SgBuf& B, const float* th, const SgLayout& Lo, int steps) {
  const int P = g.P, d = g.d, nb = g.nb;
  const unsigned ge = sg_grid((long long)P * d);
  k_sg_graph<<<nb, SG_THREADS, 0, st>>>(g, B.h(0));
  for (int k = 0; k < steps; k++) {
    const float* H = B.h(k);
    float* A = B.at(B.A, 2 * d, k);
    nm_gemm<NM_ENCODER>(st, nullptr, H, d, 1, th + Lo.Win, d, 1, B.XI, d, P, d, d);
    nm_gemm<NM_ENCODER>(st, nullptr, H, d, 1, th + Lo.Wout, d, 1, B.XO, d, P, d, d);
    nm_gemm<NM_ENCODER>(st, nullptr, H, d, 1, th + Lo.Whh, 3 * d, 1, B.GH, 3 * d, P, 3 * d, d);
    k_sg_agg<<<ge, 256, 0, st>>>(g, B.XI, B.XO, th + Lo.bin, th + Lo.bout, th + Lo.biah, th + Lo.boah, A);
    nm_gemm<NM_ENCODER>(st, nullptr, A, 2 * d, 1, th + Lo.Wih, 3 * d, 1, B.GI, 3 * d, P, 3 * d, 2 * d);
    k_sg_gate<<<ge, 256, 0, st>>>(P, d, B.GI, B.GH, th + Lo.bih, th + Lo.bhh, H, B.at(B.R, d, k), B.at(B.Z, d, k), B.at(B.N, d, k),
                                  B.at(B.GHN, d, k), B.h(k + 1));
  }
  k_sg_rows<<<sg_grid((long long)(P + nb) * d), 256, 0, st>>>(g, B.h(steps), B.HP, B.SL);
  nm_gemm<NM_ENCODER>(st, nullptr, B.SL, d, 1, th + Lo.W1, d, 1, B.Q1, d, nb, d, d);
  nm_gemm<NM_ENCODER>(st, nullptr, B.HP, d, 1, th + Lo.W2, d, 1, B.Q2, d, P, d, d);
  k_sg_readout<<<nb, SG_THREADS, 0, st>>>(g, B.HP, B.SL, B.Q1, B.Q2, th + Lo.b1, th + Lo.b2, th + Lo.q, B.ALPHA, B.CAT);
  nm_gemm<NM_ENCODER>(st, nullptr, B.CAT, 2 * d, 1, th + Lo.W3, d, 1, B.SH, d, nb, d, 2 * d);
  k_sg_bias<<<sg_grid((long long)nb * d), 256, 0, st>>>(B.SH, th + Lo.b3, (long long)nb * d, d);
}

// G[off ..] = the column sums of X [rows x w] in row order
static void sg_colsum(cudaStream_t st, float* part, const float* ones, const float* X, long long ldx, float* G, int rows, int w) {
  nm_gemm<NM_BACKWARD>(st, part, ones, 0, 0, X, ldx, 1, G, w, 1, w, rows);
}

// a batch's loss and gradient G of the loss (flat, the parameters' layout) at th; loss_out a device float
static void sg_grad(cudaStream_t st, const SgDev& g, const SgBuf& B, const NmScratch& ns, const float* th, const SgLayout& Lo, int steps, int NI,
                    float* G, const float* ones, float* loss_out) {
  const int P = g.P, d = g.d, nb = g.nb;
  const unsigned ge = sg_grid((long long)P * d);
  float* part = ns.part;
  sg_encode(st, g, B, th, Lo, steps);
  // the catalogue: logits, the softmax gradient, dL/ds_h and dE
  NmDev nd{};
  nd.P = nb; nd.d = d; nd.NI = NI; nd.S = ns.S; nd.PY = g.PY; nd.LOSS = B.LOSS; nd.re = 1.f;
  const float* E = th + Lo.E;
  nm_gemm<NM_CATALOGUE>(st, part, B.SH, d, 1, E, 1, d, ns.S, NI, nb, NI, d);
  k_nm_softmax<<<nb, 256, 0, st>>>(nd);
  k_nm_mean<<<1, 1024, 0, st>>>(B.LOSS, nb, loss_out);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, NI, 1, E, d, 1, B.DSH, d, nb, d, NI);
  nm_gemm<NM_CATALOGUE>(st, part, ns.S, 1, NI, B.SH, d, 1, G + Lo.E, d, NI, d, nb);
  // s_h = [s_g ; s_l] W3 + b3
  nm_gemm<NM_BACKWARD>(st, part, B.CAT, 1, 2 * d, B.DSH, d, 1, G + Lo.W3, d, 2 * d, d, nb);
  sg_colsum(st, part, ones, B.DSH, d, G + Lo.b3, nb, d);
  nm_gemm<NM_BACKWARD>(st, part, B.DSH, d, 1, th + Lo.W3, 1, d, B.DCAT, 2 * d, nb, 2 * d, d);
  // the readout
  k_sg_readout_bwd<<<nb, SG_THREADS, 0, st>>>(g, B.HP, B.Q1, B.Q2, th + Lo.b1, th + Lo.b2, th + Lo.q, B.ALPHA, B.DCAT, B.DHP, B.DQ2, B.DQV, B.DQ1);
  nm_gemm<NM_BACKWARD>(st, part, B.HP, 1, d, B.DQ2, d, 1, G + Lo.W2, d, d, d, P);
  sg_colsum(st, part, ones, B.DQ2, d, G + Lo.b2, P, d);
  sg_colsum(st, part, ones, B.DQV, d, G + Lo.q, P, d);
  nm_gemm<NM_BACKWARD>(st, part, B.DQ2, d, 1, th + Lo.W2, 1, d, B.TP, d, P, d, d);
  nm_gemm<NM_BACKWARD>(st, part, B.SL, 1, d, B.DQ1, d, 1, G + Lo.W1, d, d, d, nb);
  sg_colsum(st, part, ones, B.DQ1, d, G + Lo.b1, nb, d);
  nm_gemm<NM_BACKWARD>(st, part, B.DQ1, d, 1, th + Lo.W1, 1, d, B.TS, d, nb, d, d);
  k_sg_node_bwd<<<nb, SG_THREADS, 0, st>>>(g, B.DHP, B.TP, B.DCAT, B.TS, B.DH);
  // the propagation steps in reverse: dL/dH_k = DHD + DGH W_hh^T + DXI W_in^T + DXO W_out^T
  for (int k = steps - 1; k >= 0; k--) {
    const bool top = k == steps - 1;
    float *DGI = B.at(B.DGI, 3 * d, k), *DGH = B.at(B.DGH, 3 * d, k), *DA = B.at(B.DA, 2 * d, k), *DXI = B.at(B.DXI, d, k), *DXO = B.at(B.DXO, d, k);
    k_sg_gate_bwd<<<ge, 256, 0, st>>>(P, d, top ? B.DH : B.DHD, top ? nullptr : B.T1, B.T2, B.T3, B.h(k), B.at(B.R, d, k), B.at(B.Z, d, k),
                                      B.at(B.N, d, k), B.at(B.GHN, d, k), DGI, DGH, B.DHD);
    nm_gemm<NM_BACKWARD>(st, part, DGI, 3 * d, 1, th + Lo.Wih, 1, 3 * d, DA, 2 * d, P, 2 * d, 3 * d);
    k_sg_agg_bwd<<<ge, 256, 0, st>>>(g, DA, DXI, DXO);
    nm_gemm<NM_BACKWARD>(st, part, DGH, 3 * d, 1, th + Lo.Whh, 1, 3 * d, B.T1, d, P, d, 3 * d);
    nm_gemm<NM_BACKWARD>(st, part, DXI, d, 1, th + Lo.Win, 1, d, B.T2, d, P, d, d);
    nm_gemm<NM_BACKWARD>(st, part, DXO, d, 1, th + Lo.Wout, 1, d, B.T3, d, P, d, d);
  }
  // the shared weights over every step at once: rows k P + p of the stacked arrays
  const int R = steps * P;
  nm_gemm<NM_BACKWARD>(st, part, B.A, 1, 2 * d, B.DGI, 3 * d, 1, G + Lo.Wih, 3 * d, 2 * d, 3 * d, R);
  sg_colsum(st, part, ones, B.DGI, 3 * d, G + Lo.bih, R, 3 * d);
  nm_gemm<NM_BACKWARD>(st, part, B.H, 1, d, B.DGH, 3 * d, 1, G + Lo.Whh, 3 * d, d, 3 * d, R);
  sg_colsum(st, part, ones, B.DGH, 3 * d, G + Lo.bhh, R, 3 * d);
  nm_gemm<NM_BACKWARD>(st, part, B.H, 1, d, B.DXI, d, 1, G + Lo.Win, d, d, d, R);
  sg_colsum(st, part, ones, B.DXI, d, G + Lo.bin, R, d);
  nm_gemm<NM_BACKWARD>(st, part, B.H, 1, d, B.DXO, d, 1, G + Lo.Wout, d, d, d, R);
  sg_colsum(st, part, ones, B.DXO, d, G + Lo.bout, R, d);
  sg_colsum(st, part, ones, B.DA, 2 * d, G + Lo.biah, R, d);
  sg_colsum(st, part, ones, B.DA + d, 2 * d, G + Lo.boah, R, d);
  // the node embeddings: dL/dH0 rows added to E's rows, slots sorted by (item, slot)
  k_sg_dsum<<<ge, 256, 0, st>>>((long long)P * d, B.DHD, B.T1, B.T2, B.T3, B.DH);
  NmDev ne{};
  ne.P = P; ne.d = d; ne.DEMB = B.DH; ne.PS = g.ALIAS; ne.re = 1.f;
  k_nm_keys<<<(P + 255) / 256, 256, 0, st>>>(g.NX, P, ns.keys);
  int end_bit = 33;
  while (end_bit < 64 && ((unsigned long long)NI >> (end_bit - 32)) != 0ull) end_bit++;
  size_t cb = ns.cub_bytes;
  cub::DeviceRadixSort::SortKeys(ns.cub, cb, ns.keys, ns.keys2, P, 0, end_bit, st);
  k_nm_scatter<<<ge, 256, 0, st>>>(ne, ns.keys2, G + Lo.E);
}

static bool sg_shape_ok(int step, int len) { return step >= 1 && step <= SG_STEP_MAX && len >= 1 && len <= SG_LEN_MAX; }
#define SG_SHAPE_MSG ": need step in 1 .. 8 and max_len in 1 .. 512"

// the model buffers of an SR-GNN handle (NARM's fields): parameters, double(E) and zero biases for bpr_blocks, a device 1.0f
static int sg_set_model(g4r_baselines* h, int32_t step, int32_t max_len, const float* params, int64_t n_params, const char* who) {
  if (!params) FAIL(G4R_ERR_INVALID, std::string(who) + ": null parameters");
  if (!sg_shape_ok(step, max_len)) FAIL(G4R_ERR_INVALID, std::string(who) + SG_SHAPE_MSG);
  const SgLayout L = sg_layout(h->n_items, h->n_keep);
  if (n_params != (int64_t)L.n) FAIL(G4R_ERR_INVALID, std::string(who) + ": need n_params = n_items d + 15 d^2 + 14 d = " + std::to_string(L.n));
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
  h->sg_step = step; h->nm_len = max_len; h->nm_n = L.n;
  const size_t nE = (size_t)h->n_items * h->n_keep;
  k_nm_to_double<<<(unsigned)((nE + 255) / 256), 256, 0, st>>>(h->dNmTh, nE, h->dI);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  h->ready = true;
  return G4R_OK;
}

extern "C" int g4r_bl_srgnn_import(g4r_baselines* h, int32_t step, int32_t max_len, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SRGNN) FAIL(G4R_ERR_STATE, "g4r_bl_srgnn_import: the handle is not an SR-GNN");
  return sg_set_model(h, step, max_len, params, n_params, "g4r_bl_srgnn_import");
}

extern "C" int g4r_bl_srgnn_export(g4r_baselines* h, float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SRGNN || !h->dNmTh) FAIL(G4R_ERR_STATE, "g4r_bl_srgnn_export: no SR-GNN parameters (g4r_bl_srgnn_begin or g4r_bl_srgnn_import)");
  if (!params || n_params != (int64_t)h->nm_n) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_export: need n_params floats");
  cudaSetDevice(h->device);
  CK(cudaMemcpyAsync(params, h->dNmTh, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// the samples of a fit (SR-GNN's and STAMP's): per session every (prefix, next item) pair, the prefix cut to its last max_len
// inputs; per sample its first input and its inputs
static void sg_samples(const int64_t* off, int64_t n_sessions, int max_len, std::vector<int64_t>& s0, std::vector<int>& sn) {
  for (int64_t s = 0; s < n_sessions; s++)
    for (int64_t j = 1; j < off[s + 1] - off[s]; j++) {
      const int64_t a = std::max<int64_t>(0, j - max_len);
      s0.push_back(off[s] + a); sn.push_back((int)(j - a));
    }
}

// the positions of the largest batch: the batch_size longest samples
static long long sg_longest(const std::vector<int>& sn, int batch_size) {
  std::vector<int> srt(sn);
  const size_t top = std::min<size_t>(batch_size, srt.size());
  std::partial_sort(srt.begin(), srt.begin() + top, srt.end(), std::greater<int>());
  long long Pmax = 0;
  for (size_t k = 0; k < top; k++) Pmax += srt[k];
  return Pmax;
}

extern "C" int g4r_bl_srgnn_begin(g4r_baselines* h, int32_t step, int32_t max_len, int32_t batch_size, const int64_t* session_offsets,
                                  int64_t n_sessions, const int32_t* items, int64_t n_entries, const float* params, int64_t n_params) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SRGNN) FAIL(G4R_ERR_STATE, "g4r_bl_srgnn_begin: the handle is not an SR-GNN");
  if (!session_offsets || !items || n_sessions < 1 || n_entries < 2 || batch_size < 1)
    FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_begin: null argument, no sessions or batch_size < 1");
  const int NI = h->n_items, dd = h->n_keep;
  if (!sg_shape_ok(step, max_len)) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_begin" SG_SHAPE_MSG);
  if (n_entries > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_begin: more than 2^31 - 1 entries");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_entries)) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_begin: session offsets must rise from 0 to n_entries");
  for (int64_t e = 0; e < n_entries; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_srgnn_begin: item index out of range");
  if ((uint64_t)batch_size * (uint64_t)max_len * (uint64_t)(step + 1) * 3ull * (uint64_t)dd >= 0x80000000ull)
    FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_begin: batch_size * max_len * (step + 1) * 3 d must stay below 2^31 (flat indices of a batch)");
  std::vector<int64_t> s0; std::vector<int> sn;
  sg_samples(session_offsets, n_sessions, max_len, s0, sn);
  if (s0.empty()) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_begin: no session of at least 2 events");
  if (s0.size() > (size_t)INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_begin: more than 2^31 - 1 samples");
  const long long Pmax = sg_longest(sn, batch_size);
  const SgLayout L = sg_layout(NI, dd);
  const size_t act = (size_t)Pmax * sg_pos_floats(dd, step, true) * 4 + (size_t)batch_size * sg_smp_floats(dd, true) * 4;
  const size_t need = (size_t)batch_size * NI * 4 + act + (size_t)Pmax * ((SG_INTS_POS + 1) * 4 + 16) + NM_PART_CAP * 4 + 3 * L.n * 4 +
                      (size_t)n_entries * 4 + s0.size() * 12 + ((size_t)64 << 20);
  int rc = sg_set_model(h, step, max_len, params, n_params, "g4r_bl_srgnn_begin");
  if (rc) return rc;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    h->err = "g4r_bl_srgnn_begin: the fit needs " + std::to_string(need) + " bytes of device memory (the logits of the largest batch " +
             std::to_string((size_t)batch_size * NI * 4) + ", its activations " + std::to_string(act) + "), " + std::to_string(free_b) + " are free";
    return G4R_ERR_CUDA;
  }
  cudaStream_t st = h->stream;
  h->ready = false;
  NmScratch& s = h->nm_s;
  s = NmScratch{};
  size_t cb = 0;
  CK(cub::DeviceRadixSort::SortKeys(nullptr, cb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)Pmax, 0, 64));
  const long long icap = std::max<long long>(Pmax, batch_size);
  CK(nm_take(h, &s.part, NM_PART_CAP)); CK(nm_take(h, &s.S, (size_t)batch_size * NI)); CK(nm_take(h, &s.keys, Pmax)); CK(nm_take(h, &s.keys2, Pmax));
  CK(nm_take(h, &s.cub, cb));
  s.cub_bytes = cb;
  CK(nm_take(h, &h->sg_f, (size_t)Pmax * sg_pos_floats(dd, step, true) + (size_t)batch_size * sg_smp_floats(dd, true)));
  CK(nm_take(h, &h->sg_i, (size_t)icap * (SG_INTS_POS + SG_INTS_SMP)));
  CK(nm_take(h, &h->dNmG, L.n)); CK(nm_take(h, &h->dNmM, L.n)); CK(nm_take(h, &h->dNmV, L.n)); CK(nm_take(h, &h->dNmItems, n_entries));
  CK(nm_take(h, &h->dNmLoss, 1));
  CK(cudaMemsetAsync(h->dNmM, 0, L.n * sizeof(float), st)); CK(cudaMemsetAsync(h->dNmV, 0, L.n * sizeof(float), st));
  CK(cudaMemcpyAsync(h->dNmItems, items, n_entries * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  h->sg_start.swap(s0); h->sg_len.swap(sn);
  h->nm_bs = batch_size; h->nm_Pmax = Pmax; h->sg_icap = icap; h->nm_step = 0; h->nm_fit = true;
  h->ready = true;
  return G4R_OK;
}

// the batches of a list of samples: per entry its first input, inputs and slot offset within its batch; per batch (first entry,
// P).  The scratch holds the positions of the batch_size longest samples (nm_Pmax); a batch that repeats a long sample can
// exceed it, and is refused here, before any device write.
static int sg_plan(g4r_baselines* h, const int32_t* samples, int64_t n, std::vector<long long>& ps, std::vector<int>& pl, std::vector<int>& po,
                   std::vector<std::pair<int64_t, int>>& batches, const char* who) {
  ps.resize(n); pl.resize(n); po.resize(n);
  for (int64_t b0 = 0; b0 < n; b0 += h->nm_bs) {
    long long P = 0;
    for (int64_t q = b0; q < std::min<int64_t>(n, b0 + h->nm_bs); q++) {
      const int k = samples[q];
      ps[q] = h->sg_start[k]; pl[q] = h->sg_len[k]; po[q] = (int)P; P += pl[q];
    }
    if (P > h->nm_Pmax)
      FAIL(G4R_ERR_INVALID, std::string(who) + ": a batch holds " + std::to_string(P) + " positions, more than the " + std::to_string(h->nm_Pmax) +
                                " of the batch_size longest samples the fit was begun with (a sample repeated in a batch?)");
    batches.push_back({b0, (int)P});
  }
  return G4R_OK;
}

static int sg_check_run(g4r_baselines* h, const int32_t* samples, int64_t n, const char* who) {
  if (h->kind != BL_SRGNN) FAIL(G4R_ERR_STATE, std::string(who) + ": the handle is not an SR-GNN");
  if (!h->nm_fit) FAIL(G4R_ERR_STATE, std::string(who) + ": no fit begun (g4r_bl_srgnn_begin)");
  if (!samples || n < 1) FAIL(G4R_ERR_INVALID, std::string(who) + ": no samples");
  const int64_t ns = (int64_t)h->sg_start.size();
  for (int64_t q = 0; q < n; q++) if (samples[q] < 0 || samples[q] >= ns) FAIL(G4R_ERR_INDEX, std::string(who) + ": sample index out of range");
  return G4R_OK;
}

// the SgDev and SgBuf of a training batch: nb samples at plan slices (device) of P positions
static void sg_train_batch(g4r_baselines* h, SgDev& g, SgBuf& B, const long long* ps, const int* pl, const int* po, int nb, int P) {
  g = SgDev{};
  g.items = h->dNmItems; g.sstart = ps; g.slen = pl; g.soff = po; g.nb = nb; g.P = P;
  g.E = h->dNmTh; g.d = h->n_keep; g.train = 1;
  sg_carve_ints(g, h->sg_i, h->sg_icap);
  sg_carve(B, h->sg_f, h->nm_Pmax, h->nm_bs, P, h->n_keep, h->sg_step, true);
}

extern "C" int g4r_bl_srgnn_grads(g4r_baselines* h, const int32_t* samples, int32_t n, float* loss, float* grads) {
  if (!h) return G4R_ERR_INVALID;
  int rc = sg_check_run(h, samples, n, "g4r_bl_srgnn_grads");
  if (rc) return rc;
  if (n > h->nm_bs || !grads) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_grads: need n <= batch_size and grads");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = sg_plan(h, samples, n, ps, pl, po, batches, "g4r_bl_srgnn_grads");
  if (rc) return rc;
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  SgDev g; SgBuf B;
  sg_train_batch(h, g, B, dps, dpl, dpo, n, batches[0].second);
  sg_grad(st, g, B, h->nm_s, h->dNmTh, sg_layout(h->n_items, h->n_keep), h->sg_step, h->n_items, h->dNmG, h->dNmOne, h->dNmLoss);
  CK(cudaGetLastError());
  float l = 0.f;
  CK(cudaMemcpyAsync(&l, h->dNmLoss, sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(grads, h->dNmG, h->nm_n * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (loss) *loss = l;
  return G4R_OK;
}

extern "C" int g4r_bl_srgnn_epoch(g4r_baselines* h, const int32_t* order, int64_t n_order, float learning_rate, float l2, float* losses,
                                  float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  int rc = sg_check_run(h, order, n_order, "g4r_bl_srgnn_epoch");
  if (rc) return rc;
  if (!(learning_rate > 0.f && std::isfinite(learning_rate))) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_epoch: learning_rate must be finite and > 0");
  if (!(l2 >= 0.f && std::isfinite(l2))) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_epoch: l2 must be finite and >= 0");
  std::vector<long long> ps; std::vector<int> pl, po; std::vector<std::pair<int64_t, int>> batches;
  rc = sg_plan(h, order, n_order, ps, pl, po, batches, "g4r_bl_srgnn_epoch");
  if (rc) return rc;
  if (h->nm_step + (int64_t)batches.size() > 0xffffffffll) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_epoch: more than 2^32 steps since the fit began");
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  const SgLayout Lo = sg_layout(h->n_items, h->n_keep);
  // the whole epoch's plan goes up once; each batch reads its slice
  BlBufs bb;
  const long long* dps = nullptr; const int *dpl = nullptr, *dpo = nullptr; float* dloss = nullptr;
  CK(bb.put(&dps, ps.data(), ps.size(), st)); CK(bb.put(&dpl, pl.data(), pl.size(), st)); CK(bb.put(&dpo, po.data(), po.size(), st));
  CK(bb.take(&dloss, batches.size()));
  CK(cudaEventRecord(h->ev0, st));
  for (size_t b = 0; b < batches.size(); b++) {
    const int64_t q0 = batches[b].first;
    SgDev g; SgBuf B;
    sg_train_batch(h, g, B, dps + q0, dpl + q0, dpo + q0, (int)std::min<int64_t>(h->nm_bs, n_order - q0), batches[b].second);
    sg_grad(st, g, B, h->nm_s, h->dNmTh, Lo, h->sg_step, h->n_items, h->dNmG, h->dNmOne, dloss + b);
    k_sg_l2<<<(unsigned)((Lo.n + 255) / 256), 256, 0, st>>>(h->dNmG, h->dNmTh, Lo.n, l2);
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

// every counted event's s_h (eval mode; its own sample of the last max_len inputs of its prefix) into qev [n_ev x d] on the
// device, in chunks of at most SG_EVAL_POS positions; a chunk's samples are consecutive counted events, so s_h lands in place
static int sg_encode_events(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* off, int64_t n_sessions, const int32_t* n_history,
                            const std::vector<int64_t>& ev0, float* qev) {
  const int dd = h->n_keep, len = h->nm_len;
  cudaStream_t st = h->stream;
  const SgLayout Lo = sg_layout(h->n_items, dd);
  BlBufs bb;
  long long* sstart = nullptr; int *slen = nullptr, *soff = nullptr, *gi = nullptr;
  float* f = nullptr;
  const int* dItems = nullptr;
  CK(bb.take(&sstart, SG_EVAL_POS)); CK(bb.take(&slen, SG_EVAL_POS)); CK(bb.take(&soff, SG_EVAL_POS));
  CK(bb.take(&gi, (size_t)SG_EVAL_POS * (SG_INTS_POS + SG_INTS_SMP)));
  CK(bb.take(&f, (size_t)SG_EVAL_POS * (sg_pos_floats(dd, 1, false) + sg_smp_floats(dd, false))));
  CK(bb.put(&dItems, items, n_events, st));
  SgDev g{};
  g.items = dItems; g.sstart = sstart; g.slen = slen; g.soff = soff; g.E = h->dNmTh; g.d = dd; g.train = 0;
  sg_carve_ints(g, gi, SG_EVAL_POS);
  std::vector<long long> ps; std::vector<int> pl, po;
  int P = 0;
  int64_t e_first = 0;
  auto flush = [&]() -> int {
    if (ps.empty()) return G4R_OK;
    const int nb = (int)ps.size();
    CK(cudaMemcpyAsync(sstart, ps.data(), nb * sizeof(long long), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(slen, pl.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(soff, po.data(), nb * sizeof(int), cudaMemcpyHostToDevice, st));
    g.nb = nb; g.P = P;
    SgBuf B;
    sg_carve(B, f, SG_EVAL_POS, SG_EVAL_POS, P, dd, 1, false);
    B.SH = qev + (size_t)e_first * dd;
    sg_encode(st, g, B, h->dNmTh, Lo, h->sg_step);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));                      // the host arrays are reused by the next chunk
    e_first += nb;
    ps.clear(); pl.clear(); po.clear(); P = 0;
    return G4R_OK;
  };
  for (int64_t sI = 0; sI < n_sessions; sI++) {
    const int64_t st0 = off[sI], en = off[sI + 1];
    const int64_t i0 = std::max<int64_t>(n_history ? n_history[sI] : 0, 1) - 1;   // input index of the first counted event
    for (int64_t i = i0; i <= en - st0 - 2; i++) {
      const int n = (int)std::min<int64_t>(i + 1, len);
      if (P + n > SG_EVAL_POS) { const int rc = flush(); if (rc) return rc; }
      ps.push_back(st0 + i + 1 - n); pl.push_back(n); po.push_back(P); P += n;
    }
  }
  return flush();
}

extern "C" int g4r_bl_srgnn_encode(g4r_baselines* h, const int32_t* items, int64_t n_events, const int64_t* session_offsets, int64_t n_sessions,
                                   const int32_t* n_history, float* q, int64_t n_q) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SRGNN || !h->ready) FAIL(G4R_ERR_STATE, "g4r_bl_srgnn_encode: no SR-GNN parameters (g4r_bl_srgnn_begin or g4r_bl_srgnn_import)");
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items) || n_q < 0 || (n_q > 0 && !q))
    FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_encode: null or out-of-range argument");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_encode: session offsets must rise from 0 to n_events");
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= h->n_items) FAIL(G4R_ERR_INDEX, "g4r_bl_srgnn_encode: item index out of range");
  std::vector<int64_t> ev0;
  int rc = bl_counted(h, "g4r_bl_srgnn_encode", session_offsets, n_sessions, n_history, ev0);
  if (rc) return rc;
  if (n_q != ev0[n_sessions]) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_encode: n_q must be the number of counted events");
  if (n_q > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_srgnn_encode: more than 2^31 - 1 counted events");
  cudaSetDevice(h->device);
  BlBufs bb;
  float* dq = nullptr;
  CK(bb.take(&dq, (size_t)n_q * h->n_keep));
  rc = sg_encode_events(h, items, n_events, session_offsets, n_sessions, n_history, ev0, dq);
  if (rc) return rc;
  if (n_q) CK(cudaMemcpyAsync(q, dq, (size_t)n_q * h->n_keep * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return G4R_OK;
}

// the ranking of a g4r_bl_evaluate call of an SR-GNN: every counted event's s_h, then BPR's ranking with I = double(E), bI = 0
static int srgnn_rank(g4r_baselines* h, BlCall& c) {
  float* dq = nullptr;
  CK(c.bb.take(&dq, (size_t)c.n_ev * h->n_keep));
  const int rc = sg_encode_events(h, c.items, c.n_events, c.off, c.n_sessions, c.n_history, c.ev0, dq);
  if (rc) return rc;
  return bpr_blocks(h, c, dq);
}
