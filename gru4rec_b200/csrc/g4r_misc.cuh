// g4r_misc.cuh -- kernels outside the per-step critical path: binary search (K2'), row gather (K1'),
// MRG31k3p uniforms, and the per-window column plan (sort of each step's score columns by item).
#pragma once
#include "g4r_kernels.cuh"

// GpuBinarySearchSorted semantics (custom_theano_ops.py:318-349): np.searchsorted(d, x, 'right') except
// x <= d[0] -> 0 and x > d[-1] -> len(d); x == d[-1] -> len(d)-1.
template <class TOut>
__global__ void __launch_bounds__(256) k_searchsorted(const float* __restrict__ d, int ld, const float* __restrict__ x, int64_t n, TOut* __restrict__ y) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float val = x[i];
  long long a = 0, b = ld - 1;
  const float minval = d[0], maxval = d[ld - 1];
  if (val > maxval) { a = ld; b = ld; }
  else if (val <= minval) { a = 0; b = 0; }
  while (b - a > 0) {
    const long long hh = (b + a) / 2;
    const float t = d[hh];
    if (val < t) b = hh; else a = hh + 1;
  }
  y[i] = (TOut)b;
}

// GpuAdvancedSubtensor1_fast semantics (custom_theano_ops.py:482-522): out[i,:] = in[idx[i],:], negative index
// wraps once, out of range sets the error flag.  One warp per row, 16-byte loads when cols % 4 == 0.
__global__ void __launch_bounds__(128) k_gather_rows(const float* __restrict__ in, int64_t rows, int64_t cols, const long long* __restrict__ idx,
                                                      int64_t n_idx, float* __restrict__ out, int* err) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int64_t i = (int64_t)blockIdx.x * nwarp + warp; i < n_idx; i += (int64_t)gridDim.x * nwarp) {
    long long r = idx[i];
    if (r < 0) r += rows;
    if (r < 0 || r >= rows) { if (lane == 0) *err = 1; continue; }
    const float* src = in + r * cols;
    float* dst = out + i * cols;
    if ((cols & 3) == 0) {
      for (int64_t c4 = lane; c4 < cols / 4; c4 += 32) st4(dst + c4 * 4, ld4(src + c4 * 4));
    } else {
      for (int64_t c = lane; c < cols; c += 32) dst[c] = src[c];
    }
  }
}

// MRG31k3p (L'Ecuyer) as used by theano.sandbox.rng_mrg: stream i produces samples i, i+n_streams, ...
__global__ void __launch_bounds__(128) k_mrg_uniform(int32_t* __restrict__ state, int n_streams, float* __restrict__ out, int64_t n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_streams) return;
  const uint32_t M1 = 2147483647u, M2 = 2147462579u;
  uint32_t x11 = state[i * 6 + 0], x12 = state[i * 6 + 1], x13 = state[i * 6 + 2], x21 = state[i * 6 + 3], x22 = state[i * 6 + 4], x23 = state[i * 6 + 5];
  for (int64_t p = i; p < n; p += n_streams) {
    uint32_t y1 = ((x12 & 511u) << 22) + (x12 >> 9) + ((x13 & 16777215u) << 7) + (x13 >> 24);
    if (y1 >= M1) y1 -= M1;
    y1 += x13;
    if (y1 >= M1) y1 -= M1;
    x13 = x12; x12 = x11; x11 = y1;
    y1 = ((x21 & 65535u) << 15) + 21069u * (x21 >> 16);
    if (y1 >= M2) y1 -= M2;
    uint32_t y2 = ((x23 & 65535u) << 15) + 21069u * (x23 >> 16);
    if (y2 >= M2) y2 -= M2;
    y2 += x23;
    if (y2 >= M2) y2 -= M2;
    y2 += y1;
    if (y2 >= M2) y2 -= M2;
    x23 = x22; x22 = x21; x21 = y2;
    const int32_t diff = (x11 <= x21) ? (int32_t)(x11 - x21 + M1) : (int32_t)(x11 - x21);
    out[p] = (float)diff * 4.6566126e-10f;
  }
  state[i * 6 + 0] = x11; state[i * 6 + 1] = x12; state[i * 6 + 2] = x13; state[i * 6 + 3] = x21; state[i * 6 + 4] = x22; state[i * 6 + 5] = x23;
}

// Catalogue growth (g4r_copy_item_tables): dst [n_new x ld] takes rows 0 .. n_old-1 of src [n_old x ld] as they are, padding
// columns included; rows n_old .. n_new-1 take `fill` ([n_new - n_old x cols], dense) in their first `cols` columns, or zero
// when fill == nullptr (optimizer state), and zero in the padding columns.
__global__ void __launch_bounds__(256) k_rows_extend(float* __restrict__ dst, const float* __restrict__ src, int64_t n_old, int64_t n_new,
                                                      int64_t ld, int64_t cols, const float* __restrict__ fill) {
  const int64_t n = n_new * ld, n_copy = n_old * ld;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    if (i < n_copy) v = src[i];
    else if (fill) { const int64_t r = i / ld, c = i - r * ld; if (c < cols) v = fill[(r - n_old) * cols + c]; }
    dst[i] = v;
  }
}

// Column plan of one step: score columns [Y | samples] sorted by (item, position); chunk boundaries that never
// split a duplicate group; target column of each lane; duplicate chains of X.  One CTA per step.
__global__ void __launch_bounds__(256) k_plan(ModelDev md, int* xnext, uint8_t* xflag, int npow2) {
  extern __shared__ __align__(16) unsigned long long keys[];
  const int s = blockIdx.x;
  const int tid = threadIdx.x;
  const int B = md.B;
  const int M = md.wM[s], sti = md.wSti[s];
  const int S = sti >= 0 ? md.S : 0, N = M + S;
  const int* Yp = md.wY + (size_t)s * B;
  const int* Xp = md.wX + (size_t)s * B;
  const int* smp = sti >= 0 ? md.ST + (size_t)sti * md.S : nullptr;
  for (int i = tid; i < npow2; i += blockDim.x) {
    unsigned long long key = ~0ULL;
    int item = -1;
    if (i < M) item = Yp[i]; else if (i < N) item = smp[i - M];
    if (item >= 0) {
      if (item >= md.n_items) { atomicExch(md.nanflag + 1, 1); item = md.n_items - 1; }
      // row-sharded tables: owner-major order (owner = item % R), so that every owner's columns are contiguous in the
      // sorted list of every rank and the lists can be merged per owner (g4r_shard.cuh)
      const unsigned hi = md.shardR > 0 ? (unsigned)(item % md.shardR) * (unsigned)md.n_items + (unsigned)item : (unsigned)item;
      key = ((unsigned long long)hi << 32) | (unsigned)i;
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < npow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          const bool up = ((i & k) == 0);
          if ((a > b) == up) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  int* pItem = md.pItem + (size_t)s * md.NP;
  int* pPos = md.pPos + (size_t)s * md.NP;
  for (int j = tid; j < N; j += blockDim.x) {
    const unsigned long long key = keys[j];
    const int hi = (int)(key >> 32), pos = (int)(key & 0xffffffffu);
    const int item = md.shardR > 0 ? hi % md.n_items : hi;
    pItem[j] = item; pPos[j] = pos;
    if (md.shardR > 0) md.pKey[(size_t)s * md.NP + j] = hi;
    if (pos < M) md.pTcol[(size_t)s * B + pos] = j;
  }
  for (int c = tid; c <= md.NCH; c += blockDim.x) {
    int j = (int)(((long long)c * N + md.NCH - 1) / md.NCH);
    if (c == md.NCH) j = N;
    // single GPU: a chunk never splits a duplicate group (its CTA owns the item's row update).  Sharded: the rows are updated by
    // their owner from the merged plan, so the chunks are plain equal splits.
    if (md.shardR == 0) while (j > 0 && j < N && (keys[j] >> 32) == (keys[j - 1] >> 32)) j++;
    md.pCbeg[(size_t)s * (md.NCH + 1) + c] = min(j, N);
  }
  __syncthreads();
  // largest chunk of the window (the role-specialised kernel handles chunks of at most 32 columns)
  for (int c = tid; c < md.NCH; c += blockDim.x) {
    const int w = md.pCbeg[(size_t)s * (md.NCH + 1) + c + 1] - md.pCbeg[(size_t)s * (md.NCH + 1) + c];
    if (w > 32) atomicMax(md.nanflag + 2, w);
  }
  for (int b = tid; b < M; b += blockDim.x) {
    const int x = Xp[b];
    uint8_t f = 1; int nx = -1;
    for (int q = 0; q < b; q++) if (Xp[q] == x) { f = 0; break; }
    for (int q = b + 1; q < M; q++) if (Xp[q] == x) { nx = q; break; }
    if (md.mode == 2 && md.shardR == 0) {   // does the item also occur among the score columns?
      int lo = 0, hi = N;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if ((int)(keys[mid] >> 32) < x) lo = mid + 1; else hi = mid; }
      if (lo < N && (int)(keys[lo] >> 32) == x) f |= 2;
    }
    xnext[(size_t)s * B + b] = nx;
    xflag[(size_t)s * B + b] = f;
  }
}
