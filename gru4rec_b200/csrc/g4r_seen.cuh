// g4r_seen.cuh -- exclude_seen in evaluation (DESIGN §3g): per scoring-state slot, the sorted distinct items its session has
// input so far.  The lists are keyed like the hidden state (slot[s][b]), so lanes compacted in the epoch's tail keep theirs, and
// a lane's zero-before flag (bit 1 of F) clears its list just as it zeroes its state.  Included by g4r_eval.cuh before the tile
// kernels (k_eval_tgt / k_eval_score / k_eval_tc / k_eval_rank take a SeenDev in their SEEN instances).
#pragma once

struct SeenDev {
  int* list = nullptr;     // [B x cap] per state slot of the schedule: the distinct inputs of its session so far, ascending
  int* n = nullptr;        // [Be] their number
  int cap = 0;             // the schedule's longest session minus one (a session of length l has l - 1 inputs)
  int* miss = nullptr;     // [Be] per lane of the current mini-batch: 1 if its target is in its seen set
};

// first position p of the sorted l[0 .. n) with l[p] >= v (also the exclusion lists of g4r_topk.cuh)
__device__ __forceinline__ int sorted_lb(const int* __restrict__ l, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (l[m] < v) lo = m + 1; else hi = m; }
  return lo;
}
// v in the sorted l[0 .. n)
__device__ __forceinline__ bool sorted_has(const int* __restrict__ l, int n, int v) {
  const int p = sorted_lb(l, n, v);
  return p < n && l[p] == v;
}

// lane b of step s, once per mini-batch (k_eval_tgt<true>, before anything reads the lists): its input joins its slot's list
// (cleared first on a zero-before flag); returns whether `target` is in the list afterwards.  Each lane owns its slot, so the
// lanes need no synchronisation.
__device__ __forceinline__ bool seen_insert(const ModelDev& md, const SeenDev& sd, int s, int b, int target) {
  const size_t o = (size_t)s * md.B + b;
  const int sl = md.wSlot[o], x = md.wX[o];
  int* l = sd.list + (size_t)sl * sd.cap;
  int n = (md.wF[o] & 2) ? 0 : sd.n[sl];
  const int p = sorted_lb(l, n, x);
  if ((p == n || l[p] != x) && n < sd.cap) {
    for (int j = n; j > p; j--) l[j] = l[j - 1];
    l[p] = x;
    n++;
  }
  sd.n[sl] = n;
  return target == x || sorted_has(l, n, target);
}

// the lists of the M lanes of step s as the sorted CSR exclusions of the top-k kernels (lane b: ex[ex_off[b] .. ex_off[b+1])),
// one block: each thread takes a run of lanes, a shared scan of the run lengths gives the offsets
constexpr int SEEN_CSR_THREADS = 1024;
__global__ void __launch_bounds__(SEEN_CSR_THREADS) k_seen_csr(int slot, int s, SeenDev sd, int* __restrict__ ex_off, int* __restrict__ ex) {
  const ModelDev& md = MD;
  __shared__ int part[SEEN_CSR_THREADS];
  const int M = md.wM[s], tid = threadIdx.x;
  const int per = (M + SEEN_CSR_THREADS - 1) / SEEN_CSR_THREADS, b0 = min(M, tid * per), b1 = min(M, b0 + per);
  const int* sl = md.wSlot + (size_t)s * md.B;
  int sum = 0;
  for (int b = b0; b < b1; b++) sum += sd.n[sl[b]];
  part[tid] = sum;
  __syncthreads();
  for (int o = 1; o < SEEN_CSR_THREADS; o <<= 1) {
    const int v = tid >= o ? part[tid - o] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  int off = part[tid] - sum;
  for (int b = b0; b < b1; b++) {
    const int n = sd.n[sl[b]];
    const int* l = sd.list + (size_t)sl[b] * sd.cap;
    ex_off[b] = off;
    for (int j = 0; j < n; j++) ex[off + j] = l[j];
    off += n;
  }
  if (tid == SEEN_CSR_THREADS - 1) ex_off[M] = part[tid];
}
