// g4r_rules.cuh -- the rule-based session baselines on the device (DESIGN §3q): sequential rules (SR) and association rules (AR).
// The fit counts, per item i, the weighted pairs (i, j) of the training sessions in uint64 and keeps each row's `pruning` largest
// weights in ItemKNN's row layout; g4r_bl_evaluate ranks SR / AR handles with the ItemKNN instance of k_bl_rank.  Included from
// g4r_lib.cu after g4r_baselines.cuh (KF_*, bl_fit_grid, bl_scan, bl_row_order, bl_keep_row, bl_fit_end, the handle).
#pragma once

constexpr int RULES_STEPS_MAX = 20;

struct RulesFitDev {
  const int64_t* off; const int* items; const int* ev_sess;   // the sessions' events in time order, the session of each event
  const int64_t* i_off; const int* i_pos;                       // per item the positions of its events
  const int* order; int* next;                                  // rows by decreasing pair work; the queue head
  unsigned long long* acc; int* touched; double* w;             // per CTA: dense W [n_items], touched columns, their weights
  unsigned long long inc[RULES_STEPS_MAX + 1];                  // SR: the addend L * f(d) of distance d
  double L;
  int n_items, n_keep, steps;
  int* out_idx; double* out_sim; int* out_len;
};

// warp per session: each event's session, its item's occurrence count and pair work (SR: min(steps, events after it); AR: the
// session's other events), and the total pair work
template <bool AR>
__global__ void __launch_bounds__(256) k_rules_events(const int64_t* off, int64_t S, const int* items, int steps, int* ev_sess,
                                                      unsigned long long* i_cnt, unsigned long long* work, unsigned long long* pairs) {
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (s >= S) return;
  const int64_t st = off[s], en = off[s + 1];
  unsigned long long tot = 0;
  for (int64_t e = st + lane; e < en; e += 32) {
    const int j = items[e];
    const unsigned long long w = AR ? (unsigned long long)(en - st - 1) : (unsigned long long)min((long long)steps, (long long)(en - 1 - e));
    ev_sess[e] = (int)s;
    atomicAdd(&i_cnt[j], 1ull);
    if (w) atomicAdd(&work[j], w);
    tot += w;
  }
  for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
  if (lane == 0 && tot) atomicAdd(pairs, tot);
}

// the counting sort's placement: every event position into its item's list.  The order inside a list depends on the atomics; the
// fit only sums integers over it, so the rows do not.
__global__ void k_rules_place(const int* items, int64_t E, const int64_t* i_off, unsigned* i_fill, int* i_pos) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int j = items[e];
  i_pos[i_off[j] + atomicAdd(&i_fill[j], 1u)] = (int)e;
}

// one CTA per row from the work queue.  W(i, .) is accumulated in the CTA's dense uint64 slice (a column enters the touched list
// when its count leaves 0): SR spreads the row's occurrences over the threads, each adding inc[q - p] for the next `steps` events
// of its session; AR gives each warp an occurrence and its lanes the session's events, each adding 1.  Then w = W / L of every
// touched column (the slice cleared on the way) and the kept entries by bl_keep_row.
template <bool AR>
__global__ void __launch_bounds__(KF_THREADS) k_rules_fit(RulesFitDev d) {
  __shared__ int sRow, sT;
  unsigned long long* acc = d.acc + (size_t)blockIdx.x * d.n_items;
  int* tl = d.touched + (size_t)blockIdx.x * d.n_items;
  double* sv = d.w + (size_t)blockIdx.x * d.n_items;
  const int tid = threadIdx.x;
  for (;;) {
    if (tid == 0) { sRow = atomicAdd(d.next, 1); sT = 0; }
    __syncthreads();
    if (sRow >= d.n_items) break;
    const int i = d.order[sRow];
    const int64_t o0 = d.i_off[i], o1 = d.i_off[i + 1];
    if (AR) {
      const int lane = tid & 31;
      for (int64_t o = o0 + (tid >> 5); o < o1; o += KF_THREADS / 32) {
        const int s = d.ev_sess[d.i_pos[o]];
        for (int64_t q = d.off[s] + lane; q < d.off[s + 1]; q += 32) {
          const int j = d.items[q];
          if (j != i && atomicAdd(&acc[j], 1ull) == 0ull) tl[atomicAdd(&sT, 1)] = j;
        }
      }
    } else {
      for (int64_t o = o0 + tid; o < o1; o += KF_THREADS) {
        const int p = d.i_pos[o];
        const long long end = min((long long)p + d.steps, (long long)d.off[d.ev_sess[p] + 1] - 1);
        for (long long q = p + 1; q <= end; q++) {
          const int j = d.items[q];
          if (j != i && atomicAdd(&acc[j], d.inc[q - p]) == 0ull) tl[atomicAdd(&sT, 1)] = j;
        }
      }
    }
    __syncthreads();
    const int T = sT;
    for (int t = tid; t < T; t += KF_THREADS) {
      const unsigned long long W = atomicExch(&acc[tl[t]], 0ull);
      sv[t] = __ddiv_rn(__ull2double_rn(W), d.L);
    }
    __syncthreads();
    bl_keep_row(sv, tl, T, d.n_keep, i, d.out_idx, d.out_sim, d.out_len);
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// C ABI (include/g4r.h)
// ---------------------------------------------------------------------------------------------------------------------------
extern "C" int g4r_bl_rules_fit(g4r_baselines* h, const int64_t* session_offsets, int64_t n_sessions, const int32_t* items, int64_t n_events,
                                int32_t steps, int32_t weighting, int64_t* pair_work, size_t* scratch_bytes, float* device_ms) {
  if (!h) return G4R_ERR_INVALID;
  if (h->kind != BL_SR && h->kind != BL_AR) FAIL(G4R_ERR_STATE, "g4r_bl_rules_fit: the handle is not an SR or AR");
  const bool ar = h->kind == BL_AR;
  if (!session_offsets || n_sessions < 0 || n_events < 0 || (n_events > 0 && !items))
    FAIL(G4R_ERR_INVALID, "g4r_bl_rules_fit: null or negative argument");
  if (ar ? (steps != 0 || weighting != 0) : (steps < 1 || steps > RULES_STEPS_MAX || weighting < 0 || weighting > 1))
    FAIL(G4R_ERR_INVALID, ar ? "g4r_bl_rules_fit: AR takes steps = 0 and weighting = 0"
                             : "g4r_bl_rules_fit: SR needs steps in 1 .. 20 and weighting 0 (div) or 1 (same)");
  if (n_sessions > INT32_MAX || n_events > INT32_MAX) FAIL(G4R_ERR_INVALID, "g4r_bl_rules_fit: more than 2^31 - 1 sessions or events");
  if (!bl_offsets_ok(session_offsets, n_sessions, n_events)) FAIL(G4R_ERR_INVALID, "g4r_bl_rules_fit: session offsets must rise from 0 to n_events");
  const int NI = h->n_items, K = h->n_keep;
  for (int64_t e = 0; e < n_events; e++) if (items[e] < 0 || items[e] >= NI) FAIL(G4R_ERR_INDEX, "g4r_bl_rules_fit: item index out of range");
  // L = lcm(1 .. steps) for 'div' (every L / d is an integer), else 1
  unsigned long long L = 1;
  if (!ar && weighting == 0)
    for (unsigned long long d = 2; d <= (unsigned long long)steps; d++) { unsigned long long a = L, b = d; while (b) { const unsigned long long t = a % b; a = b; b = t; } L = L / a * d; }
  // the per-row bound of W: SR occ_i * min(steps, longest session - 1) * L, AR sum of n_s over i's occurrences; it must stay below 2^63
  int64_t max_len = 0;
  for (int64_t s = 0; s < n_sessions; s++) max_len = std::max(max_len, session_offsets[s + 1] - session_offsets[s]);
  std::vector<unsigned __int128> bound(NI, 0);
  const unsigned __int128 per = ar ? 0 : (unsigned __int128)std::min<int64_t>(steps, std::max<int64_t>(max_len - 1, 0)) * L;
  for (int64_t s = 0; s < n_sessions; s++)
    for (int64_t e = session_offsets[s]; e < session_offsets[s + 1]; e++)
      bound[items[e]] += ar ? (unsigned __int128)(session_offsets[s + 1] - session_offsets[s]) : per;
  for (int i = 0; i < NI; i++)
    if (bound[i] >= ((unsigned __int128)1 << 63)) FAIL(G4R_ERR_INVALID, "g4r_bl_rules_fit: a row's weight bound reaches 2^63 (uint64 counts could overflow)");
  const int grid = bl_fit_grid(h, sizeof(unsigned long long), scratch_bytes);
  const int64_t S = n_sessions, E = n_events;
  const unsigned gs = (unsigned)((S + 7) / 8), ge = (unsigned)((E + 255) / 256);
  cudaSetDevice(h->device);
  cudaStream_t st = h->stream;
  BlBufs bb;
  RulesFitDev d{};
  const int* dItems = nullptr; const int64_t* dOff = nullptr;
  int *ev_sess, *i_pos, *order, *next;
  long long *i_off, *tot;
  unsigned long long *i_cnt, *work, *pairs;
  unsigned *i_fill, *bkt;
  CK(bb.put(&dItems, items, E, st));
  CK(bb.put(&dOff, session_offsets, S + 1, st));
  CK(bb.take(&ev_sess, E)); CK(bb.take(&i_pos, E));
  CK(bb.take(&i_cnt, NI)); CK(bb.take(&work, NI)); CK(bb.take(&pairs, 1)); CK(bb.take(&i_off, NI + 1)); CK(bb.take(&tot, (NI + SCAN_B - 1) / SCAN_B));
  CK(bb.take(&i_fill, NI)); CK(bb.take(&bkt, 65)); CK(bb.take(&order, NI)); CK(bb.take(&next, 1));
  CK(bb.take(&d.acc, (size_t)NI * grid));
  CK(bb.take(&d.touched, (size_t)NI * grid));
  CK(bb.take(&d.w, (size_t)NI * grid));
  CK(cudaMemsetAsync(i_cnt, 0, NI * sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(work, 0, NI * sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(pairs, 0, sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(i_fill, 0, NI * sizeof(unsigned), st));
  CK(cudaMemsetAsync(bkt, 0, 65 * sizeof(unsigned), st));
  CK(cudaMemsetAsync(next, 0, sizeof(int), st));
  CK(cudaMemsetAsync(d.acc, 0, (size_t)NI * grid * sizeof(unsigned long long), st));
  h->ready = false;
  // everything from here to ev1 runs on the device without a host round trip: the occurrence lists, the row order, the fit and
  // the rows by index
  CK(cudaEventRecord(h->ev0, st));
  if (S > 0) {
    if (ar) k_rules_events<true><<<gs, 256, 0, st>>>(dOff, S, dItems, steps, ev_sess, i_cnt, work, pairs);
    else k_rules_events<false><<<gs, 256, 0, st>>>(dOff, S, dItems, steps, ev_sess, i_cnt, work, pairs);
  }
  CK(bl_scan((const long long*)i_cnt, NI, i_off, tot, st));
  if (E > 0) k_rules_place<<<ge, 256, 0, st>>>(dItems, E, (const int64_t*)i_off, i_fill, i_pos);
  bl_row_order(work, NI, bkt, order, st);
  d.off = dOff; d.items = dItems; d.ev_sess = ev_sess; d.i_off = (const int64_t*)i_off; d.i_pos = i_pos;
  d.order = order; d.next = next; d.n_items = NI; d.n_keep = K; d.steps = steps; d.L = (double)L;
  for (int q = 1; q <= RULES_STEPS_MAX; q++) d.inc[q] = (!ar && weighting == 0) ? L / (unsigned long long)q : 1ull;
  d.out_idx = h->dIdx; d.out_sim = h->dSim; d.out_len = h->dLen;
  if (ar) k_rules_fit<true><<<grid, KF_THREADS, 0, st>>>(d);
  else k_rules_fit<false><<<grid, KF_THREADS, 0, st>>>(d);
  return bl_fit_end(h, pairs, pair_work, device_ms);
}
