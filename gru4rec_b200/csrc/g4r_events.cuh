// g4r_events.cuh -- g4r_eval_events (DESIGN §3f): the evaluation schedule of g4r_eval_schedule with per-event outputs, the
// (#greater, #equal) counts of every event and optionally its top-k list.  Included at the end of g4r_eval.cuh (uses eval_run,
// the top-k context and kernels of g4r_topk.cuh).
//
// The unit of this work is the RankUnit that eval_rank ranks: a mini-batch, or a ranking block of a history schedule
// (g4r_history.cuh).  Everything runs on the ranking stream inside eval_rank, around the kernels g4r_eval_schedule launches for
// the same unit, so the Recall / MRR sums are those of g4r_eval_schedule and the forward of mini-batch i+1 still overlaps the
// ranking of i:
//   stage   right after the target scores: the unit's y rows are copied to the top-k descriptor's own buffer (read by the
//           unchanged top-k kernels through a descriptor slot of their own) and to the window's y buffer
//   counts  after k_eval_rank: the rows' counts into the window's per-event buffer
//   top-k   topk_rank's pipeline (topk_tiles, topk_select) with the window's survivor counters; the lists go straight into the
//           window's per-event lists.  A lane whose survivors overflowed keeps its softmax normaliser and is redone at the end
//           of the window
//   flush   one read of the window's survivor counters; every overflowed lane is rescored over the whole catalogue in fp32 from
//           the saved y (k_topk_rows / k_topk_final, in chunks of rows), then the window's outputs go to the host
// exclude_seen (g4r_seen.cuh): the unit's seen lists, gathered into the CSR exclusions the top-k kernels read (k_seen_csr), with a
// prefix of at least k + cap items; an overflowed row's seen set at its own schedule step and lane, which the unit gives for
// every row (the lists have moved on by the flush), is rebuilt from the schedule on the host
// The per-event window (w units, bounded by the size of its buffers) is separate from eval_run's staging window: eval_run stages
// the schedule in windows of e->cap mini-batches exactly as g4r_eval_schedule does, so every kernel of the evaluation sees the
// same step index (the tiebreaking noise hashes it), and the per-event buffers are flushed every w units within it and at its end.
#pragma once

constexpr size_t EVENTS_WINDOW_BYTES = (size_t)256 << 20;   // per-window buffers (y rows, counters, lists): shorter windows, not more
constexpr size_t EVENTS_ROWS_BYTES = (size_t)256 << 20;     // fp32 catalogue rows of one chunk of overflowed lanes

struct EventsCtx {
  int slot = -1;                                          // the scoring descriptor with the last layer's y at dYk and wM at dMk
  float* dYk = nullptr;                                   // [Be x ldL] y of the mini-batch the top-k kernels rank
  int* dMk = nullptr;                                     // its number of lanes
  int* dIdent = nullptr;                                  // 0 .. Be - 1
  int max_window = 0;                                     // G4R_EVENTS_WINDOW at creation (> 0: windows of at most that many mini-batches)
  float* dYw = nullptr; size_t yw_cap = 0;                // [w x Be x ldL] y rows of the window's mini-batches
  int* dSurvN = nullptr; size_t survn_cap = 0;            // [w x Be] survivors appended per (mini-batch, lane)
  float2* dNorm = nullptr; size_t norm_cap = 0;           // [w x Be] softmax normaliser (max, sum) of overflowed lanes
  int* dCnt = nullptr; size_t cnt_cap = 0;                // [window events x 2] (#greater, #equal)
  int* dItems = nullptr; size_t items_cap = 0;            // [window events x k] lists
  float* dScores = nullptr; size_t scores_cap = 0;
  int* dOvSrc = nullptr; size_t ov_src_cap = 0;           // a chunk of overflowed lanes: window row (mini-batch * Be + lane)
  int* dOvEv = nullptr; size_t ov_ev_cap = 0;             //   and window event
  float2* dOvNorm = nullptr; size_t ov_norm_cap = 0;      //   their normalisers
  int* dOvItems = nullptr; size_t ov_items_cap = 0;       //   their lists
  float* dOvScores = nullptr; size_t ov_scores_cap = 0;
  int* dOvExOff = nullptr; size_t ov_ex_off_cap = 0;      //   their exclusions (exclude_seen)
  int* dOvEx = nullptr; size_t ov_ex_cap = 0;
};

// one g4r_eval_events call
struct EventsRun {
  int32_t k = 0;
  int32_t* out_counts = nullptr; int32_t* out_items = nullptr; float* out_scores = nullptr;   // host [n_events x 2] / [n_events x k]
  EventsCtx* x = nullptr;
  TopkPlan plan;                                          // k > 0: the top-k constants, for units of up to the schedule's lanes
  int w = 0;                                              // units per per-event window
  int n = 0;                                              // units in the window so far
  int64_t ev_done = 0;                                    // events of the flushed windows
  int64_t win_ev = 0;                                     // events of the window so far
  std::vector<int64_t> off;                               // window event of row 0 of every unit of the window
  std::vector<int> survn;                                 // host copy of dSurvN
  const g4r_schedule* sched = nullptr;
  bool seen = false;                                      // exclude_seen: the lists exclude ex_off / ex (k_seen_csr's output)
  const int* ex_off = nullptr; const int* ex = nullptr;
  std::vector<int> m;                                     // rows of every unit of the window
  std::vector<int64_t> rstep; std::vector<int> rlane;     // exclude_seen lists: [w x Be] schedule step and lane of every row
};
static bool events_lists(const EventsRun* ev) { return ev->k > 0; }

static void events_release(EvalCtx& e) {
  if (!e.events) return;
  EventsCtx& x = *static_cast<EventsCtx*>(e.events);
  for (void* p : {(void*)x.dYk, (void*)x.dMk, (void*)x.dIdent, (void*)x.dYw, (void*)x.dSurvN, (void*)x.dNorm, (void*)x.dCnt,
                  (void*)x.dItems, (void*)x.dScores, (void*)x.dOvSrc, (void*)x.dOvEv, (void*)x.dOvNorm, (void*)x.dOvItems, (void*)x.dOvScores,
                  (void*)x.dOvExOff, (void*)x.dOvEx})
    if (p) cudaFree(p);
  slot_free(x.slot);
  delete static_cast<EventsCtx*>(e.events);
  e.events = nullptr;
}

// y rows b < M of step s (the scoring descriptor's last layer) into yk and yw; *mk = M
__global__ void __launch_bounds__(256) k_ev_stage(int slot, int s, float* __restrict__ yk, float* __restrict__ yw, int* mk) {
  const ModelDev& md = MD;
  const int M = md.wM[s];
  const float* y = md.layer[md.n_layers - 1].y;
  if (blockIdx.x == 0 && threadIdx.x == 0) *mk = M;
  const int n4 = M * md.ldL / 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    const float4 v = ld4(y + 4 * i);
    st4(yk + 4 * i, v); st4(yw + 4 * i, v);
  }
}

// the (#greater, #equal) pairs of the M lanes of step s; SEEN: (-1, -1) for a lane flagged in miss
template <bool SEEN = false>
__global__ void __launch_bounds__(256) k_ev_counts(int slot, int s, const int* __restrict__ cnt, int* __restrict__ out, const int* __restrict__ miss = nullptr) {
  const ModelDev& md = MD;
  const int n = 2 * md.wM[s];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = (SEEN && miss[i >> 1]) ? -1 : cnt[i];
}

// softmax normaliser (max, sum) of every lane whose survivors overflowed, reduced from the tile partials exactly as k_topk_final
// reduces them (same block size, same order)
__global__ void __launch_bounds__(TOPK_THREADS) k_ev_norm(const int* __restrict__ cnt, int C, const float2* __restrict__ part, int n_part, float2* norm) {
  const int b = blockIdx.x, tid = threadIdx.x;
  if (cnt[b] <= C) return;
  __shared__ float redf[TOPK_THREADS / 32];
  __shared__ double redd[TOPK_THREADS / 32];
  const float2* pr = part + (size_t)b * n_part;
  float m = -INFINITY;
  for (int j = tid; j < n_part; j += blockDim.x) m = fmaxf(m, pr[j].x);
  m = warp_max(m);
  if ((tid & 31) == 0) redf[tid >> 5] = m;
  __syncthreads();
  m = redf[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); w++) m = fmaxf(m, redf[w]);
  double zz = 0.0;
  for (int j = tid; j < n_part; j += blockDim.x) {
    const float2 p = pr[j];
    if (p.x != -INFINITY) zz += (double)p.y * exp((double)p.x - (double)m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) zz += __shfl_xor_sync(0xffffffffu, zz, o);
  if ((tid & 31) == 0) redd[tid >> 5] = zz;
  __syncthreads();
  zz = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) zz += redd[w];
  if (tid == 0) norm[b] = make_float2(m, (float)zz);
}

// a chunk of n overflowed lanes: their saved y rows yw[src[j]] into yk (*mk = n) and their normalisers; k_topk_final reads a
// normaliser as one partial (max, sum), which gives back exactly that pair
__global__ void __launch_bounds__(256) k_ev_gather(const float* __restrict__ yw, const int* __restrict__ src, int n, int ldL, float* __restrict__ yk,
                                                   int* mk, const float2* __restrict__ norm, float2* __restrict__ onorm) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *mk = n;
  const int kw = ldL / 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * kw; i += gridDim.x * blockDim.x) {
    const int r = i / kw, c4 = i % kw;
    st4(yk + (size_t)r * ldL + 4 * c4, ld4(yw + (size_t)src[r] * ldL + 4 * c4));
  }
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) onorm[j] = norm[src[j]];
}

// the lists of a chunk (row j) to their window events ev[j]
__global__ void __launch_bounds__(256) k_ev_scatter(const int* __restrict__ items, const float* __restrict__ scores, const int* __restrict__ ev, int n, int k,
                                                    int* __restrict__ out_items, float* __restrict__ out_scores) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * k; i += gridDim.x * blockDim.x) {
    const size_t o = (size_t)ev[i / k] * k + i % k;
    out_items[o] = items[i]; out_scores[o] = scores[i];
  }
}

// appends to ex the seen set of lane b at schedule step g (its session's inputs up to and including that step: the lane's slot is
// followed back through the steps until its zero-before flag or the schedule's start), sorted and distinct
static void seen_rebuild(const g4r_schedule* s, int64_t g, int b, std::vector<int>& ex) {
  const int B = s->B, sl = s->slots[(size_t)(g * B + b)];
  const size_t e0 = ex.size();
  for (int64_t t = g; t >= 0; t--) {
    if (t < g) {                 // the lane that held the slot at step t (tail compaction moves lanes, never slots)
      int lb = -1;
      for (int c = 0; c < s->M[(size_t)t]; c++) if (s->slots[(size_t)(t * B + c)] == sl) { lb = c; break; }
      if (lb < 0) break;
      b = lb;
    }
    ex.push_back(s->X[(size_t)(t * B + b)]);
    if (s->F[(size_t)(t * B + b)] & 2) break;
  }
  std::sort(ex.begin() + e0, ex.end());
  ex.erase(std::unique(ex.begin() + e0, ex.end()), ex.end());
}

static int events_ctx(g4r_handle* h, EvalCtx* e, EventsCtx** out) {
  if (!e->events) {
    const int slot = slot_alloc();
    if (slot < 0) FAIL(G4R_ERR_STATE, "too many live g4r handles in this process");
    e->events = new EventsCtx();
    EventsCtx& x = *static_cast<EventsCtx*>(e->events);
    x.slot = slot;
    const int Be = e->Be;
    CK(cudaMalloc(&x.dYk, (size_t)Be * h->md.ldL * sizeof(float)));
    CK(cudaMalloc(&x.dMk, sizeof(int)));
    CK(cudaMalloc(&x.dIdent, (size_t)Be * sizeof(int)));
    std::vector<int> id((size_t)Be);
    for (int b = 0; b < Be; b++) id[(size_t)b] = b;
    CK(cudaMemcpy(x.dIdent, id.data(), (size_t)Be * sizeof(int), cudaMemcpyHostToDevice));
    ModelDev md = e->mde;
    md.layer[md.n_layers - 1].y = x.dYk;
    md.wM = x.dMk;
    CK(slot_upload(x.slot, md, h->stream));
    const char* w = getenv("G4R_EVENTS_WINDOW");
    x.max_window = w ? std::max(0, atoi(w)) : 0;
  }
  *out = static_cast<EventsCtx*>(e->events);
  return G4R_OK;
}

// checks k, sizes the per-event window and its buffers, prepares the top-k operands
static int events_begin(g4r_handle* h, EvalCtx* e, const g4r_schedule* s, EventsRun* ev, const SeenDev* sd) {
  const int Be = e->Be, ldL = h->md.ldL, k = ev->k;
  ev->sched = s;
  ev->seen = sd != nullptr;
  ev->ex_off = sd ? e->dSeenOff : nullptr; ev->ex = sd ? e->dSeenEx : nullptr;
  TopkFilter f;
  if (k > 0) {
    int rc = topk_filter(h, k, e->n_cand > 0 ? e->hCand.data() : nullptr, e->n_cand, &f);
    if (rc) return rc;
  }
  int rc = events_ctx(h, e, &ev->x);
  if (rc) return rc;
  EventsCtx* x = ev->x;
  const size_t per_step = (size_t)Be * (2 * sizeof(int) + (k > 0 ? ldL * sizeof(float) + sizeof(int) + sizeof(float2) + (size_t)k * (sizeof(int) + sizeof(float)) : 0));
  int64_t w = std::min<int64_t>(e->cap, std::max<int64_t>(1, (int64_t)(EVENTS_WINDOW_BYTES / per_step)));
  if (x->max_window > 0) w = std::min<int64_t>(w, x->max_window);
  ev->w = (int)w;
  ev->off.assign((size_t)w, 0);
  ev->m.assign((size_t)w, 0);
  CK(dev_grow(&x->dCnt, &x->cnt_cap, (size_t)w * Be * 2));
  if (k == 0) return G4R_OK;
  if (sd) { ev->rstep.assign((size_t)w * Be, 0); ev->rlane.assign((size_t)w * Be, 0); }
  rc = topk_plan(h, e, f, k, sd ? sd->cap : 0, s->B, &ev->plan);   // exclude_seen: at most cap exclusions per lane
  if (rc) return rc;
  CK(dev_grow(&x->dYw, &x->yw_cap, (size_t)w * Be * ldL));
  CK(dev_grow(&x->dSurvN, &x->survn_cap, (size_t)w * Be));
  CK(dev_grow(&x->dNorm, &x->norm_cap, (size_t)w * Be));
  CK(dev_grow(&x->dItems, &x->items_cap, (size_t)w * Be * k));
  CK(dev_grow(&x->dScores, &x->scores_cap, (size_t)w * Be * k));
  ev->survn.assign((size_t)w * Be, 0);
  return G4R_OK;
}

// unit u, right after its target scores: its events' place in the per-event window (unit j of it), its rows' schedule step and
// lane (for the seen sets of the flush), and its y rows saved for the top-k
static int events_stage(g4r_handle* h, EvalCtx* e, EventsRun* ev, const RankUnit& u, cudaStream_t rk) {
  EventsCtx* x = ev->x;
  const TopkPlan& p = ev->plan;
  if (ev->n == 0) {
    ev->win_ev = 0;
    if (ev->k > 0 && !p.no_tile) CK(cudaMemsetAsync(x->dSurvN, 0, ev->survn.size() * sizeof(int), rk));
  }
  const int j = ev->n++, M = u.M, Be = e->Be;
  ev->off[(size_t)j] = ev->win_ev;
  ev->m[(size_t)j] = M;
  ev->win_ev += M;
  if (!ev->rstep.empty())
    for (int b = 0; b < M; b++) {
      ev->rstep[(size_t)j * Be + b] = u.steps ? u.steps[b] : u.step;
      ev->rlane[(size_t)j * Be + b] = u.lanes ? u.lanes[b] : b;
    }
  if (ev->k > 0) {
    const size_t rows = (size_t)Be * h->md.ldL;
    k_ev_stage<<<std::min<int>((int)((rows / 4 + 255) / 256), 2 * h->n_sm), 256, 0, rk>>>(u.slot, u.s, x->dYk, x->dYw + (size_t)j * rows, x->dMk);
    h->launches++;
  }
  return G4R_OK;
}

// the lists of unit j of the per-event window (M rows, window events o ..) by topk_rank's pipeline on the staged y rows; a lane
// whose survivors overflowed keeps its softmax normaliser, selects from its truncated list here and is redone by the flush
static int events_topk(g4r_handle* h, EvalCtx* e, EventsRun* ev, int M, int j, int64_t o, cudaStream_t rk) {
  EventsCtx* x = ev->x;
  const TopkPlan& p = ev->plan;
  const int Be = e->Be, k = ev->k;
  int* cnt = x->dSurvN + (size_t)j * Be;
  const int n_part = topk_tiles(h, e, p, x->slot, x->dYk, M, cnt, ev->ex_off, ev->ex, rk);
  if (!p.no_tile && h->md.fact.kind > G4R_ACT_SELU) {
    k_ev_norm<<<M, TOPK_THREADS, 0, rk>>>(cnt, p.C, p.t->dPart, n_part, x->dNorm + (size_t)j * Be);
    h->launches++;
  }
  topk_select(h, p, x->slot, M, p.no_tile ? nullptr : cnt, nullptr, nullptr, p.t->dPart, n_part, x->dItems + o * k, x->dScores + o * k, ev->ex_off, ev->ex, rk);
  CK(cudaGetLastError());
  return G4R_OK;
}

// unit u after k_eval_rank: its counts and lists; a full per-event window is flushed
static int events_step(g4r_handle* h, EvalCtx* e, EventsRun* ev, const RankUnit& u, cudaStream_t rk) {
  EventsCtx* x = ev->x;
  const int Be = e->Be, j = ev->n - 1;
  const int64_t o = ev->off[(size_t)j];
  if (ev->seen) k_ev_counts<true><<<(2 * Be + 255) / 256, 256, 0, rk>>>(u.slot, u.s, h->dRankCnt, x->dCnt + 2 * o, u.sd.miss);
  else k_ev_counts<<<(2 * Be + 255) / 256, 256, 0, rk>>>(u.slot, u.s, h->dRankCnt, x->dCnt + 2 * o);
  h->launches++;
  if (ev->k > 0) {
    int rc = events_topk(h, e, ev, u.M, j, o, rk);
    if (rc) return rc;
  }
  return ev->n == ev->w ? events_flush(h, e, ev, rk) : G4R_OK;
}

// end of a per-event window (its ev->n units): the overflowed lanes rescored exactly, then the window's outputs to the host
static int events_flush(g4r_handle* h, EvalCtx* e, EventsRun* ev, cudaStream_t rk) {
  EventsCtx* x = ev->x;
  const int Be = e->Be, k = ev->k, I = h->md.n_items, w = ev->n;
  const int64_t E = ev->win_ev;
  if (w == 0) return G4R_OK;
  CK(cudaMemcpyAsync(ev->out_counts + 2 * ev->ev_done, x->dCnt, (size_t)E * 2 * sizeof(int), cudaMemcpyDeviceToHost, rk));
  if (k > 0) {
    const TopkPlan& p = ev->plan;
    if (!p.no_tile) {
      CK(cudaMemcpyAsync(ev->survn.data(), x->dSurvN, (size_t)w * Be * sizeof(int), cudaMemcpyDeviceToHost, rk));
      CK(cudaStreamSynchronize(rk));
      std::vector<int> src, evw;
      for (int64_t i = 0; i < w; i++)
        for (int b = 0; b < ev->m[(size_t)i]; b++)
          if (ev->survn[(size_t)(i * Be + b)] > p.C) { src.push_back((int)(i * Be + b)); evw.push_back((int)(ev->off[(size_t)i] + b)); }
      const int chunk = (int)std::min<int64_t>(Be, std::max<int64_t>(1, (int64_t)(EVENTS_ROWS_BYTES / ((size_t)I * sizeof(float)))));
      for (size_t j0 = 0; j0 < src.size(); j0 += (size_t)chunk) {
        const int n = (int)std::min<size_t>((size_t)chunk, src.size() - j0);
        CK(dev_grow(&e->dOut, &e->out_cap, (size_t)n * I));
        CK(dev_grow(&x->dOvSrc, &x->ov_src_cap, (size_t)chunk));
        CK(dev_grow(&x->dOvEv, &x->ov_ev_cap, (size_t)chunk));
        CK(dev_grow(&x->dOvNorm, &x->ov_norm_cap, (size_t)chunk));
        CK(dev_grow(&x->dOvItems, &x->ov_items_cap, (size_t)chunk * k));
        CK(dev_grow(&x->dOvScores, &x->ov_scores_cap, (size_t)chunk * k));
        CK(cudaMemcpyAsync(x->dOvSrc, src.data() + j0, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, rk));
        CK(cudaMemcpyAsync(x->dOvEv, evw.data() + j0, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, rk));
        if (ev->seen) {                        // the chunk's seen sets at their own steps, rebuilt from the schedule
          std::vector<int> eo(1, 0), ex;
          for (int j = 0; j < n; j++) {
            const size_t r = (size_t)src[j0 + (size_t)j];
            seen_rebuild(ev->sched, ev->rstep[r], ev->rlane[r], ex);
            eo.push_back((int)ex.size());
          }
          CK(dev_grow(&x->dOvExOff, &x->ov_ex_off_cap, eo.size()));
          CK(dev_grow(&x->dOvEx, &x->ov_ex_cap, std::max<size_t>(1, ex.size())));
          CK(cudaMemcpyAsync(x->dOvExOff, eo.data(), eo.size() * sizeof(int), cudaMemcpyHostToDevice, rk));
          if (!ex.empty()) CK(cudaMemcpyAsync(x->dOvEx, ex.data(), ex.size() * sizeof(int), cudaMemcpyHostToDevice, rk));
        }
        k_ev_gather<<<std::min(2 * h->n_sm, (n * h->md.ldL / 4 + 255) / 256 + 1), 256, 0, rk>>>(x->dYw, x->dOvSrc, n, h->md.ldL, x->dYk, x->dMk, x->dNorm, x->dOvNorm);
        k_topk_rows<<<dim3((I + 127) / 128, n), 128, 0, rk>>>(x->slot, x->dIdent, e->dOut);
        topk_select(h, p, x->slot, n, x->dIdent, x->dIdent, e->dOut, x->dOvNorm, 1, x->dOvItems, x->dOvScores,
                    ev->seen ? x->dOvExOff : nullptr, ev->seen ? x->dOvEx : nullptr, rk);
        k_ev_scatter<<<std::min(2 * h->n_sm, (n * k + 255) / 256), 256, 0, rk>>>(x->dOvItems, x->dOvScores, x->dOvEv, n, k, x->dItems, x->dScores);
        h->launches += 3;
        CK(cudaGetLastError());
      }
    }
    CK(cudaMemcpyAsync(ev->out_items + ev->ev_done * k, x->dItems, (size_t)E * k * sizeof(int), cudaMemcpyDeviceToHost, rk));
    CK(cudaMemcpyAsync(ev->out_scores + ev->ev_done * k, x->dScores, (size_t)E * k * sizeof(float), cudaMemcpyDeviceToHost, rk));
  }
  CK(cudaStreamSynchronize(rk));
  ev->ev_done += E;
  ev->n = 0;
  return G4R_OK;
}

extern "C" int g4r_eval_events(g4r_handle* h, const g4r_schedule* s, const int32_t* cut_off, int32_t n_cut, int32_t mode, int32_t k,
                               double* recall_sum, double* mrr_sum, int64_t* n_events, int32_t* out_counts, int32_t* out_items, float* out_scores) {
  if (!h || !s || !cut_off || n_cut <= 0 || n_cut > 64 || !recall_sum || !mrr_sum || !out_counts) return G4R_ERR_INVALID;
  if (k < 0) FAIL(G4R_ERR_INVALID, "k must be >= 0");
  if (k > 0 && (!out_items || !out_scores)) FAIL(G4R_ERR_INVALID, "out_items / out_scores are NULL with k > 0");
  EventsRun ev;
  ev.k = k; ev.out_counts = out_counts; ev.out_items = out_items; ev.out_scores = out_scores;
  return eval_run(h, s, cut_off, n_cut, mode, recall_sum, mrr_sum, n_events, &ev);
}
