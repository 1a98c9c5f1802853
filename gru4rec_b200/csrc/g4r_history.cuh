// g4r_history.cuh -- evaluation from each session's history (DESIGN §3h): g4r_eval_schedule / g4r_eval_events on a schedule of
// g4r_schedule_build_history.  Each session there is its history events followed by its test events, walked by the unchanged
// evaluation schedule; only the lanes whose target is a test event (flag bit 2) are counted.  Included at the end of g4r_eval.cuh.
//
// One pass over the concatenated sessions, so every lane, step and tiebreaking key is that of the plain evaluation of the
// concatenated data:
//   forward  every step runs eval_forward (and, with exclude_seen, the seen-list insert of every lane) on the forward stream
//   enqueue  right after the forward of step i, on the same stream, its counted lanes are copied into a ranking block in (step,
//            lane) order: the final-layer y row, the target, the (step, lane) pair the tiebreaking noise hashes and, with
//            exclude_seen, a snapshot of the lane's seen list and miss flag (the live list keeps growing after the event).  The
//            positions come from the schedule on the host: no atomics, a deterministic order
//   rank     a block is ranked on the ranking stream when it holds the schedule's batch size of rows, and at the end of each
//            staging window, through a scoring descriptor of its own (y = the block's rows, wY = its targets, wSlot = identity,
//            so the block's row r reads snapshot r).  It is a RankUnit of eval_rank, the sequence that ranks a plain mini-batch,
//            with per-row noise keys (the KEY instances), its snapshots as the seen lists, and each row's schedule step and lane
//            for g4r_eval_events' per-event work.  A step with no counted lane ranks nothing.
// Two blocks alternate: the forward stream fills one while the ranking stream ranks the other, and waits only when it comes back to
// a block whose ranking has not finished.
#pragma once

struct HistBlock {
  int slot = -1;                                          // scoring descriptor: layer[last].y = dY, wY = dT, wM = dM, wSlot = dIdent
  float* dY = nullptr;                                    // [Be x ldL] final-layer y rows
  int* dT = nullptr;                                      // [Be] targets
  int* dKey = nullptr;                                    // [Be x 2] (window step, lane) of every row
  int* dM = nullptr;                                      // rows
  int* dSeen = nullptr; size_t seen_cap = 0;              // exclude_seen: [Be x cap] snapshots of the rows' seen lists
  int* dSeenN = nullptr;                                  //   [Be] their lengths
  int* dMiss = nullptr;                                   //   [Be] the rows' miss flags
  cudaEvent_t filled = nullptr, done = nullptr;           // enqueued (forward stream) / ranked (ranking stream)
  std::vector<int64_t> step; std::vector<int> lane;       // host: schedule step and lane of every row
};

struct HistCtx {
  HistBlock q[2];
  int* dIdent = nullptr;                                  // 0 .. Be - 1
  int* hLanes = nullptr; int* dLanes = nullptr;           // [cap x Be] counted lanes of the window's steps, step after step
  std::vector<int> off;                                   // [w + 1] offsets of the steps in hLanes
};

// frees whatever of c exists (also a context whose creation failed half way)
static void hist_free(HistCtx* p) {
  HistCtx& c = *p;
  for (HistBlock& q : c.q) {
    for (void* p : {(void*)q.dY, (void*)q.dT, (void*)q.dKey, (void*)q.dM, (void*)q.dSeen, (void*)q.dSeenN, (void*)q.dMiss}) if (p) cudaFree(p);
    if (q.filled) cudaEventDestroy(q.filled);
    if (q.done) cudaEventDestroy(q.done);
    slot_free(q.slot);
  }
  if (c.dIdent) cudaFree(c.dIdent);
  if (c.dLanes) cudaFree(c.dLanes);
  if (c.hLanes) cudaFreeHost(c.hLanes);
  delete p;
}

static void hist_release(EvalCtx& e) {
  if (!e.hist) return;
  hist_free(static_cast<HistCtx*>(e.hist));
  e.hist = nullptr;
}

// exclude_seen on a history schedule: lane b of step s adds its input to its slot's list and flags whether its target is in it
// (k_eval_tgt<true>'s insertion, without the target score)
__global__ void __launch_bounds__(128) k_hist_seen(int slot, int s, SeenDev sd) {
  const ModelDev& md = MD;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= md.wM[s]) return;
  sd.miss[b] = seen_insert(md, sd, s, b, md.wY[(size_t)s * md.B + b]) ? 1 : 0;
}

// the n counted lanes lanes[0 .. n) of step s (descriptor `slot`) into rows q0 .. q0 + n - 1 of a ranking block, one CTA per
// lane; *qm = q0 + n.  With sd.list: the lane's seen list, its length and miss flag as they are after step s's insertion
__global__ void __launch_bounds__(128) k_hist_enqueue(int slot, int s, const int* __restrict__ lanes, int n, int q0, float* __restrict__ qy,
                                                      int* __restrict__ qt, int* __restrict__ qkey, int* __restrict__ qm, SeenDev sd,
                                                      int* __restrict__ qseen, int* __restrict__ qseen_n, int* __restrict__ qmiss) {
  const ModelDev& md = MD;
  const int j = blockIdx.x, r = q0 + j, b = lanes[j], tid = threadIdx.x;
  const size_t o = (size_t)s * md.B + b;
  const float* y = md.layer[md.n_layers - 1].y + (size_t)b * md.ldL;
  for (int c4 = tid; c4 < md.ldL / 4; c4 += blockDim.x) st4(qy + (size_t)r * md.ldL + 4 * c4, ld4(y + 4 * c4));
  if (tid == 0) {
    qt[r] = md.wY[o]; qkey[2 * r] = s; qkey[2 * r + 1] = b;
    if (j == 0) *qm = q0 + n;
  }
  if (sd.list) {
    const int sl = md.wSlot[o], ns = sd.n[sl];
    const int* l = sd.list + (size_t)sl * sd.cap;
    for (int c = tid; c < ns; c += blockDim.x) qseen[(size_t)r * sd.cap + c] = l[c];
    if (tid == 0) { qseen_n[r] = ns; qmiss[r] = sd.miss[b]; }
  }
}

// the slots, buffers and events of a new context c: the two descriptor slots first, then the device memory
static int hist_create(g4r_handle* h, EvalCtx* e, HistCtx& c) {
  const int Be = e->Be, ldL = h->md.ldL;
  for (HistBlock& q : c.q) {
    q.slot = slot_alloc();
    if (q.slot < 0) FAIL(G4R_ERR_STATE, "too many live g4r handles in this process");
  }
  CK(cudaMalloc(&c.dIdent, (size_t)Be * sizeof(int)));
  std::vector<int> id((size_t)Be);
  for (int b = 0; b < Be; b++) id[(size_t)b] = b;
  CK(cudaMemcpy(c.dIdent, id.data(), (size_t)Be * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMallocHost(&c.hLanes, (size_t)e->cap * Be * sizeof(int)));
  CK(cudaMalloc(&c.dLanes, (size_t)e->cap * Be * sizeof(int)));
  for (HistBlock& q : c.q) {
    CK(cudaMalloc(&q.dY, (size_t)Be * ldL * sizeof(float)));
    CK(cudaMalloc(&q.dT, (size_t)Be * sizeof(int)));
    CK(cudaMalloc(&q.dKey, (size_t)Be * 2 * sizeof(int)));
    CK(cudaMalloc(&q.dM, sizeof(int)));
    CK(cudaEventCreateWithFlags(&q.filled, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&q.done, cudaEventDisableTiming));
    ModelDev md = e->mde;
    md.layer[md.n_layers - 1].y = q.dY;
    md.wY = q.dT; md.wM = q.dM; md.wSlot = c.dIdent;
    CK(slot_upload(q.slot, md, h->stream));
  }
  return G4R_OK;
}

// the handle's context (made on first use and kept only if complete), with snapshot room for blocks of the schedule's batch size
static int hist_begin(g4r_handle* h, EvalCtx* e, const g4r_schedule* s, const SeenDev* sd, HistCtx** out) {
  const int Be = e->Be, Bs = s->B;
  if (!e->hist) {
    HistCtx* c = new HistCtx();
    const int rc = hist_create(h, e, *c);
    if (rc) { hist_free(c); return rc; }
    e->hist = c;
  }
  HistCtx* c = static_cast<HistCtx*>(e->hist);
  for (HistBlock& q : c->q) {
    q.step.clear(); q.lane.clear();
    if (sd) {                  // a block holds at most Bs rows
      CK(dev_grow(&q.dSeen, &q.seen_cap, (size_t)Bs * sd->cap));
      if (!q.dSeenN) CK(cudaMalloc(&q.dSeenN, (size_t)Be * sizeof(int)));
      if (!q.dMiss) CK(cudaMalloc(&q.dMiss, (size_t)Be * sizeof(int)));
    }
  }
  *out = c;
  return G4R_OK;
}

// the counted lanes of the staged window (w steps of e->hX .. hF) to the device, on the forward stream
static int hist_stage(g4r_handle* h, EvalCtx* e, HistCtx* c, int64_t w) {
  const int Be = e->Be;
  c->off.assign((size_t)w + 1, 0);
  int n = 0;
  for (int64_t i = 0; i < w; i++) {
    for (int b = 0; b < e->hM[i]; b++) if (e->hF[i * Be + b] & 4) c->hLanes[n++] = b;
    c->off[(size_t)i + 1] = n;
  }
  if (n) CK(cudaMemcpyAsync(c->dLanes, c->hLanes, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  return G4R_OK;
}

// the w staged steps of a history schedule (first schedule step `done`): forward, seen insert and enqueue on the forward stream,
// every full block and the window's last partial block ranked on the ranking stream
static int hist_window(g4r_handle* h, EvalCtx* e, HistCtx* c, const g4r_schedule* s, int64_t w, int64_t done, const RankConsts& cs, EventsRun* ev) {
  const int Bs = s->B;
  cudaStream_t st = h->stream, rk = h->side;
  const SeenDev* sd = cs.seen ? &cs.sd : nullptr;
  int rc = hist_stage(h, e, c, w);
  if (rc) return rc;
  // block q, its M rows enqueued on the forward stream, ranked against its snapshots on the ranking stream
  auto rank = [&](HistBlock& q, int M) -> int {
    CK(cudaEventRecord(q.filled, st)); CK(cudaStreamWaitEvent(rk, q.filled, 0));
    RankUnit u;
    u.slot = q.slot; u.M = M; u.y = q.dY; u.key = q.dKey;
    if (sd) u.sd = SeenDev{q.dSeen, q.dSeenN, sd->cap, q.dMiss};
    u.steps = q.step.data(); u.lanes = q.lane.data();
    int r = eval_rank(h, e, u, cs, ev, rk, nullptr);
    if (r) return r;
    CK(cudaEventRecord(q.done, rk));
    CK(cudaGetLastError());
    q.step.clear(); q.lane.clear();
    return G4R_OK;
  };
  int qi = 0, qn = 0;
  for (int64_t i = 0; i < w; i++) {
    eval_forward(h, e, (int)i, h->He);
    if (sd) {
      k_hist_seen<<<(e->Be + 127) / 128, 128, 0, st>>>(e->slot, (int)i, *sd);
      h->launches++;
    }
    const int n = c->off[(size_t)i + 1] - c->off[(size_t)i];
    for (int p = 0; p < n;) {
      HistBlock& q = c->q[qi];
      if (qn == 0) CK(cudaStreamWaitEvent(st, q.done, 0));     // its last ranking has read it
      const int take = std::min(n - p, Bs - qn);
      const int l0 = c->off[(size_t)i] + p;
      k_hist_enqueue<<<take, 128, 0, st>>>(e->slot, (int)i, c->dLanes + l0, take, qn, q.dY, q.dT, q.dKey, q.dM, sd ? *sd : SeenDev{},
                                          q.dSeen, q.dSeenN, q.dMiss);
      h->launches++;
      for (int j = 0; j < take; j++) { q.step.push_back(done + i); q.lane.push_back(c->hLanes[l0 + j]); }
      qn += take; p += take;
      if (qn == Bs) {
        rc = rank(q, qn);
        if (rc) return rc;
        qi ^= 1; qn = 0;
      }
    }
  }
  if (qn > 0) {
    rc = rank(c->q[qi], qn);
    if (rc) return rc;
  }
  CK(cudaGetLastError());
  return G4R_OK;
}
