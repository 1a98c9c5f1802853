// g4r_sessions.cuh -- the session store of the scoring path (g4r_sessions_*, DESIGN §3e).  Included at the end of g4r_eval.cuh
// (uses EvalCtx, eval_forward and the shared top-k ranking topk_rank of g4r_topk.cuh).
//
// An int64 session key maps to a slot: a row of a device table of `capacity` hidden-state rows per layer, separate from the
// scoring lanes He and from the training state.  The key map, the recency order and each session's input history live on the
// host.  A call stages its events into the scoring window exactly as an evaluation mini-batch (item, slot, flags per lane) with
// the table as the forward's state array, so the GRU forward and the ranking are the kernels g4r_predict_topk runs.
//   recency   a doubly linked list over the slots, least recently used first; every event that names a session moves it to the
//             end, in call order
//   eviction  a key not in the store takes a free slot, else the slot of the least recently used session that the current call
//             does not name (that session's state and history are dropped); its first step carries flag bit 2, so the row is
//             zeroed on the device as a fresh evaluation lane is, and needs no memset
//   rounds    (feed) the r-th events of all keys of a call form round r; the rounds, each cut into steps of at most Be lanes, run
//             as consecutive steps of one uploaded window, so no two lanes of a step share a slot
// Every argument is validated before a slot is assigned or anything reaches the device: after an error the store is unchanged.
#pragma once
#include <unordered_map>
#include <unordered_set>

struct SessStore {
  int64_t cap = 0;
  float* dTab = nullptr;                                   // layer li: rows [cap x ldL] at dTab + cap * (sum of ldL of layers < li)
  float* H[G4R_MAX_LAYERS] = {};
  std::unordered_map<int64_t, int> slot_of;
  std::vector<int64_t> key;                                // per slot
  std::vector<int> prev, next;                             // recency list over the live slots; head = least recently used
  int head = -1, tail = -1;
  std::vector<int> free_slots;                             // a stack, slot 0 on top when the store is empty
  std::vector<std::vector<int32_t>> hist;                  // per slot: the session's input items since it entered the store
  int64_t n_hist = 0;
  int* dSlots = nullptr; size_t slots_cap = 0;             // export / import: slots of the packed rows
  float* dPack = nullptr; size_t pack_cap = 0;             // and the rows, all layers concatenated without padding
};

static void sessions_release(g4r_handle* h) {
  if (!h->sessions) return;
  SessStore* s = static_cast<SessStore*>(h->sessions);
  if (s->dTab) cudaFree(s->dTab);
  if (s->dSlots) cudaFree(s->dSlots);
  if (s->dPack) cudaFree(s->dPack);
  delete s;
  h->sessions = nullptr;
}

static void sess_unlink(SessStore& s, int sl) {
  const int p = s.prev[sl], n = s.next[sl];
  if (p >= 0) s.next[p] = n; else s.head = n;
  if (n >= 0) s.prev[n] = p; else s.tail = p;
  s.prev[sl] = s.next[sl] = -1;
}
static void sess_push(SessStore& s, int sl) {              // as the most recently used
  s.prev[sl] = s.tail; s.next[sl] = -1;
  if (s.tail >= 0) s.next[s.tail] = sl; else s.head = sl;
  s.tail = sl;
}
static void sess_drop(SessStore& s, int sl) {              // the session leaves the store: state, history and slot released
  sess_unlink(s, sl);
  s.slot_of.erase(s.key[sl]);
  s.n_hist -= (int64_t)s.hist[sl].size();
  std::vector<int32_t>().swap(s.hist[sl]);
  s.free_slots.push_back(sl);
}
// the slot of `key`, used now; *fresh: the key was not in the store (its row holds no state).  in_call: the keys of the current
// call, never evicted by it (the caller has checked that they fit)
static int sess_use(SessStore& s, int64_t key, const std::unordered_set<int64_t>& in_call, bool* fresh) {
  auto it = s.slot_of.find(key);
  if (it != s.slot_of.end()) {
    sess_unlink(s, it->second); sess_push(s, it->second);
    *fresh = false;
    return it->second;
  }
  if (s.free_slots.empty()) {
    int v = s.head;
    while (in_call.count(s.key[v])) v = s.next[v];
    sess_drop(s, v);
  }
  const int sl = s.free_slots.back();
  s.free_slots.pop_back();
  s.key[sl] = key;
  s.slot_of.emplace(key, sl);
  sess_push(s, sl);
  *fresh = true;
  return sl;
}

static int sess_get(g4r_handle* h, SessStore** out) {
  if (!h) return G4R_ERR_INVALID;
  if (h->shard) FAIL(G4R_ERR_STATE, "session store: not available on a row-sharded multi-GPU handle");
  if (!h->sessions) FAIL(G4R_ERR_STATE, "session store: not opened (g4r_sessions_open)");
  *out = static_cast<SessStore*>(h->sessions);
  return G4R_OK;
}

// the distinct keys of a call into `set`; G4R_ERR_INVALID if there are more than the store holds, or (distinct) if a key repeats
static int sess_call_keys(g4r_handle* h, const SessStore& s, const int64_t* keys, int64_t n, bool distinct, std::unordered_set<int64_t>& set) {
  set.reserve((size_t)std::min<int64_t>(n, s.cap) + 1);
  for (int64_t i = 0; i < n; i++) {
    if (!set.insert(keys[i]).second && distinct) FAIL(G4R_ERR_INVALID, "a session key appears more than once in the call");
    if ((int64_t)set.size() > s.cap) FAIL(G4R_ERR_INVALID, "the call names more distinct sessions than the store's capacity");
  }
  return G4R_OK;
}

static int sess_check_items(g4r_handle* h, const int32_t* X, int64_t n) {
  for (int64_t i = 0; i < n; i++) if (X[i] < 0 || X[i] >= h->md.n_items) FAIL(G4R_ERR_INDEX, "Index out of bounds");
  return G4R_OK;
}

// step s of the window: lanes b < M take item X[ev[b]], slot slots[ev[b]], flag 2 if fresh[ev[b]]
static void sess_stage(EvalCtx* e, int s, const int32_t* X, const int* slots, const uint8_t* fresh, const int64_t* ev, int M) {
  const size_t o = (size_t)s * e->Be;
  for (int b = 0; b < e->Be; b++) {
    const bool live = b < M;
    e->hX[o + b] = live ? X[ev[b]] : -1; e->hY[o + b] = 0; e->hSlot[o + b] = live ? slots[ev[b]] : 0;
    e->hF[o + b] = live && fresh[ev[b]] ? 2 : 0;
  }
  e->hM[s] = M; e->hSti[s] = -1; e->hG[s] = 0;
}

extern "C" int g4r_sessions_open(g4r_handle* h, int64_t capacity) {
  if (!h) return G4R_ERR_INVALID;
  if (h->shard) FAIL(G4R_ERR_STATE, "session store: not available on a row-sharded multi-GPU handle");
  if (capacity < 1 || capacity > INT32_MAX) FAIL(G4R_ERR_INVALID, "session capacity must be in 1 .. 2^31 - 1");
  cudaSetDevice(h->cfg.device);
  CK(cudaStreamSynchronize(h->stream));
  sessions_release(h);
  size_t ld_sum = 0;
  for (int li = 0; li < h->md.n_layers; li++) ld_sum += (size_t)h->md.layer[li].ldL;
  SessStore* s = new SessStore();
  s->cap = capacity;
  const cudaError_t r = cudaMalloc(&s->dTab, (size_t)capacity * ld_sum * sizeof(float));
  if (r != cudaSuccess) { delete s; FAIL(G4R_ERR_CUDA, std::string("session table: ") + cudaGetErrorString(r)); }
  size_t off = 0;
  for (int li = 0; li < h->md.n_layers; li++) { s->H[li] = s->dTab + (size_t)capacity * off; off += (size_t)h->md.layer[li].ldL; }
  s->key.assign((size_t)capacity, 0);
  s->prev.assign((size_t)capacity, -1);
  s->next.assign((size_t)capacity, -1);
  s->hist.resize((size_t)capacity);
  s->free_slots.resize((size_t)capacity);
  for (int64_t i = 0; i < capacity; i++) s->free_slots[(size_t)i] = (int)(capacity - 1 - i);
  h->sessions = s;
  return G4R_OK;
}

extern "C" int64_t g4r_sessions_count(const g4r_handle* h, int64_t* n_history_items) {
  if (!h) return G4R_ERR_INVALID;
  const SessStore* s = static_cast<const SessStore*>(h->sessions);
  if (n_history_items) *n_history_items = s ? s->n_hist : 0;
  return s ? (int64_t)s->slot_of.size() : 0;
}

extern "C" int g4r_sessions_feed(g4r_handle* h, const int64_t* keys, const int32_t* X, int64_t n) {
  SessStore* s = nullptr;
  int rc = sess_get(h, &s);
  if (rc) return rc;
  if (n < 0 || (n > 0 && (!keys || !X))) FAIL(G4R_ERR_INVALID, "keys / X missing or n < 0");
  if (n == 0) return G4R_OK;
  rc = sess_check_items(h, X, n);
  if (rc) return rc;
  std::unordered_set<int64_t> in_call;
  rc = sess_call_keys(h, *s, keys, n, false, in_call);
  if (rc) return rc;
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  rc = eval_ctx(h, &e);
  if (rc) return rc;
  // slots in call order; the r-th event of a key goes to round r
  std::vector<int> slots((size_t)n), occ((size_t)n);
  std::vector<uint8_t> fresh((size_t)n);
  std::unordered_map<int64_t, int> seen;
  seen.reserve(in_call.size());
  int n_rounds = 0;
  for (int64_t i = 0; i < n; i++) {
    bool f;
    slots[(size_t)i] = sess_use(*s, keys[i], in_call, &f);
    fresh[(size_t)i] = f;
    occ[(size_t)i] = seen[keys[i]]++;
    n_rounds = std::max(n_rounds, occ[(size_t)i] + 1);
    s->hist[(size_t)slots[(size_t)i]].push_back(X[i]);
  }
  s->n_hist += n;
  std::vector<int64_t> order((size_t)n), start((size_t)n_rounds + 1, 0);   // events by round, call order within a round
  for (int64_t i = 0; i < n; i++) start[(size_t)occ[(size_t)i] + 1]++;
  for (int r = 0; r < n_rounds; r++) start[(size_t)r + 1] += start[(size_t)r];
  {
    std::vector<int64_t> pos(start.begin(), start.end() - 1);
    for (int64_t i = 0; i < n; i++) order[(size_t)pos[(size_t)occ[(size_t)i]]++] = i;
  }
  const int Be = e->Be;
  cudaStream_t st = h->stream;
  int w = 0;
  for (int r = 0; r < n_rounds; r++) {
    for (int64_t c0 = start[(size_t)r]; c0 < start[(size_t)r + 1]; c0 += Be) {
      const int M = (int)std::min<int64_t>(Be, start[(size_t)r + 1] - c0);
      sess_stage(e, w++, X, slots.data(), fresh.data(), order.data() + c0, M);
      const bool last = r == n_rounds - 1 && c0 + M == start[(size_t)r + 1];
      if (w == e->cap || last) {                           // a full window (or the call's last step): upload and run it
        rc = eval_upload(h, e, w);
        if (rc) return rc;
        for (int i = 0; i < w; i++) eval_forward(h, e, i, s->H);
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(st));                     // the staging buffers are reused
        w = 0;
      }
    }
  }
  return G4R_OK;
}

extern "C" int g4r_sessions_topk(g4r_handle* h, const int64_t* keys, const int32_t* X, int64_t n, int32_t k,
                                 const int32_t* cand, int64_t n_cand, const int64_t* excl_off, const int32_t* excl_items,
                                 int32_t exclude_seen, int32_t* out_items, float* out_scores) {
  SessStore* s = nullptr;
  int rc = sess_get(h, &s);
  if (rc) return rc;
  if (n < 0 || (n > 0 && (!keys || !X || !out_items || !out_scores))) FAIL(G4R_ERR_INVALID, "keys / X / outputs missing or n < 0");
  TopkFilter f;
  rc = topk_filter(h, k, cand, n_cand, &f);
  if (rc) return rc;
  if (n == 0) return G4R_OK;
  rc = sess_check_items(h, X, n);
  if (rc) return rc;
  if (excl_off) {
    rc = topk_check_excl(h, n, excl_off, excl_items);
    if (rc) return rc;
  }
  std::unordered_set<int64_t> in_call;
  rc = sess_call_keys(h, *s, keys, n, true, in_call);
  if (rc) return rc;
  cudaSetDevice(h->cfg.device);
  EvalCtx* e = nullptr;
  rc = eval_ctx(h, &e);
  if (rc) return rc;
  std::vector<int> slots((size_t)n);
  std::vector<uint8_t> fresh((size_t)n);
  for (int64_t i = 0; i < n; i++) {
    bool fr;
    slots[(size_t)i] = sess_use(*s, keys[i], in_call, &fr);
    fresh[(size_t)i] = fr;
    s->hist[(size_t)slots[(size_t)i]].push_back(X[i]);
  }
  s->n_hist += n;
  // chunks of at most Be lanes, each staged at step 0 and ranked by the top-k of g4r_predict_topk_filtered
  const int Be = e->Be;
  std::vector<int64_t> ev((size_t)Be);
  std::vector<int> ex_off, ex;
  for (int64_t c0 = 0; c0 < n; c0 += Be) {
    const int M = (int)std::min<int64_t>(Be, n - c0);
    for (int b = 0; b < M; b++) ev[(size_t)b] = c0 + b;
    sess_stage(e, 0, X, slots.data(), fresh.data(), ev.data(), M);
    rc = eval_upload(h, e, 1);
    if (rc) return rc;
    ex_off.clear(); ex.clear();
    if (excl_off || exclude_seen) {
      ex_off.push_back(0);
      for (int b = 0; b < M; b++) {
        const int64_t i = c0 + b;
        const size_t e0 = ex.size();
        if (excl_off) topk_add_excl(f, excl_items + excl_off[i], excl_off[i + 1] - excl_off[i], ex);
        if (exclude_seen) { const std::vector<int32_t>& hs = s->hist[(size_t)slots[(size_t)i]]; topk_add_excl(f, hs.data(), (int64_t)hs.size(), ex); }
        rc = topk_close_lane(h, ex_off, ex, e0);
        if (rc) return rc;
      }
    }
    rc = topk_rank(h, e, s->H, M, k, f, ex_off, ex, out_items + c0 * k, out_scores + c0 * k);
    if (rc) return rc;
  }
  return G4R_OK;
}

extern "C" int g4r_sessions_end(g4r_handle* h, const int64_t* keys, int64_t n) {
  SessStore* s = nullptr;
  int rc = sess_get(h, &s);
  if (rc) return rc;
  if (!keys) {
    while (s->head >= 0) sess_drop(*s, s->head);
    for (int64_t i = 0; i < s->cap; i++) s->free_slots[(size_t)i] = (int)(s->cap - 1 - i);   // the order of a new store
    return G4R_OK;
  }
  if (n < 0) FAIL(G4R_ERR_INVALID, "n < 0");
  for (int64_t i = 0; i < n; i++) {
    auto it = s->slot_of.find(keys[i]);
    if (it != s->slot_of.end()) sess_drop(*s, it->second);
  }
  return G4R_OK;
}

// packed row i (all layers, sum of L floats) <-> table row slots[i]; to_table: 1 scatter, 0 gather
struct SessRows { float* H[G4R_MAX_LAYERS]; int L[G4R_MAX_LAYERS], ld[G4R_MAX_LAYERS], n_layers, Lsum; };
__global__ void __launch_bounds__(256) k_sess_rows(SessRows r, const int* __restrict__ slots, int64_t n, float* packed, int to_table) {
  const int64_t total = n * r.Lsum;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / r.Lsum;
    int c = (int)(i % r.Lsum), li = 0;
    while (c >= r.L[li]) c -= r.L[li++];
    float* t = r.H[li] + (size_t)slots[row] * r.ld[li] + c;
    if (to_table) *t = packed[i]; else packed[i] = *t;
  }
}
static int sess_rows(g4r_handle* h, SessStore* s, const std::vector<int>& slots, float* host, int to_table) {
  SessRows r;
  r.n_layers = h->md.n_layers; r.Lsum = 0;
  for (int li = 0; li < r.n_layers; li++) { r.H[li] = s->H[li]; r.L[li] = h->md.layer[li].L; r.ld[li] = h->md.layer[li].ldL; r.Lsum += r.L[li]; }
  const int64_t n = (int64_t)slots.size();
  if (n == 0) return G4R_OK;
  cudaStream_t st = h->stream;
  const size_t nf = (size_t)n * r.Lsum;
  CK(dev_grow(&s->dSlots, &s->slots_cap, slots.size()));
  CK(dev_grow(&s->dPack, &s->pack_cap, nf));
  CK(cudaMemcpyAsync(s->dSlots, slots.data(), slots.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  if (to_table) CK(cudaMemcpyAsync(s->dPack, host, nf * sizeof(float), cudaMemcpyHostToDevice, st));
  k_sess_rows<<<(int)std::min<int64_t>((int64_t)(nf + 255) / 256, 4 * h->n_sm), 256, 0, st>>>(r, s->dSlots, n, s->dPack, to_table);
  h->launches++;
  CK(cudaGetLastError());
  if (!to_table) CK(cudaMemcpyAsync(host, s->dPack, nf * sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return G4R_OK;
}

extern "C" int g4r_sessions_export(g4r_handle* h, int64_t* keys, float* states, int64_t* hist_off, int32_t* hist_items) {
  SessStore* s = nullptr;
  int rc = sess_get(h, &s);
  if (rc) return rc;
  std::vector<int> slots;
  slots.reserve(s->slot_of.size());
  for (int sl = s->head; sl >= 0; sl = s->next[sl]) slots.push_back(sl);
  int64_t o = 0;
  for (size_t i = 0; i < slots.size(); i++) {
    const std::vector<int32_t>& hs = s->hist[(size_t)slots[i]];
    if (keys) keys[i] = s->key[(size_t)slots[i]];
    if (hist_off) hist_off[i] = o;
    if (hist_items) std::copy(hs.begin(), hs.end(), hist_items + o);
    o += (int64_t)hs.size();
  }
  if (hist_off) hist_off[slots.size()] = o;
  if (!states) return G4R_OK;
  cudaSetDevice(h->cfg.device);
  return sess_rows(h, s, slots, states, 0);
}

extern "C" int g4r_sessions_import(g4r_handle* h, const int64_t* keys, const float* states, const int64_t* hist_off,
                                   const int32_t* hist_items, int64_t n) {
  SessStore* s = nullptr;
  int rc = sess_get(h, &s);
  if (rc) return rc;
  if (n < 0 || (n > 0 && (!keys || !states))) FAIL(G4R_ERR_INVALID, "keys / states missing or n < 0");
  if (n == 0) return G4R_OK;
  if (hist_off) {
    if (hist_off[0] != 0) FAIL(G4R_ERR_INVALID, "hist_off[0] must be 0");
    for (int64_t i = 0; i < n; i++) if (hist_off[i + 1] < hist_off[i]) FAIL(G4R_ERR_INVALID, "hist_off must be non-decreasing");
    if (hist_off[n] > 0 && !hist_items) FAIL(G4R_ERR_INVALID, "hist_items is NULL");
    rc = sess_check_items(h, hist_items, hist_off[n]);
    if (rc) return rc;
  }
  std::unordered_set<int64_t> in_call;
  rc = sess_call_keys(h, *s, keys, n, true, in_call);
  if (rc) return rc;
  cudaSetDevice(h->cfg.device);
  std::vector<int> slots((size_t)n);
  for (int64_t i = 0; i < n; i++) {
    bool fr;
    const int sl = sess_use(*s, keys[i], in_call, &fr);
    slots[(size_t)i] = sl;
    std::vector<int32_t>& hs = s->hist[(size_t)sl];
    s->n_hist -= (int64_t)hs.size();
    hs.clear();
    if (hist_off) hs.assign(hist_items + hist_off[i], hist_items + hist_off[i + 1]);
    s->n_hist += (int64_t)hs.size();
  }
  return sess_rows(h, s, slots, const_cast<float*>(states), 1);
}
