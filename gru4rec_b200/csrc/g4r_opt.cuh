// g4r_opt.cuh -- the parameter update rule of every training kernel: the adaptive scalers (gru4rec.py:300-381) and the
// dense / sparse update that follows (gru4rec.py:390-431).  Kernels keep their own loads, stores and thread mapping and call
// these for the arithmetic.  Included by g4r_kernels.cuh once ModelDev is defined.
//
// Every multiply, add and subtract is written as __fmul_rn / __fadd_rn / __fsub_rn, which the compiler never contracts
// into an FMA.  The results therefore do not depend on the register allocation of the kernel the update is inlined into,
// and equal what a build with contraction off (-fmad=false) computes.
#pragma once

#define G4R_EPS_ADA 1e-6f

__device__ __forceinline__ float grad_scale(const ModelDev& md) { return md.gscale ? *md.gscale : 1.0f; }

// Adagrad (gru4rec.py:335-340): accumulator a = a0 + g^2; returns the scaled gradient g / sqrt(a + eps)
__device__ __forceinline__ float ada_step(float a0, float g, float& a) {
  a = __fadd_rn(a0, __fmul_rn(g, g));
  return __fdiv_rn(g, sqrtf(__fadd_rn(a, G4R_EPS_ADA)));
}
// one member of a sparse element's duplicate group (gru4rec.py:407-431): the L2 term reads p0 and the velocity starts from v0,
// the element's values before the step; p accumulates the members' steps
__device__ __forceinline__ void sparse_step(const ModelDev& md, bool mom, float gs, float p0, float v0, float& p, float& v) {
  const float d = md.lmbd > 0.f ? __fmul_rn(md.lr, __fadd_rn(gs, __fmul_rn(md.lmbd, p0))) : __fmul_rn(md.lr, gs);
  if (mom) { v = __fsub_rn(__fmul_rn(md.mom, v0), d); p = __fadd_rn(p, v); }
  else p = __fsub_rn(p, d);
}
// dense element (gru4rec.py:390-406)
__device__ __forceinline__ void dense_step(const ModelDev& md, bool mom, float gs, float& p, float& v) {
  if (mom) { v = __fsub_rn(__fmul_rn(md.mom, v), __fmul_rn(md.lr, __fadd_rn(gs, __fmul_rn(md.lmbd, p)))); p = __fadd_rn(p, v); }
  else p = __fsub_rn(__fmul_rn(p, __fsub_rn(1.0f, __fmul_rn(md.lr, md.lmbd))), __fmul_rn(md.lr, gs));
}
// SGD / Adagrad (+momentum) update of one dense element in memory; a / v are only touched with ada / mom
__device__ __forceinline__ void dense_elem(const ModelDev& md, bool ada, bool mom, float g, float* p, float* a, float* v) {
  const float gs = ada ? ada_step(*a, g, *a) : g;
  float pv = *p, vv = mom ? *v : 0.f;
  dense_step(md, mom, gs, pv, vv);
  *p = pv;
  if (mom) *v = vv;
}

// SGD / Adagrad (+momentum) update of one sparse element (float) or 16-byte quad (float4) by a duplicate group, members
// added in position order: every member is scaled with the group's initial accumulator; acc / velocity keep the LAST
// member's values (set_subtensor), the parameter accumulates all members (inc_subtensor).  begin(p, pl2, a, v): pl2 is the
// operand of the L2 term, the row itself except for phase_sparse_in's shared mode.  add(g): kernels that run with grad_cap
// pass g already multiplied by grad_scale(md).
__device__ __forceinline__ void chain_add(const ModelDev& md, bool ada, bool mom, float g, float p0, float a0, float v0, float& al, float& vl, float& ps) {
  const float gs = ada ? ada_step(a0, g, al) : g;
  sparse_step(md, mom, gs, p0, v0, ps, vl);
}
template <class T>
struct RowChain {
  T p0, a0, v0, al, vl, ps;
  __device__ __forceinline__ void begin(T p, T pl2, T a, T v) { ps = p; p0 = pl2; a0 = a; v0 = v; al = a; vl = v; }
  __device__ __forceinline__ void add(const ModelDev& md, T g, bool ada, bool mom);
};
template <>
__device__ __forceinline__ void RowChain<float>::add(const ModelDev& md, float g, bool ada, bool mom) { chain_add(md, ada, mom, g, p0, a0, v0, al, vl, ps); }
template <>
__device__ __forceinline__ void RowChain<float4>::add(const ModelDev& md, float4 g, bool ada, bool mom) {
  chain_add(md, ada, mom, g.x, p0.x, a0.x, v0.x, al.x, vl.x, ps.x);
  chain_add(md, ada, mom, g.y, p0.y, a0.y, v0.y, al.y, vl.y, ps.y);
  chain_add(md, ada, mom, g.z, p0.z, a0.z, v0.z, al.z, vl.z, ps.z);
  chain_add(md, ada, mom, g.w, p0.w, a0.w, v0.w, al.w, vl.w, ps.w);
}

// ------------------------------------------------------------------------------------------------
// Adaptive scalers other than Adagrad (gru4rec.py:300-329 adam, 341-366 adadelta, 367-381 rmsprop) and the update that follows
// (gru4rec.py:390-431), for ONE element of a parameter with n gradient contributions in position order (n = 1: dense).
// Sparse ("sampled") parameters use the reference's duplicate-accurate forms: the decayed state receives the squared
// gradients of ALL duplicates, every duplicate is scaled with that common state (and adam's sparse first moment accumulates
// grad**2 -- sic, gru4rec.py:325); velocity: last duplicate wins; parameter: all duplicates accumulate.
// States of an element: s0 = acc, s1 = upd (adadelta) | meang (adam), s2 = countt (adam).  Only for adapt > G4R_ADAPT_ADAGRAD.
// ------------------------------------------------------------------------------------------------
struct OptE { float p, s0, s1, s2, v; };
template <bool SPARSE, class FG>
__device__ __forceinline__ void opt_elem(const ModelDev& md, OptE& e, float p0l, int n, FG gk) {
  const float gsc = grad_scale(md);
  const int ad = md.adapt;
  const bool mom = md.mom > 0.f;
  float sclr = 1.f, common = 0.f;
  if (ad == G4R_ADAPT_RMSPROP || ad == G4R_ADAPT_ADADELTA) {
    float A = __fmul_rn(e.s0, md.ap1);
    for (int k = 0; k < n; k++) { const float g = __fmul_rn(gk(k), gsc); A = __fadd_rn(A, __fmul_rn(__fmul_rn(md.ap1c, g), g)); }
    if (ad == G4R_ADAPT_ADADELTA) {
      sclr = __fdiv_rn(__fadd_rn(e.s1, G4R_EPS_ADA), __fadd_rn(A, G4R_EPS_ADA));
      float U = __fmul_rn(e.s1, md.ap1);
      for (int k = 0; k < n; k++) { const float g = __fmul_rn(gk(k), gsc); U = __fadd_rn(U, __fmul_rn(__fmul_rn(__fmul_rn(md.ap1c, sclr), g), g)); }
      e.s1 = U;
      sclr = sqrtf(sclr);
    } else sclr = __fdiv_rn(1.0f, sqrtf(__fadd_rn(A, G4R_EPS_ADA)));
    e.s0 = A;
  } else {                                  // adam
    float A = __fmul_rn(e.s0, md.ap2);
    float Mg = __fmul_rn(e.s1, md.ap1);
    for (int k = 0; k < n; k++) {
      const float g = __fmul_rn(gk(k), gsc);
      A = __fadd_rn(A, __fmul_rn(__fmul_rn(md.ap2c, g), g));
      Mg = __fadd_rn(Mg, __fmul_rn(md.ap1c, SPARSE ? __fmul_rn(g, g) : g));
    }
    const float ct = __fadd_rn(e.s2, 1.0f);
    const float bias = __fsub_rn(1.0f, powf(md.ap1, ct));
    common = __fdiv_rn(__fdiv_rn(Mg, bias), __fadd_rn(sqrtf(__fdiv_rn(A, bias)), G4R_EPS_ADA));
    e.s0 = A; e.s1 = Mg; e.s2 = ct;
  }
  const float v0 = e.v;
  float ps = e.p, vl = e.v;
  for (int k = 0; k < n; k++) {
    const float gs = ad == G4R_ADAPT_ADAM ? common : __fmul_rn(__fmul_rn(gk(k), gsc), sclr);
    if (SPARSE) sparse_step(md, mom, gs, p0l, v0, ps, vl);
    else dense_step(md, mom, gs, ps, vl);
  }
  e.p = ps; e.v = vl;
}
// number of adaptive state arrays per parameter (they sit one after the other, `stride` elements apart, behind `*.acc`)
__host__ __device__ inline int opt_states(int adapt) { return adapt == G4R_ADAPT_ADAM ? 3 : (adapt == G4R_ADAPT_ADADELTA ? 2 : (adapt == G4R_ADAPT_NONE ? 0 : 1)); }
// generic (any scaler) row update: one row of `ld` elements, n members, element-wise over the lanes of a warp / threads of a CTA
template <class FG>
__device__ __forceinline__ void opt_row_generic(const ModelDev& md, float* prow, float* arow, size_t ast, float* vrow, const float* p0row, int ld,
                                                int n, int t0, int tstep, bool write_state, FG grow /* (member k, column c) -> gradient */) {
  const int ns = opt_states(md.adapt);
  for (int c = t0; c < ld; c += tstep) {
    OptE e;
    e.p = prow[c];
    e.s0 = ns > 0 ? arow[c] : 0.f; e.s1 = ns > 1 ? arow[ast + c] : 0.f; e.s2 = ns > 2 ? arow[2 * ast + c] : 0.f;
    e.v = vrow ? vrow[c] : 0.f;
    opt_elem<true>(md, e, p0row ? p0row[c] : e.p, n, [&](int k) { return grow(k, c); });
    prow[c] = e.p;
    if (write_state) {
      if (ns > 0) arow[c] = e.s0;
      if (ns > 1) arow[ast + c] = e.s1;
      if (ns > 2) arow[2 * ast + c] = e.s2;
      if (vrow) vrow[c] = e.v;
    }
  }
}
