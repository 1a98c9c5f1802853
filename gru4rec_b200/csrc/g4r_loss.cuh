// g4r_loss.cuh -- the loss rule of every training kernel (gru4rec.py:200-248): which columns a loss weights by their softmax,
// the per-column summands of a row's statistics, how partial statistics merge, the final row statistics RS[b], the label
// smoothing terms and dL/do of one element.  Kernels keep their own loads, stores, thread mapping and accumulation order and
// call these for the arithmetic.  Included by g4r_kernels.cuh once ModelDev is defined.
//
// Row statistics of lane b: m (row max), Z (sum-exp), A, Q, D (loss-specific sums), T (target score), and for the pairwise
// losses t (target activation); RS[b] = {m, Z, A', Q', D', t or target score, loss_b, 0}.
#pragma once

__device__ __forceinline__ bool loss_xe(int loss) { return loss == G4R_LOSS_XE || loss == G4R_LOSS_XE_LOGIT; }
__device__ __forceinline__ bool loss_pairwise(int loss) { return loss == G4R_LOSS_BPR_MAX || loss == G4R_LOSS_TOP1_MAX || loss == G4R_LOSS_BPR || loss == G4R_LOSS_TOP1; }
__device__ __forceinline__ bool loss_softmaxneg(int loss) { return loss == G4R_LOSS_BPR_MAX || loss == G4R_LOSS_TOP1_MAX; }
// the row statistics are softmax-weighted sums relative to the row max (every loss but BPR and TOP1, whose sums are plain)
__device__ __forceinline__ bool loss_weighted(int loss) { return !(loss == G4R_LOSS_BPR || loss == G4R_LOSS_TOP1); }

// the summands of one score column of a row: y is the column's value (loss_xe: the score, otherwise its activation), t the
// target's activation.  Calls add(wt, A, Q, D) once: wt says A, Q, D are weighted by the column's softmax weight exp(y - m),
// which also adds to Z and the row max; otherwise they are plain sums.  add runs inside the loss's branch, so a product in a
// summand and the caller's sum are one expression, as when each kernel wrote the summands out.
template <class F>
__device__ __forceinline__ void loss_terms(int loss, float y, bool is_t, float t, F&& add) {
  if (loss_xe(loss)) {
    add(true, 0.f, 0.f, 0.f);
  } else if (loss == G4R_LOSS_BPR_MAX) {
    if (is_t) add(false, 0.f, 0.f, 0.f);
    else { const float sg = sigmoidf_(t - y); add(true, sg, y * y, sg * (1.f - sg)); }
  } else if (loss == G4R_LOSS_TOP1_MAX) {
    if (is_t) add(false, 0.f, 0.f, 0.f);
    else { const float a1 = sigmoidf_(y - t), b1 = sigmoidf_(y * y); add(true, a1 + b1, 0.f, a1 * (1.f - a1)); }
  } else if (loss == G4R_LOSS_BPR) {
    const float sg = sigmoidf_(t - y);
    if (is_t) add(false, -logf(sg), 0.f, 0.f);
    else add(false, -logf(sg), 0.f, 1.f - sg);
  } else {  // TOP1
    const float a1 = sigmoidf_(y - t), b1 = sigmoidf_(y * y);
    if (is_t) add(false, a1 + b1, 0.f, 0.f);
    else add(false, a1 + b1, 0.f, a1 * (1.f - a1));
  }
}

// merge (m,Z,A,Q,D) of two partial softmax-weighted sums
__device__ __forceinline__ void stat_merge(float& m, float& Z, float& A, float& Q, float& D, float m2, float Z2, float A2, float Q2, float D2) {
  const float mn = fmaxf(m, m2);
  const float e1 = (m == -INFINITY) ? 0.f : expf(m - mn), e2 = (m2 == -INFINITY) ? 0.f : expf(m2 - mn);
  Z = Z * e1 + Z2 * e2; A = A * e1 + A2 * e2; Q = Q * e1 + Q2 * e2; D = D * e1 + D2 * e2; m = mn;
}

// accumulate one score column into a row's running statistics (online softmax-style merge)
__device__ __forceinline__ void stat_add_elem(const ModelDev& md, float o, bool is_t, float t, float& m, float& Z, float& A, float& Q, float& D, float& T, float& has) {
  const bool xe = loss_xe(md.loss);
  const float y = xe ? o : act_fwd(md.fact, o);
  if (is_t) { has = 1.f; if (xe) T = o; }
  loss_terms(md.loss, y, is_t, t, [&](bool wt, float a, float q, float d) {
    if (wt) stat_merge(m, Z, A, Q, D, y, 1.f, a, q, d);
    else { A += a; D += d; }
  });
}
__device__ __forceinline__ void stat_combine(const ModelDev& md, float& m, float& Z, float& A, float& Q, float& D, float& T, float& has,
                                             float m2, float Z2, float A2, float Q2, float D2, float T2, float has2) {
  if (!loss_weighted(md.loss)) { A += A2; D += D2; }
  else stat_merge(m, Z, A, Q, D, m2, Z2, A2, Q2, D2);
  if (has2 > 0.f) { T = T2; has = 1.f; }
}

// final row statistics RS[b] from the merged sums (gru4rec.py:225-248): all eight slots, the ones a loss does not use as 0
__device__ __forceinline__ void stats_finalize(const ModelDev& md, int b, int M, int N, float m, float Z, float A, float Q, float D, float T, float tt) {
  float loss = 0.f, r2 = 0.f, r3 = 0.f, r4 = 0.f, r5 = tt;
  if (md.loss == G4R_LOSS_XE) { const float pt = __fdiv_rn(expf(T - m), Z); loss = -logf(pt + G4R_EPS_LOG); r2 = pt; r5 = T; }
  else if (md.loss == G4R_LOSS_XE_LOGIT) { loss = logf(Z) - (T - m); r5 = T; }
  else if (md.loss == G4R_LOSS_BPR_MAX) { r2 = __fdiv_rn(A, Z); r3 = __fdiv_rn(Q, Z); r4 = __fdiv_rn(D, Z); loss = -logf(r2 + G4R_EPS_LOG) + md.bpreg * r3; }
  else if (md.loss == G4R_LOSS_TOP1_MAX) { r2 = __fdiv_rn(A, Z); r4 = __fdiv_rn(D, Z); loss = r2; }
  else if (md.loss == G4R_LOSS_BPR) { loss = A; r4 = D; }
  else {  // TOP1 (gru4rec.py:242-244): mean over the N columns, last term over M + n_sample; the reference subtracts a
    // COLUMN from the row-mean vector, which broadcasts to [M x M] before the sum: everything is M times the row expression
    const float c = sigmoidf_(tt * tt);
    loss = (float)M * (__fdiv_rn(A, (float)N) - __fdiv_rn(c, (float)(M + md.S_cfg)));
    r4 = D;
  }
  float* rs = md.RS + (size_t)b * G4R_NSTAT;
  st4(rs, make_float4(m, Z, r2, r3));
  st4(rs + 4, make_float4(r4, r5, loss, 0.f));
}

// label smoothing (gru4rec.py:226-228, 232-234): loss_i = c1 * l(target) + c2 * sum_j l(j), n_out = M + n_sample
__device__ __forceinline__ void smooth_coefs(const ModelDev& md, int M, float& c1, float& c2) {
  const float n_out = (float)(M + md.S_cfg);
  c1 = 1.0f - __fdiv_rn(n_out, n_out - 1.0f) * md.smoothing;
  c2 = __fdiv_rn(md.smoothing, n_out - 1.0f);
}
// one column's terms given the row's final m, Z: l(j) into s1 (-log(p_j + eps) for softmax outputs, the log-softmax itself for
// xe_logit) and, for xe, p_j / (p_j + eps) into f
__device__ __forceinline__ void smooth_add_elem(int loss, float o, float m, float Z, float& s1, float& f) {
  if (loss == G4R_LOSS_XE) { const float p = __fdiv_rn(expf(o - m), Z); s1 += -logf(p + G4R_EPS_LOG); f += __fdiv_rn(p, p + G4R_EPS_LOG); }
  else s1 += logf(Z) - (o - m);
}
// the smoothed loss of a row from its statistics rs and s1 = sum_j l(j)
__device__ __forceinline__ float smooth_loss(const ModelDev& md, int M, const float* rs, float s1) {
  float c1, c2;
  smooth_coefs(md, M, c1, c2);
  if (md.loss == G4R_LOSS_XE) return c1 * (-logf(rs[2] + G4R_EPS_LOG)) + c2 * s1;
  return c1 * (logf(rs[1]) - (rs[5] - rs[0])) + c2 * s1;
}

// dL/do for element (b, column j) given final row statistics (already divided by batch_size)
__device__ __forceinline__ float loss_grad_elem(const ModelDev& md, const float* rs, float o, bool is_t, int M, int N) {
  const float invB = __fdiv_rn(1.0f, (float)md.B);
  if (md.smoothing > 0.f && loss_xe(md.loss)) {
    float c1, c2;
    smooth_coefs(md, M, c1, c2);
    const float p = __fdiv_rn(expf(o - rs[0]), rs[1]);
    if (md.loss == G4R_LOSS_XE) {
      const float f = __fdiv_rn(p, p + G4R_EPS_LOG), ft = __fdiv_rn(rs[2], rs[2] + G4R_EPS_LOG);
      return (-c2 * f - (is_t ? c1 * ft : 0.f) + p * (c2 * rs[3] + c1 * ft)) * invB;       // rs[3] = sum_j p_j / (p_j + eps)
    }
    return (-(c2 + (is_t ? c1 : 0.f)) + p * (c2 * (float)N + c1)) * invB;
  }
  if (md.loss == G4R_LOSS_XE) {
    const float p = __fdiv_rn(expf(o - rs[0]), rs[1]);
    const float fac = __fdiv_rn(rs[2], rs[2] + G4R_EPS_LOG);
    return fac * (p - (is_t ? 1.f : 0.f)) * invB;
  }
  if (md.loss == G4R_LOSS_XE_LOGIT) {
    const float p = __fdiv_rn(expf(o - rs[0]), rs[1]);
    return (p - (is_t ? 1.f : 0.f)) * invB;
  }
  const float y = act_fwd(md.fact, o);
  const float fd = act_der(md.fact, o, y);
  const float t = rs[5];
  float dy;
  if (md.loss == G4R_LOSS_BPR_MAX) {
    const float Ap = rs[2], Qp = rs[3], Dp = rs[4];
    const float invA = __fdiv_rn(1.0f, Ap + G4R_EPS_LOG);
    if (is_t) dy = -invA * Dp;
    else {
      const float sj = __fdiv_rn(expf(y - rs[0]), rs[1]);
      const float sg = sigmoidf_(t - y);
      const float dLds = -invA * sg + md.bpreg * y * y;
      const float mean = -invA * Ap + md.bpreg * Qp;
      dy = sj * (dLds - mean) + invA * sj * sg * (1.f - sg) + 2.f * md.bpreg * y * sj;
    }
  } else if (md.loss == G4R_LOSS_TOP1_MAX) {
    const float Ap = rs[2], Dp = rs[4];
    if (is_t) dy = -Dp;
    else {
      const float sj = __fdiv_rn(expf(y - rs[0]), rs[1]);
      const float a1 = sigmoidf_(y - t), b1 = sigmoidf_(y * y);
      dy = sj * ((a1 + b1) - Ap) + sj * a1 * (1.f - a1) + sj * b1 * (1.f - b1) * 2.f * y;
    }
  } else if (md.loss == G4R_LOSS_BPR) {
    if (is_t) dy = -rs[4];
    else dy = 1.f - sigmoidf_(t - y);
  } else {  // TOP1 (M times the row expression, see stats_finalize)
    const float invN = __fdiv_rn(1.0f, (float)N);
    if (is_t) {
      const float c = sigmoidf_(t * t);
      dy = -rs[4] * invN + c * (1.f - c) * 2.f * t * invN - __fdiv_rn(c * (1.f - c) * 2.f * t, (float)(M + md.S_cfg));
    } else {
      const float a1 = sigmoidf_(y - t), b1 = sigmoidf_(y * y);
      dy = (a1 * (1.f - a1) + b1 * (1.f - b1) * 2.f * y) * invN;
    }
    dy *= (float)M;
  }
  return dy * fd * invB;
}
