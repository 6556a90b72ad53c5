// Per-element functions of the in-batch pairwise ranking losses (the reference's losses/pairwise.py), shared by the
// forward statistics kernel and the two backward kernels (inbatch_flash.cu, Pairwise<KIND>) so that they evaluate one
// formula.  The
// dq kernel recomputes the forward's scores bit for bit; the dn kernel's S^T = N Q^T may differ in the last bit, so an
// element within rounding of an eps0 / relu boundary can fall on the other side there (one element of c / T).
//
// s = a negative's score (already masked and divided by T), sp = the row's positive score, d = sp - s, u = s - sp.
// eps0(x) = where(x == 0, x + 1e-24, x) (utils/tf_utils.py add_epsilon_to_zeros): the `== 0` tests below run on float32
// values computed WITHOUT flush-to-zero (expf and the round-to-nearest reciprocal, no ex2.approx.ftz), because a
// subnormal weight is nonzero in the reference's float32 graph.
#pragma once
#include <cuda_runtime.h>

namespace mm {
namespace pw {

enum Kind { BPR = 0, BPR_MAX = 1, TOP1 = 2, TOP1_V2 = 3, TOP1_MAX = 4, LOGISTIC = 5, HINGE = 6, N_KINDS = 7 };

template <int K>
struct is_max {
  static constexpr bool value = K == BPR_MAX || K == TOP1_MAX;
};

constexpr float EPS0_LOSS = 55.262043f;  // -log(1e-24): the loss of an element whose eps0 argument is exactly 0

// sigmoid(x), sigmoid(-x), sigmoid'(x) and softplus(-|x|) from ONE exp and one reciprocal: e = exp(-|x|) (subnormal
// results kept, so sigmoid(-100) = e^-100 is nonzero as in float32), r = 1 / (1 + e).
struct Sig {
  float e, r;
  bool neg;
  __device__ __forceinline__ explicit Sig(float x) : e(expf(-fabsf(x))), neg(x < 0.0f) { r = __frcp_rn(1.0f + e); }
  __device__ __forceinline__ float pos() const { return neg ? e * r : r; }   // sigmoid(x)
  __device__ __forceinline__ float mirror() const { return neg ? r : e * r; }  // sigmoid(-x)
  __device__ __forceinline__ float deriv() const { return e * r * r; }        // sigmoid(x) sigmoid(-x)
  __device__ __forceinline__ float log1p_e() const { return log1pf(e); }      // softplus(x) - max(x, 0)
};
// sigmoid(v) and sigmoid'(v) of v = s^2 >= 0
struct SigSq {
  float e, r;
  __device__ __forceinline__ explicit SigSq(float v) : e(expf(-v)) { r = __frcp_rn(1.0f + e); }
};

// running sums of one row in the forward: the loss, dloss/dsp, and for BPR-max the count of elements off the eps0
// branch and sum s^2 w
struct RowAcc {
  float loss = 0.0f, gp = 0.0f, cnt = 0.0f, sq = 0.0f;
};

// adds element (s) of a row to its sums when `valid`; lse = the row's log-sum-exp over the negatives (-max kinds only)
template <int K>
__device__ __forceinline__ void fwd_elem(bool valid, float s, float sp, float lse, float lambda, RowAcc& a) {
  const float d = sp - s;
  float loss, gp, cnt = 0.0f, sq = 0.0f;
  if (K == BPR || K == LOGISTIC) {
    const Sig g(d);
    const float sp_ = fmaxf(-d, 0.0f) + g.log1p_e();  // softplus(-d) = -log(sigmoid(d))
    if (K == BPR) {
      const bool eps = g.pos() == 0.0f;                // its gradient is -1e24 * dsigmoid = 0
      loss = eps ? EPS0_LOSS : sp_;
      gp = eps ? 0.0f : -g.mirror();
    } else {  // relu(u) + log1p(eps0(exp(-|u|))): eps0 only moves log1p(0) to log1p(1e-24); TF's relu'(0) = sign(0) = 0
      loss = sp_;
      gp = d == 0.0f ? 0.0f : -g.mirror();
    }
  } else if (K == BPR_MAX) {
    const float w = expf(s - lse);
    const float s2w = s * s * w;
    const Sig g(d);
    const bool eps = g.pos() * w == 0.0f;
    sq = s2w;
    loss = (eps ? EPS0_LOSS : fmaxf(-d, 0.0f) + g.log1p_e() + (lse - s)) + lambda * s2w;  // -log(sigmoid(d) w)
    gp = eps ? 0.0f : -g.mirror();
    cnt = eps ? 0.0f : 1.0f;
  } else if (K == TOP1 || K == TOP1_V2 || K == TOP1_MAX) {
    const Sig g(-d);
    const SigSq q(s * s);
    const float w = K == TOP1_MAX ? expf(s - lse) : 1.0f;
    loss = (g.pos() + q.r) * w;
    gp = -g.deriv() * w;
  } else {  // HINGE
    const float m = 1.0f - d;
    loss = fmaxf(m, 0.0f);
    gp = m > 0.0f ? -1.0f : 0.0f;
  }
  if (valid) {
    a.loss += loss;
    a.gp += gp;
    if (K == BPR_MAX) {
      a.cnt += cnt;
      a.sq += sq;
    }
  }
}

// the row's terms outside the elements; returns the coefficient A the backward reads (-max kinds)
template <int K>
__device__ __forceinline__ float fwd_row(float sp, float lambda, RowAcc& a) {
  if (K == TOP1_V2) {  // - sigmoid(sp^2), the per-row term of top1_v2 (times N: the mean over the negatives is c's)
    const SigSq q(sp * sp);
    a.loss -= q.r;
    a.gp -= 2.0f * sp * q.e * q.r * q.r;
  }
  if (K == BPR_MAX) return a.cnt - lambda * a.sq;
  if (K == TOP1_MAX) return -a.loss;
  return 0.0f;
}

// dloss/ds of one unmasked element (the row's loss depends on s through this element and, for the -max kinds, through
// the soft-max weights of all elements; A carries the row's share of the latter)
template <int K>
__device__ __forceinline__ float bwd_elem(float s, float sp, float lse, float A, float lambda) {
  const float d = sp - s;
  if (K == BPR) {
    const Sig g(d);
    return g.pos() == 0.0f ? 0.0f : g.mirror();
  } else if (K == BPR_MAX) {
    const float w = expf(s - lse);
    const Sig g(d);
    const float sg = g.pos();
    return (sg * w == 0.0f ? 0.0f : -sg) + w * (A + lambda * (2.0f * s + s * s));
  } else if (K == TOP1 || K == TOP1_V2) {
    const Sig g(-d);
    const SigSq q(s * s);
    return g.deriv() + 2.0f * s * q.e * q.r * q.r;
  } else if (K == TOP1_MAX) {
    const float w = expf(s - lse);
    const Sig g(-d);
    const SigSq q(s * s);
    return w * (g.deriv() + 2.0f * s * q.e * q.r * q.r + g.pos() + q.r + A);
  } else if (K == LOGISTIC) {
    return d == 0.0f ? 0.0f : Sig(d).mirror();
  } else {
    return 1.0f - d > 0.0f ? 1.0f : 0.0f;
  }
}

}  // namespace pw
}  // namespace mm
