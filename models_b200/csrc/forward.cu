// Whole-op C entry points over fp32 Keras-layout weights: a caller that is not this package's Python host
// (the TF-side stub of INTEGRATION.md, a C++ server) runs an MLPBlock or a CrossBlock with ONE call and a
// caller-provided workspace — nothing is allocated here, no pre-split weights are needed.
//
//   mm_mlp_forward   : MLPBlock (merlin/models/tf/blocks/mlp.py:97-139, Dense :275-280)
//   mm_cross_forward : CrossBlock stack x_{l+1} = x0 * (x_l W_l + b_l) + x_l (blocks/cross.py:29-109, :188-202)
//
// Both split the fp32 operands to bf16 (hi, lo) pairs inside the workspace and run the wgmma kernels with the
// 3-pass fp32-grade accumulation; the MLP uses the whole-tower kernel (mm_mlp_tc) when the widths allow it and
// one mm_dense_tc launch per layer otherwise.
#include <cuda_bf16.h>

#include "mm_common.cuh"

namespace {

constexpr int64_t kAlign = 256;
inline int64_t align_up(int64_t v) { return (v + kAlign - 1) / kAlign * kAlign; }

struct MlpPlan {
  int64_t a_off, act_off[2], w_off[8], total;
  int64_t act_bytes;
};

bool plan_mlp(int64_t M, int K, int n_layers, const int* widths, MlpPlan& p) {
  if (n_layers < 1 || n_layers > 8) return false;
  int64_t off = 0;
  p.a_off = off;
  off += align_up(M * 2 * (int64_t)mm_tc_padded_k(K) * 2);
  int64_t act = 0;
  int k = K;
  for (int l = 0; l < n_layers; ++l) {
    p.w_off[l] = off;
    off += align_up((int64_t)mm_tc_padded_n(widths[l]) * 2 * mm_tc_padded_k(k) * 2);
    if (l + 1 < n_layers) {
      const int64_t b = M * 2 * (int64_t)mm_tc_padded_k(widths[l]) * 2;
      act = b > act ? b : act;
    }
    k = widths[l];
  }
  p.act_bytes = align_up(act);
  p.act_off[0] = off;
  off += p.act_bytes;
  p.act_off[1] = off;
  off += p.act_bytes;
  p.total = off;
  return true;
}

}  // namespace

extern "C" {

int64_t mm_mlp_workspace_bytes(int64_t M, int K, int n_layers, const int* widths) {
  if (M < 0 || K <= 0 || !widths) return -1;
  for (int l = 0; l < n_layers; ++l)
    if (widths[l] <= 0) return -1;
  MlpPlan p;
  return plan_mlp(M, K, n_layers, widths, p) ? p.total : -1;
}

int mm_mlp_forward(const float* x, int64_t M, int K, int64_t x_stride, int n_layers, const float* const* kernels,
                   const float* const* biases, const int* widths, const int* acts, float* out, int64_t out_stride,
                   void* workspace, int64_t workspace_bytes, void* stream) {
  MM_REQUIRE(x && kernels && biases && widths && acts && out && M >= 0 && K > 0 && x_stride >= K, MM_ERR_ARG,
             "mm_mlp_forward: null pointer or bad M/K/stride");
  MM_REQUIRE(n_layers >= 1 && n_layers <= 8, MM_ERR_UNSUPPORTED, "mm_mlp_forward: 1..8 layers (got %d)", n_layers);
  for (int l = 0; l < n_layers; ++l) {
    MM_REQUIRE(kernels[l] && widths[l] > 0, MM_ERR_ARG, "mm_mlp_forward: layer %d: null kernel or non-positive width", l);
    MM_REQUIRE(acts[l] >= MM_ACT_LINEAR && acts[l] <= MM_ACT_GELU, MM_ERR_ARG, "mm_mlp_forward: unknown activation %d", acts[l]);
  }
  MM_REQUIRE(out_stride >= widths[n_layers - 1], MM_ERR_ARG, "mm_mlp_forward: out_stride < last width");
  MlpPlan p;
  plan_mlp(M, K, n_layers, widths, p);
  MM_REQUIRE(workspace && workspace_bytes >= p.total && ((uintptr_t)workspace % 256) == 0, MM_ERR_ARG,
             "mm_mlp_forward: workspace must be 256-B aligned and hold mm_mlp_workspace_bytes() = %lld bytes", (long long)p.total);
  if (M == 0) return MM_OK;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  void* a = ws + p.a_off;
  int rc = mm_split_rows(x, M, K, x_stride, a, mm_tc_padded_k(K), stream);
  if (rc) return rc;
  const void* w[8];
  int k = K;
  for (int l = 0; l < n_layers; ++l) {
    rc = mm_split_weights(kernels[l], k, widths[l], ws + p.w_off[l], mm_tc_padded_k(k), mm_tc_padded_n(widths[l]), stream);
    if (rc) return rc;
    w[l] = ws + p.w_off[l];
    k = widths[l];
  }
  if (n_layers >= 2 && n_layers <= 4 && mm_mlp_tc_supported(K, n_layers, widths, 0))
    return mm_mlp_tc(a, M, K, n_layers, w, widths, biases, acts, out, out_stride, nullptr, 0.0f, MM_ACT_LINEAR, nullptr, stream);
  const void* cur = a;
  k = K;
  for (int l = 0; l < n_layers; ++l) {
    const bool last = l == n_layers - 1;
    void* nxt = nullptr;
    int nxt_kp = 0;
    if (!last) {
      nxt = ws + p.act_off[l & 1];
      nxt_kp = mm_tc_padded_k(widths[l]);
      if (mm_tc_padded_n(widths[l]) < nxt_kp) {
        // the epilogue writes the columns of its n-tiles only (Np < Kp): clear the operand's zero padding
        cudaError_t e = cudaMemsetAsync(nxt, 0, (size_t)M * 2 * nxt_kp * 2, (cudaStream_t)stream);
        if (e != cudaSuccess) {
          mm::set_error("mm_mlp_forward: cudaMemsetAsync failed: %s", cudaGetErrorString(e));
          return (int)e;
        }
      }
    }
    rc = mm_dense_tc(cur, M, k, mm_tc_padded_k(k), w[l], widths[l], mm_tc_padded_n(widths[l]), biases[l], acts[l], 3, nullptr,
                     nullptr, 0, last ? out : nullptr, last ? out_stride : 0, nxt, nxt_kp, stream);
    if (rc) return rc;
    cur = nxt;
    k = widths[l];
  }
  return MM_OK;
}

int64_t mm_cross_workspace_bytes(int64_t M, int d, int depth) {
  if (M < 0 || d <= 0 || depth <= 0) return -1;
  const int64_t a = align_up(M * 2 * (int64_t)mm_tc_padded_k(d) * 2);
  const int64_t f = align_up(M * (int64_t)d * 4);
  const int64_t w = align_up((int64_t)mm_tc_padded_n(d) * 2 * mm_tc_padded_k(d) * 2);
  return 2 * a + 2 * f + depth * w;
}

int mm_cross_forward(const float* x0, int64_t M, int d, int64_t x_stride, int depth, const float* const* kernels,
                     const float* const* biases, float* out, int64_t out_stride, void* workspace, int64_t workspace_bytes,
                     void* stream) {
  MM_REQUIRE(x0 && kernels && biases && out && M >= 0 && d > 0 && x_stride >= d && out_stride >= d, MM_ERR_ARG,
             "mm_cross_forward: null pointer or bad M/d/stride");
  MM_REQUIRE(depth >= 1, MM_ERR_ARG, "mm_cross_forward: Number of cross layers (depth) should be positive but is %d.", depth);
  const int64_t need = mm_cross_workspace_bytes(M, d, depth);
  MM_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace % 256) == 0, MM_ERR_ARG,
             "mm_cross_forward: workspace must be 256-B aligned and hold mm_cross_workspace_bytes() = %lld bytes", (long long)need);
  if (M == 0) return MM_OK;
  const int Kp = mm_tc_padded_k(d), Np = mm_tc_padded_n(d);
  const int64_t a_bytes = align_up(M * 2 * (int64_t)Kp * 2), f_bytes = align_up(M * (int64_t)d * 4);
  const int64_t w_bytes = align_up((int64_t)Np * 2 * Kp * 2);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  void* a[2] = {ws, ws + a_bytes};
  float* f[2] = {reinterpret_cast<float*>(ws + 2 * a_bytes), reinterpret_cast<float*>(ws + 2 * a_bytes + f_bytes)};
  uint8_t* wbase = ws + 2 * a_bytes + 2 * f_bytes;
  MM_REQUIRE(depth == 1 || x_stride == d, MM_ERR_UNSUPPORTED,
             "mm_cross_forward: depth > 1 needs densely packed rows (x_stride == d): x0 and x_l share one row stride");
  int rc = mm_split_rows(x0, M, d, x_stride, a[0], Kp, stream);  // zero padded up to Kp
  if (rc) return rc;
  if (depth > 1 && Np < Kp) {
    // operand columns [Np, Kp) are never written by the epilogue: a[0] keeps the zeros of the split above,
    // a[1] is cleared once
    cudaError_t e = cudaMemsetAsync(a[1], 0, (size_t)a_bytes, (cudaStream_t)stream);
    if (e != cudaSuccess) {
      mm::set_error("mm_cross_forward: cudaMemsetAsync failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
  }
  const float* xres = x0;
  for (int l = 0; l < depth; ++l) {
    MM_REQUIRE(kernels[l], MM_ERR_ARG, "mm_cross_forward: layer %d: null kernel", l);
    void* w = wbase + (int64_t)l * w_bytes;
    rc = mm_split_weights(kernels[l], d, d, w, Kp, Np, stream);
    if (rc) return rc;
    const bool last = l == depth - 1;
    float* o = last ? out : f[l & 1];
    rc = mm_dense_tc(a[l & 1], M, d, Kp, w, d, Np, biases[l], MM_ACT_LINEAR, 3, x0, xres, x_stride, o, last ? out_stride : d,
                     last ? nullptr : a[(l + 1) & 1], last ? 0 : Kp, stream);
    if (rc) return rc;
    xres = o;
  }
  return MM_OK;
}

}  // extern "C"
