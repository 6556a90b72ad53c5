// Column concat (+cast to fp32) and row-wise L2 normalisation.
// Replaces ConcatFeatures (merlin/models/tf/core/aggregation.py:54-66), ContinuousFeatures'
// expand_dims (inputs/continuous.py:134-138) and L2Norm (transforms/regularization.py:27-82).
#include <cuda_bf16.h>

#include <cstring>

#include "mm_common.cuh"
#include "warp_mma.cuh"

namespace mm {

constexpr int MAX_PIECES = 64;
struct ConcatParams {
  mm_concat_piece p[MAX_PIECES];
  int n;
  int total_width;
};

// One thread per (row, piece-column); consecutive threads walk the pieces of one row, so the
// writes of a row are contiguous and the reads of width-1 pieces are coalesced across rows in
// the transposed launch below.
__global__ void concat_columns_kernel(const __grid_constant__ ConcatParams cp, long long B,
                                      float* __restrict__ out, long long out_stride) {
  // blockDim.x threads cover 32 rows x (piece columns); smem transposes so that both the
  // per-column reads (stride 1 across rows) and the row writes are coalesced.
  extern __shared__ float tile[];  // [32][W+1]
  const int W = cp.total_width;
  const long long b0 = (long long)blockIdx.x * 32;
  // read: thread -> (column c, row r) with r fastest
  for (int e = threadIdx.x; e < W * 32; e += blockDim.x) {
    const int r = e & 31, c = e >> 5;
    // find the piece of flat column c
    int pi = 0, base = 0;
    while (pi < cp.n - 1 && c >= base + cp.p[pi].width) {
      base += cp.p[pi].width;
      ++pi;
    }
    const long long b = b0 + r;
    float v = 0.0f;
    if (b < B) v = load_as_f32(cp.p[pi].src, b * cp.p[pi].src_stride + (c - base), cp.p[pi].dtype);
    tile[r * (W + 1) + c] = v;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < W * 32; e += blockDim.x) {
    const int c = e % W, r = e / W;
    int pi = 0, base = 0;
    while (pi < cp.n - 1 && c >= base + cp.p[pi].width) {
      base += cp.p[pi].width;
      ++pi;
    }
    const long long b = b0 + r;
    if (b < B) out[b * out_stride + cp.p[pi].out_col + (c - base)] = tile[r * (W + 1) + c];
  }
}

// Concat fused with the bf16 split of the tensor-core dense path: same transposing read as above, but the
// rows leave as the (B, 2*Kp) [hi | lo] operand of mm_dense_tc / mm_mlp_tc (zero padded to Kp), so the
// fp32 (B, W) matrix never exists.  Pieces sit at their out_col offsets inside the row.
template <int ROWS>
__global__ void __launch_bounds__(256)
concat_split_kernel(const __grid_constant__ ConcatParams cp, long long B, __nv_bfloat16* __restrict__ out, int Kp) {
  extern __shared__ float tile[];  // [ROWS][Kp+1], zero outside the pieces
  const long long b0 = (long long)blockIdx.x * ROWS;
  const int ld = Kp + 1;
  for (int e = threadIdx.x; e < ROWS * ld; e += blockDim.x) tile[e] = 0.0f;
  __syncthreads();
  const int W = cp.total_width;
  for (int e = threadIdx.x; e < W * ROWS; e += blockDim.x) {
    const int r = e % ROWS, c = e / ROWS;  // r fastest: a warp reads 32 consecutive rows of one column (coalesced)
    int pi = 0, base = 0;
    while (pi < cp.n - 1 && c >= base + cp.p[pi].width) {
      base += cp.p[pi].width;
      ++pi;
    }
    const long long b = b0 + r;
    if (b < B) tile[r * ld + cp.p[pi].out_col + (c - base)] = load_as_f32(cp.p[pi].src, b * cp.p[pi].src_stride + (c - base), cp.p[pi].dtype);
  }
  __syncthreads();
  const int groups = Kp >> 3;  // 8 bf16 = 16 bytes per store
  for (int e = threadIdx.x; e < ROWS * groups; e += blockDim.x) {
    const int g = e % groups, r = e / groups;
    const long long b = b0 + r;
    if (b >= B) continue;
    __align__(16) __nv_bfloat16 h[8], l[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) split_bf16(tile[r * ld + g * 8 + j], h[j], l[j]);
    __nv_bfloat16* o = out + b * (2ll * Kp) + g * 8;
    *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(h);
    *reinterpret_cast<uint4*>(o + Kp) = *reinterpret_cast<const uint4*>(l);
  }
}

__global__ void l2_normalize_kernel(const float* __restrict__ x, long long B, int D, long long x_stride,
                                    float* __restrict__ out, long long out_stride) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long b = warp0; b < B; b += n_warps) {
    float ss = 0.0f;
    for (int d = lane; d < D; d += 32) {
      const float v = x[b * x_stride + d];
      ss = fmaf(v, v, ss);
    }
    ss = warp_sum(ss);
    const float nrm = sqrtf(fmaxf(ss, 1e-12f));
    for (int d = lane; d < D; d += 32) out[b * out_stride + d] = x[b * x_stride + d] / nrm;
  }
}

// Backward of l2_normalize_kernel, y = x / sqrt(max(sum(x^2), 1e-12)) (transforms/regularization.py:27-82).  TF's gradient
// of tf.math.maximum(s, eps) flows to s where s >= eps, so: s >= 1e-12: dx = (dy - y (y . dy)) / n, n = sqrt(s);
// otherwise the denominator is the constant 1e-6 and dx = dy / 1e-6.  Each lane reads x[d], dy[d] before it writes dx[d]:
// dx may alias x or dy.
__global__ void l2_normalize_backward_kernel(const float* x, const float* dy, long long B, int D, long long x_stride,
                                             long long dy_stride, float* dx, long long dx_stride) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long b = warp0; b < B; b += n_warps) {
    float ss = 0.0f, xg = 0.0f;
    for (int d = lane; d < D; d += 32) {
      const float v = x[b * x_stride + d], g = dy[b * dy_stride + d];
      ss = fmaf(v, v, ss);
      xg = fmaf(v, g, xg);
    }
    ss = warp_sum(ss);
    xg = warp_sum(xg);
    const bool on = ss >= 1e-12f;
    const float nrm = on ? sqrtf(ss) : 1e-6f;
    const float yg = on ? xg / nrm : 0.0f;  // y . dy
    for (int d = lane; d < D; d += 32) {
      const float y = x[b * x_stride + d] / nrm;
      dx[b * dx_stride + d] = (dy[b * dy_stride + d] - y * yg) / nrm;
    }
  }
}

// out[b, c] = x[b, c] * scale[c] + shift[c]: tf.keras.layers.BatchNormalization at inference with
// scale = gamma / sqrt(moving_var + eps), shift = beta - moving_mean * scale (blocks/mlp.py:131-135).
// Only the LAST normalization of a block reaches this kernel; the others are folded into the next Dense.
__global__ void scale_shift_kernel(const float* __restrict__ x, long long B, int D, long long x_stride,
                                   const float* __restrict__ scale, const float* __restrict__ shift,
                                   float* __restrict__ out, long long out_stride) {
  const long long total = B * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / D;
    const int c = (int)(i - b * D);
    out[b * out_stride + c] = fmaf(x[b * x_stride + c], scale[c], shift[c]);
  }
}


// x = mask > 0 ? x : 0 in place over (B, D) row-major views: the relu derivative applied to a gradient (training step; the
// narrow-layer dgrad kernel fuses it, the tensor-core path for wide layers applies it afterwards)
__global__ void relu_mask_kernel(float* __restrict__ x, long long B, int D, long long sx, const float* __restrict__ mask, long long sm) {
  const long long total = B * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / D;
    const int k = (int)(i - r * D);
    if (!(mask[r * sm + k] > 0.0f)) x[r * sx + k] = 0.0f;
  }
}

// out = a * b + c elementwise over (B, D) row-major views (the DCN-v2 cross combine x0 * projection + x when the
// projection is not produced by a GEMM with the fused cross epilogue: low-rank kernels on the exact-fp32 engine)
__global__ void fma3_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
                            long long B, int D, long long sa, long long sb, long long sc, float* __restrict__ out, long long so) {
  const long long total = B * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / D;
    const int k = (int)(i - r * D);
    out[r * so + k] = fmaf(a[r * sa + k], b[r * sb + k], c[r * sc + k]);
  }
}

}  // namespace mm

extern "C" {

int mm_concat_columns(const mm_concat_piece* pieces_host, int n_pieces, int64_t B, float* out,
                      int64_t out_stride, void* stream) {
  MM_REQUIRE(pieces_host && out && n_pieces > 0 && B >= 0, MM_ERR_ARG,
             "mm_concat_columns: null pointer or no pieces");
  if (B == 0) return MM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  for (int s = 0; s < n_pieces; s += mm::MAX_PIECES) {
    mm::ConcatParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.n = (n_pieces - s < mm::MAX_PIECES) ? n_pieces - s : mm::MAX_PIECES;
    for (int i = 0; i < cp.n; ++i) {
      const mm_concat_piece& pc = pieces_host[s + i];
      MM_REQUIRE(pc.src && pc.width > 0 && pc.src_stride >= 0 && pc.out_col >= 0 &&
                     (int64_t)pc.out_col + pc.width <= out_stride,
                 MM_ERR_ARG, "mm_concat_columns: piece %d: null src, bad width or out of row", s + i);
      MM_REQUIRE(pc.dtype >= MM_I32 && pc.dtype <= MM_F64, MM_ERR_ARG,
                 "mm_concat_columns: piece %d: unknown dtype %d", s + i, pc.dtype);
      cp.p[i] = pc;
      cp.total_width += pc.width;
    }
    const size_t smem = (size_t)32 * (cp.total_width + 1) * sizeof(float);
    MM_REQUIRE(smem <= 48 * 1024, MM_ERR_UNSUPPORTED,
               "mm_concat_columns: %d columns per launch exceed the 48 KB tile", cp.total_width);
    const unsigned blocks = (unsigned)((B + 31) / 32);
    mm::concat_columns_kernel<<<blocks, 256, smem, st>>>(cp, B, out, out_stride);
    int rc = mm::check_launch("mm_concat_columns");
    if (rc) return rc;
  }
  return MM_OK;
}

int mm_concat_split(const mm_concat_piece* pieces_host, int n_pieces, int64_t B, void* out_split, int Kp,
                    void* stream) {
  MM_REQUIRE(pieces_host && out_split && n_pieces > 0 && B >= 0, MM_ERR_ARG, "mm_concat_split: null pointer or no pieces");
  MM_REQUIRE(n_pieces <= mm::MAX_PIECES, MM_ERR_UNSUPPORTED, "mm_concat_split: more than %d pieces", mm::MAX_PIECES);
  MM_REQUIRE(Kp > 0 && Kp % 64 == 0, MM_ERR_ARG, "mm_concat_split: Kp must be a positive multiple of 64");
  MM_REQUIRE(((uintptr_t)out_split % 16) == 0, MM_ERR_ALIGN, "mm_concat_split: out_split must be 16-B aligned");
  if (B == 0) return MM_OK;
  mm::ConcatParams cp;
  memset(&cp, 0, sizeof(cp));
  cp.n = n_pieces;
  for (int i = 0; i < n_pieces; ++i) {
    const mm_concat_piece& pc = pieces_host[i];
    MM_REQUIRE(pc.src && pc.width > 0 && pc.src_stride >= 0 && pc.out_col >= 0 && (int64_t)pc.out_col + pc.width <= Kp,
               MM_ERR_ARG, "mm_concat_split: piece %d: null src, bad width or beyond Kp", i);
    MM_REQUIRE(pc.dtype >= MM_I32 && pc.dtype <= MM_F64, MM_ERR_ARG, "mm_concat_split: piece %d: unknown dtype %d", i, pc.dtype);
    cp.p[i] = pc;
    cp.total_width += pc.width;
  }
  MM_REQUIRE((size_t)32 * (Kp + 1) * sizeof(float) <= 48 * 1024, MM_ERR_UNSUPPORTED,
             "mm_concat_split: Kp = %d exceeds the 48 KB tile", Kp);
  // 32-row blocks: 128-row blocks (4x fewer, fatter CTAs) measured slower, 12.5 vs 10.4 us at B = 65 536
  mm::concat_split_kernel<32><<<(unsigned)((B + 31) / 32), 256, (size_t)32 * (Kp + 1) * sizeof(float), (cudaStream_t)stream>>>(
      cp, B, (__nv_bfloat16*)out_split, Kp);
  return mm::check_launch("mm_concat_split");
}

int mm_l2_normalize(const float* x, int64_t B, int D, int64_t x_stride, float* out,
                    int64_t out_stride, void* stream) {
  MM_REQUIRE(x && out && B >= 0 && D > 0 && x_stride >= D && out_stride >= D, MM_ERR_ARG,
             "mm_l2_normalize: null pointer, D<=0 or stride < D");
  if (B == 0) return MM_OK;
  const int threads = 256;
  long long blocks = (B * 32 + threads - 1) / threads;
  const long long cap = (long long)mm::sm_count() * 32;
  if (blocks > cap) blocks = cap;
  mm::l2_normalize_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(x, B, D, x_stride, out,
                                                                                out_stride);
  return mm::check_launch("mm_l2_normalize");
}

int mm_l2_normalize_backward(const float* x, const float* dy, int64_t B, int D, int64_t x_stride, int64_t dy_stride, float* dx,
                             int64_t dx_stride, void* stream) {
  MM_REQUIRE(x && dy && dx && B >= 0 && D > 0 && x_stride >= D && dy_stride >= D && dx_stride >= D, MM_ERR_ARG,
             "mm_l2_normalize_backward: null pointer, D<=0 or stride < D");
  if (B == 0) return MM_OK;
  const int threads = 256;
  long long blocks = (B * 32 + threads - 1) / threads;
  const long long cap = (long long)mm::sm_count() * 32;
  if (blocks > cap) blocks = cap;
  mm::l2_normalize_backward_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(x, dy, B, D, x_stride, dy_stride, dx,
                                                                                         dx_stride);
  return mm::check_launch("mm_l2_normalize_backward");
}

int mm_scale_shift(const float* x, int64_t B, int D, int64_t x_stride, const float* scale, const float* shift,
                   float* out, int64_t out_stride, void* stream) {
  MM_REQUIRE(x && out && scale && shift && B >= 0 && D > 0 && x_stride >= D && out_stride >= D, MM_ERR_ARG,
             "mm_scale_shift: null pointer, D<=0 or stride < D");
  if (B == 0) return MM_OK;
  const int threads = 256;
  long long blocks = (B * D + threads - 1) / threads;
  const long long cap = (long long)mm::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  mm::scale_shift_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(x, B, D, x_stride, scale, shift, out,
                                                                               out_stride);
  return mm::check_launch("mm_scale_shift");
}

int mm_relu_mask(float* x, int64_t B, int D, int64_t x_stride, const float* mask, int64_t mask_stride, void* stream) {
  MM_REQUIRE(x && mask && B >= 0 && D > 0 && x_stride >= D && mask_stride >= D, MM_ERR_ARG, "mm_relu_mask: null pointer, D<=0 or stride < D");
  if (B == 0) return MM_OK;
  const int threads = 256;
  long long blocks = (B * D + threads - 1) / threads;
  const long long cap = (long long)mm::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  mm::relu_mask_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(x, B, D, x_stride, mask, mask_stride);
  return mm::check_launch("mm_relu_mask");
}

int mm_cross_combine(const float* x0, const float* proj, const float* x, int64_t B, int D, int64_t x0_stride,
                     int64_t proj_stride, int64_t x_stride, float* out, int64_t out_stride, void* stream) {
  MM_REQUIRE(x0 && proj && x && out && B >= 0 && D > 0 && x0_stride >= D && proj_stride >= D && x_stride >= D && out_stride >= D,
             MM_ERR_ARG, "mm_cross_combine: null pointer, D<=0 or stride < D");
  if (B == 0) return MM_OK;
  const int threads = 256;
  long long blocks = (B * D + threads - 1) / threads;
  const long long cap = (long long)mm::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  mm::fma3_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(x0, proj, x, B, D, x0_stride, proj_stride, x_stride, out,
                                                                        out_stride);
  return mm::check_launch("mm_cross_combine");
}

}  // extern "C"
