// Backward of the Dense layers of the DLRM path (training step, SURVEY §8(f)-4): what tf.GradientTape
// (merlin/models/tf/models/base.py:1121-1231, `train_step`) computes for blocks/mlp.py:275-280 and the
// BinaryOutput head (outputs/classification.py:114), written for narrow layers (K, N <= a few hundred) over a huge
// batch: the whole backward is 19 GFLOP against ~1 GB of activations per 65 536 samples, so every kernel
// here is organised around streaming the activations once.
//
//   mm_heads_fwd_bwd     z_h = x.W[:, h] + b_h, loss += sum BCE / MSE(z_h, y_h), dz_h = lambda_h sw_i l'_h / M,
//                        dx = sum_h dz_h W[:, h]^T [x > 0], dW += x^T dz, db += sum dz   (one warp per row, no GEMM)
//   mm_dense_wgrad       dW += X^T dZ, db += column sums of dZ                  (reduction over the batch)
//   mm_dense_dgrad       dX = (dZ W^T) [mask > 0]                                (mask: the layer input = the
//                        previous layer's relu output, so the result is that layer's pre-activation gradient)
//
// Arithmetic: mma.sync.m16n8k16 bf16 with the library's 3-pass split (hi*lo + lo*hi + hi*hi, fp32 accumulate):
// fp32-grade (|err| ~ 2^-16 relative) like the forward layers.  The batch reduction of wgrad runs over CTAs and ends in
// fp32 atomics: the summation ORDER is not fixed, results agree with autograd to fp32 rounding, not bit for bit.
#include <cuda_bf16.h>

#include <cstring>

#include "mm_common.cuh"
#include "warp_mma.cuh"

namespace mm {
namespace trn {

// ---------------------------------------------------------------------------------------------------------------
// Heads: H <= 8 outputs Dense(K -> 1) on the same body vector, forward and backward in one pass over x.
//   BCE (BinaryOutput): Keras evaluates BCE on the logits cached by the sigmoid activation (`_keras_logits`):
//     l_i = max(z,0) - z*y + log(1 + exp(-|z|)),   dl/dz = sigmoid(z) - y
//   MSE (RegressionOutput, linear):  l_i = (z - y)^2,   dl/dz = 2 (z - y)
// loss_h = sum_i sw_i l_h,i / M (Keras "sum_over_batch_size"), total = sum_h lambda_h loss_h, dz_h = lambda_h sw_i l'_h / M.
// H and TRAIN are template parameters; the loss kind of a head is a uniform runtime branch.  H = 1 (a model with one
// output head) is its own instantiation, so the single-head step pays for no loop over unused heads.
// ---------------------------------------------------------------------------------------------------------------
constexpr int HEAD_MAX = 8;

struct HeadParams {
  const float* x;
  long long ldx;
  long long M;
  int K;
  const float* w;     // (K, H) Keras layout
  const float* bias;  // (H,) device or null
  const void* y[HEAD_MAX];
  int y_dtype[HEAD_MAX];
  int kind[HEAD_MAX];    // MM_LOSS_BCE / MM_LOSS_MSE
  float lw[HEAD_MAX];    // loss weights lambda_h
  const float* sample_w[HEAD_MAX];  // (M,) or null
  float inv_m;            // 1 / M  (Keras "sum_over_batch_size")
  float* logits;          // (H, M) or null; forward only: the activated predictions
  float* loss;            // total, accumulated (device scalar) or null
  float* loss_heads;      // (H,) unweighted per-head losses, accumulated, or null
  float* dx;
  long long lddx;
  int mask_relu;
  float* dw;  // (K, H) accumulated
  float* db;  // (H,) accumulated
};

constexpr int HEAD_KMAX = 256;  // 8 columns per lane

template <int H, bool TRAIN>
__global__ void __launch_bounds__(256, H == 1 ? 2 : 1) head_kernel(const HeadParams p) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  constexpr int C = HEAD_KMAX / 32;
  float w[H][C], dw[H][C];
  float b[H], loss[H], db[H];
#pragma unroll
  for (int h = 0; h < H; ++h) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const int k = lane + 32 * c;
      w[h][c] = k < p.K ? p.w[k * H + h] : 0.0f;
      dw[h][c] = 0.0f;
    }
    b[h] = p.bias ? p.bias[h] : 0.0f;
    loss[h] = db[h] = 0.0f;
  }
  for (long long m = warp; m < p.M; m += n_warps) {
    float x[C];
    float dot[H];
#pragma unroll
    for (int h = 0; h < H; ++h) dot[h] = 0.0f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const int k = lane + 32 * c;
      x[c] = k < p.K ? p.x[m * p.ldx + k] : 0.0f;
#pragma unroll
      for (int h = 0; h < H; ++h) dot[h] = fmaf(x[c], w[h][c], dot[h]);
    }
    float dz[H];
#pragma unroll
    for (int h = 0; h < H; ++h) {
      const float z = warp_sum(dot[h]) + b[h];
      if (!TRAIN) {
        if (lane == 0) p.logits[h * p.M + m] = head_pred(p.kind[h], z);
        continue;
      }
      const float y = load_as_f32(p.y[h], m, p.y_dtype[h]);
      const float sw = p.sample_w[h] ? p.sample_w[h][m] : 1.0f;
      float l, g;
      head_loss(p.kind[h], z, y, l, g);
      dz[h] = g * sw * p.inv_m;
      dz[h] *= p.lw[h];  // exact for lambda = 1
      if (lane == 0) {
        loss[h] += l * sw * p.inv_m;
        db[h] += dz[h];
        if (p.logits) p.logits[h * p.M + m] = z;
      }
    }
    if (!TRAIN) continue;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const int k = lane + 32 * c;
      if (k < p.K) {
        float d = dz[0] * w[0][c];
#pragma unroll
        for (int h = 0; h < H; ++h) {
          dw[h][c] = fmaf(x[c], dz[h], dw[h][c]);
          if (h > 0) d = fmaf(dz[h], w[h][c], d);
        }
        if (p.dx) p.dx[m * p.lddx + k] = (!p.mask_relu || x[c] > 0.0f) ? d : 0.0f;
      }
    }
  }
  if (!TRAIN) return;
  // block-level reduction of dw / db / loss before the atomics, one head at a time
  __shared__ float red[8][HEAD_KMAX + 2];
  const int wid = threadIdx.x >> 5;
  const int nw = blockDim.x >> 5;
#pragma unroll
  for (int h = 0; h < H; ++h) {
    if (h > 0) __syncthreads();  // the previous head's sums have been read
#pragma unroll
    for (int c = 0; c < C; ++c) red[wid][lane + 32 * c] = dw[h][c];
    if (lane == 0) {
      red[wid][HEAD_KMAX] = db[h];
      red[wid][HEAD_KMAX + 1] = loss[h];
    }
    __syncthreads();
    for (int k = threadIdx.x; k < HEAD_KMAX + 2; k += blockDim.x) {
      float s = 0.0f;
      for (int i = 0; i < nw; ++i) s += red[i][k];
      if (k < p.K) {
        if (p.dw) atomicAdd(p.dw + k * H + h, s);
      } else if (k == HEAD_KMAX) {
        if (p.db) atomicAdd(p.db + h, s);
      } else if (k == HEAD_KMAX + 1) {
        if (p.loss) atomicAdd(p.loss, p.lw[h] * s);
        if (p.loss_heads) atomicAdd(p.loss_heads + h, s);
      }
    }
  }
}

// K a multiple of 4 with 16-byte aligned rows: G = K/4 (rounded up to a power of two, <= 32) lanes own one row as
// float4 pieces, a warp processes 32/G rows at a time (K = 32: 4 rows per warp, one 128-byte row per 8 lanes).
template <int G, int H, bool TRAIN>
__global__ void __launch_bounds__(256, H == 1 ? 2 : 1) head_kernel_v4(const HeadParams p) {
  const int lane = threadIdx.x & 31;
  const int c = lane % G, sub = lane / G;
  constexpr int RPW = 32 / G;  // rows per warp and iteration
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const bool on = 4 * c < p.K;
  float4 w[H], dw[H];
  float b[H], loss[H], db[H];
#pragma unroll
  for (int h = 0; h < H; ++h) {
    if (H == 1) {
      w[h] = on ? *reinterpret_cast<const float4*>(p.w + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      w[h] = on ? make_float4(p.w[(4 * c) * H + h], p.w[(4 * c + 1) * H + h], p.w[(4 * c + 2) * H + h], p.w[(4 * c + 3) * H + h])
                : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    dw[h] = make_float4(0.f, 0.f, 0.f, 0.f);
    b[h] = p.bias ? p.bias[h] : 0.0f;
    loss[h] = db[h] = 0.0f;
  }
  const long long groups = (p.M + RPW - 1) / RPW;
  for (long long gi = warp; gi < groups; gi += n_warps) {
    const long long m = gi * RPW + sub;
    const bool live = m < p.M;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live && on) x = __ldg(reinterpret_cast<const float4*>(p.x + m * p.ldx + 4 * c));
    float dz[H];
#pragma unroll
    for (int h = 0; h < H; ++h) {
      float dot = x.x * w[h].x + x.y * w[h].y + x.z * w[h].z + x.w * w[h].w;
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      const float z = dot + b[h];
      dz[h] = 0.0f;
      if (!TRAIN) {
        if (live && c == 0) p.logits[h * p.M + m] = head_pred(p.kind[h], z);
        continue;
      }
      if (live) {
        const float y = load_as_f32(p.y[h], m, p.y_dtype[h]);
        const float sw = p.sample_w[h] ? p.sample_w[h][m] : 1.0f;
        float l, g;
        head_loss(p.kind[h], z, y, l, g);
        dz[h] = g * sw * p.inv_m;
        dz[h] *= p.lw[h];  // exact for lambda = 1
        if (c == 0) {
          loss[h] += l * sw * p.inv_m;
          db[h] += dz[h];
          if (p.logits) p.logits[h * p.M + m] = z;
        }
      }
    }
    if (!TRAIN) continue;
#pragma unroll
    for (int h = 0; h < H; ++h) {
      dw[h].x = fmaf(x.x, dz[h], dw[h].x);
      dw[h].y = fmaf(x.y, dz[h], dw[h].y);
      dw[h].z = fmaf(x.z, dz[h], dw[h].z);
      dw[h].w = fmaf(x.w, dz[h], dw[h].w);
    }
    if (live && on && p.dx) {
      float4 g = make_float4(dz[0] * w[0].x, dz[0] * w[0].y, dz[0] * w[0].z, dz[0] * w[0].w);
#pragma unroll
      for (int h = 1; h < H; ++h) {
        g.x = fmaf(dz[h], w[h].x, g.x);
        g.y = fmaf(dz[h], w[h].y, g.y);
        g.z = fmaf(dz[h], w[h].z, g.z);
        g.w = fmaf(dz[h], w[h].w, g.w);
      }
      float4 d;
      d.x = (!p.mask_relu || x.x > 0.0f) ? g.x : 0.0f;
      d.y = (!p.mask_relu || x.y > 0.0f) ? g.y : 0.0f;
      d.z = (!p.mask_relu || x.z > 0.0f) ? g.z : 0.0f;
      d.w = (!p.mask_relu || x.w > 0.0f) ? g.w : 0.0f;
      *reinterpret_cast<float4*>(p.dx + m * p.lddx + 4 * c) = d;
    }
  }
  if (!TRAIN) return;
  // lanes with the same c hold partial sums of the same columns: fold the row groups of the warp, then the block
#pragma unroll
  for (int h = 0; h < H; ++h) {
#pragma unroll
    for (int o = G; o < 32; o <<= 1) {
      dw[h].x += __shfl_xor_sync(0xffffffffu, dw[h].x, o);
      dw[h].y += __shfl_xor_sync(0xffffffffu, dw[h].y, o);
      dw[h].z += __shfl_xor_sync(0xffffffffu, dw[h].z, o);
      dw[h].w += __shfl_xor_sync(0xffffffffu, dw[h].w, o);
      loss[h] += __shfl_xor_sync(0xffffffffu, loss[h], o);
      db[h] += __shfl_xor_sync(0xffffffffu, db[h], o);
    }
  }
  __shared__ float red[8][4 * G + 2];
  const int wid = threadIdx.x >> 5;
  const int nw = blockDim.x >> 5;
#pragma unroll
  for (int h = 0; h < H; ++h) {
    if (h > 0) __syncthreads();  // the previous head's sums have been read
    if (lane < G) {
      red[wid][4 * lane] = dw[h].x;
      red[wid][4 * lane + 1] = dw[h].y;
      red[wid][4 * lane + 2] = dw[h].z;
      red[wid][4 * lane + 3] = dw[h].w;
    }
    if (lane == 0) {
      red[wid][4 * G] = db[h];
      red[wid][4 * G + 1] = loss[h];
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 4 * G + 2; k += blockDim.x) {
      float s = 0.0f;
      for (int i = 0; i < nw; ++i) s += red[i][k];
      if (k < 4 * G) {
        if (k < p.K && p.dw) atomicAdd(p.dw + k * H + h, s);
      } else if (k == 4 * G) {
        if (p.db) atomicAdd(p.db + h, s);
      } else {
        if (p.loss) atomicAdd(p.loss, p.lw[h] * s);
        if (p.loss_heads) atomicAdd(p.loss_heads + h, s);
      }
    }
  }
}

template <int H, bool TRAIN>
static void launch_heads(const HeadParams& p, bool vec, unsigned blocks, cudaStream_t st) {
  if (vec) {
    const int g = p.K / 4;
    if (g <= 2) head_kernel_v4<2, H, TRAIN><<<blocks, 256, 0, st>>>(p);
    else if (g <= 4) head_kernel_v4<4, H, TRAIN><<<blocks, 256, 0, st>>>(p);
    else if (g <= 8) head_kernel_v4<8, H, TRAIN><<<blocks, 256, 0, st>>>(p);
    else if (g <= 16) head_kernel_v4<16, H, TRAIN><<<blocks, 256, 0, st>>>(p);
    else head_kernel_v4<32, H, TRAIN><<<blocks, 256, 0, st>>>(p);
  } else {
    head_kernel<H, TRAIN><<<blocks, 256, 0, st>>>(p);
  }
}

// the instantiation for p's head count
template <bool TRAIN>
static void launch_heads(const HeadParams& p, int H, bool vec, unsigned blocks, cudaStream_t st) {
  switch (H) {
    case 1: launch_heads<1, TRAIN>(p, vec, blocks, st); break;
    case 2: launch_heads<2, TRAIN>(p, vec, blocks, st); break;
    case 3: launch_heads<3, TRAIN>(p, vec, blocks, st); break;
    case 4: launch_heads<4, TRAIN>(p, vec, blocks, st); break;
    case 5: launch_heads<5, TRAIN>(p, vec, blocks, st); break;
    case 6: launch_heads<6, TRAIN>(p, vec, blocks, st); break;
    case 7: launch_heads<7, TRAIN>(p, vec, blocks, st); break;
    default: launch_heads<8, TRAIN>(p, vec, blocks, st); break;
  }
}

static void run_heads(const HeadParams& p, int H, bool train, cudaStream_t st) {
  long long blocks = (p.M + 7) / 8;
  const long long cap = 4LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  // float4 weights need 16-byte aligned kernel rows: only one head's (K, 1) kernel is read as float4
  const bool vec = (p.K & 3) == 0 && p.K <= 128 && (p.ldx & 3) == 0 && ((uintptr_t)p.x & 15) == 0 &&
                   (H > 1 || ((uintptr_t)p.w & 15) == 0) && (!p.dx || ((p.lddx & 3) == 0 && ((uintptr_t)p.dx & 15) == 0));
  if (train) launch_heads<true>(p, H, vec, (unsigned)blocks, st);
  else launch_heads<false>(p, H, vec, (unsigned)blocks, st);
}

// ---------------------------------------------------------------------------------------------------------------
// wgrad:  dW[K, N] += sum_m X[m, :]^T dZ[m, :],  db[N] += sum_m dZ[m, :]
// MMA view: M' = K (rows of dW), N' = N, K' = batch rows.  A CTA owns a (KS x NS) tile of dW and a contiguous slice of
// the batch; 32-row chunks of X and dZ are split into bf16 (hi, lo) while they are stored to shared memory ([m][k]
// row-major, +16 B row padding) and both operands are fetched with ldmatrix.trans (the reduction index m is the slow
// index of both).  Global loads of chunk i+1 are in flight while chunk i is multiplied.
// ---------------------------------------------------------------------------------------------------------------
struct WgradParams {
  const float* x;
  long long ldx;
  const float* dz;
  long long ldz;
  long long M;
  int K, N;
  float* dw;  // (K, N) contiguous, accumulated
  float* db;  // (N,) accumulated or null
  long long rows_per_cta;  // multiple of 32
  int x_vec, z_vec;        // 16-byte loads are legal
  const __nv_bfloat16* x_split;  // XSPLIT: X as split-bf16 rows (M, 2*Kp) = [hi | lo] (mm_split_rows layout) instead of fp32
  int Kp;
};

__device__ __forceinline__ float4 load4(const float* row, int c, int C, bool vec) {
  if (vec && c + 3 < C) return __ldg(reinterpret_cast<const float4*>(row + c));
  float4 v;
  v.x = c < C ? __ldg(row + c) : 0.0f;
  v.y = c + 1 < C ? __ldg(row + c + 1) : 0.0f;
  v.z = c + 2 < C ? __ldg(row + c + 2) : 0.0f;
  v.w = c + 3 < C ? __ldg(row + c + 3) : 0.0f;
  return v;
}

template <int WM, int MT, int WN, int NT, bool XSPLIT>
__global__ void __launch_bounds__(32 * WM * WN) wgrad_kernel(const WgradParams p) {
  constexpr int T = 32 * WM * WN;
  constexpr int KS = WM * MT * 16, NS = WN * NT * 8;
  constexpr int SX = KS * 2 + 16, SZ = NS * 2 + 16;  // bytes per staged row
  constexpr int XQ = KS / 4, ZQ = NS / 4;            // float4 per staged row
  constexpr int XV = (32 * XQ + T - 1) / T, ZV = (32 * ZQ + T - 1) / T;
  static_assert(T % ZQ == 0, "a thread stages a fixed column group of dZ (bias-gradient partial sums)");
  __shared__ __align__(16) uint8_t smem[2 * 32 * SX + 2 * 32 * SZ];
  uint8_t* xh = smem;
  uint8_t* xl = smem + 32 * SX;
  uint8_t* zh = smem + 64 * SX;
  uint8_t* zl = zh + 32 * SZ;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp / WN, wn = warp % WN;
  const int k0 = blockIdx.y * KS, n0 = blockIdx.z * NS;
  const long long m_begin = (long long)blockIdx.x * p.rows_per_cta;
  const long long m_end = min(p.M, m_begin + p.rows_per_cta);
  if (m_begin >= m_end) return;

  float acc[MT][NT][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0f;
  float4 dbs = make_float4(0.f, 0.f, 0.f, 0.f);

  float4 xr[XV], zr[ZV];
  auto prefetch = [&](long long mb) {
#pragma unroll
    for (int i = 0; i < XV; ++i) {
      const int e = tid + i * T;
      const int r = e / XQ, c = (e % XQ) * 4;
      const long long m = mb + r;
      if (XSPLIT) {
        // four bf16 hi values and four lo values, already split: bit patterns travel through the float4
        uint2 h = make_uint2(0u, 0u), l = h;
        if (e < 32 * XQ && m < m_end && k0 + c < p.Kp) {
          const __nv_bfloat16* row = p.x_split + m * (2ll * p.Kp) + k0 + c;
          h = __ldg(reinterpret_cast<const uint2*>(row));
          l = __ldg(reinterpret_cast<const uint2*>(row + p.Kp));
        }
        xr[i] = make_float4(__uint_as_float(h.x), __uint_as_float(h.y), __uint_as_float(l.x), __uint_as_float(l.y));
      } else {
        xr[i] = (e < 32 * XQ && m < m_end) ? load4(p.x + m * p.ldx, k0 + c, p.K, p.x_vec) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int i = 0; i < ZV; ++i) {
      const int e = tid + i * T;
      const int r = e / ZQ, c = (e % ZQ) * 4;
      const long long m = mb + r;
      zr[i] = (e < 32 * ZQ && m < m_end) ? load4(p.dz + m * p.ldz, n0 + c, p.N, p.z_vec) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto stage = [&]() {
#pragma unroll
    for (int i = 0; i < XV; ++i) {
      const int e = tid + i * T;
      if (e < 32 * XQ) {
        const int r = e / XQ, c = (e % XQ) * 4;
        uint32_t h0, l0, h1, l1;
        if (XSPLIT) {
          h0 = __float_as_uint(xr[i].x);
          h1 = __float_as_uint(xr[i].y);
          l0 = __float_as_uint(xr[i].z);
          l1 = __float_as_uint(xr[i].w);
        } else {
          split_pair(xr[i].x, xr[i].y, h0, l0);
          split_pair(xr[i].z, xr[i].w, h1, l1);
        }
        *reinterpret_cast<uint2*>(xh + r * SX + c * 2) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(xl + r * SX + c * 2) = make_uint2(l0, l1);
      }
    }
#pragma unroll
    for (int i = 0; i < ZV; ++i) {
      const int e = tid + i * T;
      if (e < 32 * ZQ) {
        const int r = e / ZQ, c = (e % ZQ) * 4;
        uint32_t h0, l0, h1, l1;
        split_pair(zr[i].x, zr[i].y, h0, l0);
        split_pair(zr[i].z, zr[i].w, h1, l1);
        *reinterpret_cast<uint2*>(zh + r * SZ + c * 2) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(zl + r * SZ + c * 2) = make_uint2(l0, l1);
        dbs.x += zr[i].x;
        dbs.y += zr[i].y;
        dbs.z += zr[i].z;
        dbs.w += zr[i].w;
      }
    }
  };

  // ldmatrix row addresses of this lane (see the fragment maps in the file header of tower_small.cu):
  //   A (= X^T) quad of m-tile mt, k-step ks: matrices (kk 0-7, i 0-7) (kk 0-7, i 8-15) (kk 8-15, i 0-7) (kk 8-15, i 8-15)
  //   B (= dZ) pairs of n-tiles 2u, 2u+1:     matrices (kk 0-7, 2u) (kk 8-15, 2u) (kk 0-7, 2u+1) (kk 8-15, 2u+1)
  const int q = lane >> 3, r8 = lane & 7;
  const uint32_t xs_base = (uint32_t)__cvta_generic_to_shared(xh), zs_base = (uint32_t)__cvta_generic_to_shared(zh);
  const uint32_t a_lane = (uint32_t)(((q >> 1) * 8 + r8) * SX + (wm * MT * 16 + (q & 1) * 8) * 2);
  const uint32_t b_lane = (uint32_t)(((q & 1) * 8 + r8) * SZ + (wn * NT * 8 + (NT > 1 ? (q >> 1) * 8 : 0)) * 2);

  prefetch(m_begin);
  for (long long mb = m_begin; mb < m_end; mb += 32) {
    __syncthreads();  // the previous chunk has been consumed
    stage();
    __syncthreads();
    if (mb + 32 < m_end) prefetch(mb + 32);
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      uint32_t ah[MT][4], al[MT][4];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const uint32_t a = xs_base + a_lane + (uint32_t)(ks * 16 * SX + mt * 32);
        ldsm_x4_t(a, ah[mt][0], ah[mt][1], ah[mt][2], ah[mt][3]);
        ldsm_x4_t(a + 32 * SX, al[mt][0], al[mt][1], al[mt][2], al[mt][3]);
      }
      constexpr int NP = (NT + 1) / 2;
#pragma unroll
      for (int u = 0; u < NP; ++u) {
        uint32_t bh[4], bl[4];
        const uint32_t b = zs_base + b_lane + (uint32_t)(ks * 16 * SZ + u * 32);
        ldsm_x4_t(b, bh[0], bh[1], bh[2], bh[3]);
        ldsm_x4_t(b + 32 * SZ, bl[0], bl[1], bl[2], bl[3]);
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const int nt = 2 * u + v;
          if (nt < NT) {
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) mma16816(acc[mt][nt], ah[mt], bl[2 * v], bl[2 * v + 1]);
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) mma16816(acc[mt][nt], al[mt], bh[2 * v], bh[2 * v + 1]);
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) mma16816(acc[mt][nt], ah[mt], bh[2 * v], bh[2 * v + 1]);
          }
        }
      }
    }
  }
  // ---- this CTA's partial tile -> global (fp32 atomics)
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int k = k0 + (wm * MT + mt) * 16 + g + 8 * (c >> 1);
        const int n = n0 + (wn * NT + nt) * 8 + 2 * t + (c & 1);
        if (k < p.K && n < p.N) atomicAdd(p.dw + (long long)k * p.N + n, acc[mt][nt][c]);
      }
  if (p.db && blockIdx.y == 0) {
    // thread tid stages column group (tid % ZQ): reduce the T / ZQ threads of a group through shared memory
    __syncthreads();
    float* red = reinterpret_cast<float*>(smem);
    for (int i = tid; i < NS; i += T) red[i] = 0.0f;
    __syncthreads();
    const int c = (tid % ZQ) * 4;
    if (tid < 32 * ZQ || ZV > 1) {
      atomicAdd(red + c, dbs.x);
      atomicAdd(red + c + 1, dbs.y);
      atomicAdd(red + c + 2, dbs.z);
      atomicAdd(red + c + 3, dbs.w);
    }
    __syncthreads();
    for (int i = tid; i < NS; i += T)
      if (n0 + i < p.N) atomicAdd(p.db + n0 + i, red[i]);
  }
}

template <int WM, int MT, int WN, int NT>
static int launch_wgrad(WgradParams p, cudaStream_t st) {
  constexpr int KS = WM * MT * 16, NS = WN * NT * 8;
  const int ky = (p.K + KS - 1) / KS, nz = (p.N + NS - 1) / NS;
  long long ctas = std::max(1LL, 2LL * sm_count() / ((long long)ky * nz));
  long long rows = (p.M + ctas - 1) / ctas;
  rows = (rows + 31) / 32 * 32;
  if (rows < 256) rows = 256;
  p.rows_per_cta = rows;
  const long long gx = (p.M + rows - 1) / rows;
  if (p.x_split) wgrad_kernel<WM, MT, WN, NT, true><<<dim3((unsigned)gx, (unsigned)ky, (unsigned)nz), 32 * WM * WN, 0, st>>>(p);
  else wgrad_kernel<WM, MT, WN, NT, false><<<dim3((unsigned)gx, (unsigned)ky, (unsigned)nz), 32 * WM * WN, 0, st>>>(p);
  return check_launch("mm_dense_wgrad");
}

// ---------------------------------------------------------------------------------------------------------------
// dgrad:  dX[M, K] = dZ[M, N] W^T  (optionally zeroed where mask <= 0).   N <= 128.
// MMA view: M' = batch rows (one warp per 16 rows), N' = K, K' = N.  B[k' = n][n' = k] = W[k][n]: the Keras kernel is
// already "n'-major with k' contiguous", so a 128-row slab of W sits in shared memory as split-bf16 rows [hi | lo] and B
// fragments come from plain ldmatrix.  The A fragments (dZ rows, split once) stay in registers for the whole slab.
// ---------------------------------------------------------------------------------------------------------------
struct DgradParams {
  const float* dz;
  long long ldz;
  const float* w;  // (K, N) contiguous
  const float* mask;
  long long ldmask;
  float* dx;
  long long lddx;
  long long M;
  int K, N;
  int z_vec2, x_vec2;  // 8-byte loads of dz / 8-byte accesses of mask and dx are legal
  int x_vec4;          // 16-byte accesses of mask and dx are legal: the output leaves through a shared-memory stage
};

constexpr int DG_SLAB = 128;  // output columns (rows of W) per CTA
constexpr int DG_WARPS = 8;
constexpr int DG_STG = 72;  // floats per row of a warp's (16 x 64) output stage (+8: conflict-free 64-bit writes per half warp)

template <int KSTEPS>
__global__ void __launch_bounds__(32 * DG_WARPS, 2) dgrad_kernel(const DgradParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int NP = 16 * KSTEPS;        // padded N
  constexpr int SW = NP * 4 + 16;        // bytes per staged W row: [hi 0..NP | lo 0..NP] + pad
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int k0 = blockIdx.y * DG_SLAB;
  // ---- W slab -> shared memory (split on the fly)
  for (int e = tid; e < DG_SLAB * (NP / 2); e += blockDim.x) {
    const int r = e / (NP / 2), c = (e % (NP / 2)) * 2;
    const int k = k0 + r;
    float a = 0.0f, b = 0.0f;
    if (k < p.K) {
      if (c < p.N) a = __ldg(p.w + (long long)k * p.N + c);
      if (c + 1 < p.N) b = __ldg(p.w + (long long)k * p.N + c + 1);
    }
    uint32_t h, l;
    split_pair(a, b, h, l);
    *reinterpret_cast<uint32_t*>(smem + r * SW + c * 2) = h;
    *reinterpret_cast<uint32_t*>(smem + r * SW + NP * 2 + c * 2) = l;
  }
  __syncthreads();
  // matrices (hi, k' 0-7) (hi, k' 8-15) (lo, k' 0-7) (lo, k' 8-15) of W rows 8*nt + (lane & 7)
  const uint32_t w_lane = (uint32_t)__cvta_generic_to_shared(smem) + (uint32_t)(lane & 7) * SW + (uint32_t)((lane >> 3) & 1) * 16u +
                          (uint32_t)(lane >> 4) * (NP * 2);
  const long long tiles = (p.M + 15) >> 4;
  for (long long tile = (long long)blockIdx.x * DG_WARPS + warp; tile < tiles; tile += (long long)gridDim.x * DG_WARPS) {
    const long long r0 = tile * 16 + g, r1 = r0 + 8;
    const bool v0 = r0 < p.M, v1 = r1 < p.M;
    uint32_t ah[KSTEPS][4], al[KSTEPS][4];
    const float* z0 = p.dz + r0 * p.ldz;
    const float* z1 = p.dz + r1 * p.ldz;
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
      float2 x00 = make_float2(0.f, 0.f), x01 = x00, x10 = x00, x11 = x00;  // (row, k-half)
      const int c0 = 16 * ks + 2 * t, c1 = c0 + 8;
      if (p.z_vec2 && c1 + 1 < p.N) {
        if (v0) {
          x00 = __ldg(reinterpret_cast<const float2*>(z0 + c0));
          x01 = __ldg(reinterpret_cast<const float2*>(z0 + c1));
        }
        if (v1) {
          x10 = __ldg(reinterpret_cast<const float2*>(z1 + c0));
          x11 = __ldg(reinterpret_cast<const float2*>(z1 + c1));
        }
      } else {
        if (v0) {
          if (c0 < p.N) x00.x = __ldg(z0 + c0);
          if (c0 + 1 < p.N) x00.y = __ldg(z0 + c0 + 1);
          if (c1 < p.N) x01.x = __ldg(z0 + c1);
          if (c1 + 1 < p.N) x01.y = __ldg(z0 + c1 + 1);
        }
        if (v1) {
          if (c0 < p.N) x10.x = __ldg(z1 + c0);
          if (c0 + 1 < p.N) x10.y = __ldg(z1 + c0 + 1);
          if (c1 < p.N) x11.x = __ldg(z1 + c1);
          if (c1 + 1 < p.N) x11.y = __ldg(z1 + c1 + 1);
        }
      }
      split_pair(x00.x, x00.y, ah[ks][0], al[ks][0]);
      split_pair(x10.x, x10.y, ah[ks][1], al[ks][1]);
      split_pair(x01.x, x01.y, ah[ks][2], al[ks][2]);
      split_pair(x11.x, x11.y, ah[ks][3], al[ks][3]);
    }
#pragma unroll 1
    for (int ch = 0; ch < DG_SLAB / 64; ++ch) {  // 64 output columns at a time
      if (k0 + ch * 64 >= p.K) break;
      float acc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.0f;
#pragma unroll
      for (int ks = 0; ks < KSTEPS; ++ks) {
#pragma unroll
        for (int n4 = 0; n4 < 8; n4 += 4) {
          uint32_t bh[4][2], bl[4][2];
#pragma unroll
          for (int u = 0; u < 4; ++u)
            ldsm_x4(w_lane + (uint32_t)((ch * 8 + n4 + u) * 8 * SW + ks * 32), bh[u][0], bh[u][1], bl[u][0], bl[u][1]);
#pragma unroll
          for (int u = 0; u < 4; ++u) mma16816(acc[n4 + u], ah[ks], bl[u][0], bl[u][1]);
#pragma unroll
          for (int u = 0; u < 4; ++u) mma16816(acc[n4 + u], al[ks], bh[u][0], bh[u][1]);
#pragma unroll
          for (int u = 0; u < 4; ++u) mma16816(acc[n4 + u], ah[ks], bh[u][0], bh[u][1]);
        }
      }
      if (p.x_vec4) {
        // stage the (16 x 64) tile in shared memory and leave as full rows: 16 lanes x 16 bytes = one 256-byte row segment
        // (the fragment layout gives every lane 8-byte pieces of 8 different rows: 1.1 us per MB of output, measured)
        float* stg = reinterpret_cast<float*>(smem + DG_SLAB * SW) + warp * (16 * DG_STG);
        __syncwarp();
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          *reinterpret_cast<float2*>(stg + g * DG_STG + nt * 8 + 2 * t) = make_float2(acc[nt][0], acc[nt][1]);
          *reinterpret_cast<float2*>(stg + (g + 8) * DG_STG + nt * 8 + 2 * t) = make_float2(acc[nt][2], acc[nt][3]);
        }
        __syncwarp();
        const int c4 = (lane & 15) * 4;
        const int kc = k0 + ch * 64 + c4;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int rr = it * 2 + (lane >> 4);
          const long long r = tile * 16 + rr;
          if (r < p.M && kc < p.K) {
            float4 v = *reinterpret_cast<const float4*>(stg + rr * DG_STG + c4);
            if (kc + 3 < p.K) {
              if (p.mask) {
                const float4 mv = __ldg(reinterpret_cast<const float4*>(p.mask + r * p.ldmask + kc));
                v.x = mv.x > 0.0f ? v.x : 0.0f;
                v.y = mv.y > 0.0f ? v.y : 0.0f;
                v.z = mv.z > 0.0f ? v.z : 0.0f;
                v.w = mv.w > 0.0f ? v.w : 0.0f;
              }
              *reinterpret_cast<float4*>(p.dx + r * p.lddx + kc) = v;
            } else {  // the last, partial group of a row (K not a multiple of 4)
              const float vv[4] = {v.x, v.y, v.z, v.w};
              for (int e = 0; e < 4 && kc + e < p.K; ++e) {
                float a = vv[e];
                if (p.mask) a = __ldg(p.mask + r * p.ldmask + kc + e) > 0.0f ? a : 0.0f;
                p.dx[r * p.lddx + kc + e] = a;
              }
            }
          }
        }
        continue;
      }
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int k = k0 + ch * 64 + nt * 8 + 2 * t;
        if (k >= p.K) continue;
        const bool two = k + 1 < p.K;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long r = h ? r1 : r0;
          if (!(h ? v1 : v0)) continue;
          float a = acc[nt][2 * h], b = acc[nt][2 * h + 1];
          if (p.mask) {
            const float* mrow = p.mask + r * p.ldmask + k;
            if (p.x_vec2 && two) {
              const float2 mv = __ldg(reinterpret_cast<const float2*>(mrow));
              a = mv.x > 0.0f ? a : 0.0f;
              b = mv.y > 0.0f ? b : 0.0f;
            } else {
              a = __ldg(mrow) > 0.0f ? a : 0.0f;
              if (two) b = __ldg(mrow + 1) > 0.0f ? b : 0.0f;
            }
          }
          float* drow = p.dx + r * p.lddx + k;
          if (p.x_vec2 && two) {
            *reinterpret_cast<float2*>(drow) = make_float2(a, b);
          } else {
            drow[0] = a;
            if (two) drow[1] = b;
          }
        }
      }
    }
  }
}

template <int KSTEPS>
static int launch_dgrad(const DgradParams& p, cudaStream_t st) {
  constexpr int NP = 16 * KSTEPS;
  const size_t smem = (size_t)DG_SLAB * (NP * 4 + 16) + (size_t)DG_WARPS * 16 * DG_STG * sizeof(float);
  auto kern = dgrad_kernel<KSTEPS>;
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (smem > 48 * 1024 && (dev < 0 || dev >= 64 || !attr_set[dev])) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("mm_dense_dgrad: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const int ky = (p.K + DG_SLAB - 1) / DG_SLAB;
  const long long tiles = (p.M + 15) / 16;
  long long gx = (tiles + DG_WARPS - 1) / DG_WARPS;
  const long long cap = std::max(1LL, 2LL * sm_count() / ky);
  if (gx > cap) gx = cap;
  kern<<<dim3((unsigned)gx, (unsigned)ky), 32 * DG_WARPS, smem, st>>>(p);
  return check_launch("mm_dense_dgrad");
}

// ---------------------------------------------------------------------------------------------------------------
// DCN-v2 cross network backward, one launch per layer l (x_{l+1} = x0 * z_l + x_l, z_l = x_l W_l + b_l).  With g the
// gradient flowing into x_{l+1} and p = dz_{l+1} W_{l+1}^T the dgrad of the layer above (null for the top layer):
//   g += p (in place);  dz_l = g * x0 (fp32 for the weight gradient, split-bf16 for the transposed-kernel dgrad);
//   acc = g * z_l (first layer) or acc += g * z_l  — the x0 terms of the product rule.
// HBM-bound, one pass: one warp per row (8 rows per CTA, grid-stride over the rows), each lane a 4-column group at a time,
// so no thread divides its flat index by the row width.  Groups of the split padding columns [d, Kp) write zeros.
// ---------------------------------------------------------------------------------------------------------------
struct CrossBwdParams {
  const float* x0;
  const float* z;
  float* g;
  const float* p;
  float* acc;
  float* dz;
  __nv_bfloat16* dz_split;
  long long ldx0, ldz, ldg, ldp, ldacc, lddz;
  long long B;
  int d, Kp, acc_init;
};

// n (1..4) leading floats of a 16-byte aligned group; the missing ones read as 0
__device__ __forceinline__ float4 ld_part4(const float* p, int n) {
  if (n >= 4) return *reinterpret_cast<const float4*>(p);
  float4 v = make_float4(p[0], 0.f, 0.f, 0.f);
  if (n > 1) v.y = p[1];
  if (n > 2) v.z = p[2];
  return v;
}
__device__ __forceinline__ void st_part4(float* p, const float4& v, int n) {
  if (n >= 4) {
    *reinterpret_cast<float4*>(p) = v;
    return;
  }
  p[0] = v.x;
  if (n > 1) p[1] = v.y;
  if (n > 2) p[2] = v.z;
}

constexpr int CB_ROWS = 8;  // rows (warps) per CTA of cross_backward_kernel
__global__ void __launch_bounds__(32 * CB_ROWS) cross_backward_kernel(const CrossBwdParams q) {
  const int Q = q.Kp >> 2;
  const int lane = threadIdx.x & 31;
  for (long long m = (long long)blockIdx.x * CB_ROWS + (threadIdx.x >> 5); m < q.B; m += (long long)gridDim.x * CB_ROWS) {
    for (int qi = lane; qi < Q; qi += 32) {
      const int c = qi * 4;
      const int n = q.d - c;
      float4 dz = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n > 0) {
        float* gp = q.g + m * q.ldg + c;
        float4 g = ld_part4(gp, n);
        if (q.p) {
          const float4 p = ld_part4(q.p + m * q.ldp + c, n);
          g.x += p.x;
          g.y += p.y;
          g.z += p.z;
          g.w += p.w;
          st_part4(gp, g, n);
        }
        const float4 x0 = ld_part4(q.x0 + m * q.ldx0 + c, n);
        const float4 z = ld_part4(q.z + m * q.ldz + c, n);
        dz = make_float4(g.x * x0.x, g.y * x0.y, g.z * x0.z, g.w * x0.w);
        float* ap = q.acc + m * q.ldacc + c;
        float4 a = make_float4(g.x * z.x, g.y * z.y, g.z * z.z, g.w * z.w);
        if (!q.acc_init) {
          const float4 o = ld_part4(ap, n);
          a.x += o.x;
          a.y += o.y;
          a.z += o.z;
          a.w += o.w;
        }
        st_part4(ap, a, n);
        st_part4(q.dz + m * q.lddz + c, dz, n);
      }
      uint32_t h0, l0, h1, l1;
      split_pair(dz.x, dz.y, h0, l0);
      split_pair(dz.z, dz.w, h1, l1);
      __nv_bfloat16* o = q.dz_split + m * (2ll * q.Kp) + c;
      *reinterpret_cast<uint2*>(o) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(o + q.Kp) = make_uint2(l0, l1);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of the concatenated input block x0 = [.. table t's rows at columns [col_t, col_t + D_t) ..]: the sum of the
// addends (B, d) (the cross network's running gradient, its last dgrad, the product-rule terms, a deep branch's input
// gradient) restricted to each table's columns, written straight into that table's contiguous (B, D_t) slice buffer —
// the IndexedSlices values.  Columns of no table (continuous features) are never read.  Offsets are arbitrary (width-1
// continuous columns interleave by sorted name), so the addends are read as scalars; the slices are written as float4.
// blockIdx.y = table.
//
// L2 = true (mm_concat_backward_l2) adds the gradient of the per-table penalty l2_t * sum_b ||x0[b, cols_t]||^2, which
// the reference adds to the loss for every looked-up (pooled) embedding of the batch: slice_t += 2 l2_t x0[b, cols_t].
// Each CTA also writes l2_t times its share of sum ||x0||^2 to partials[blockIdx.y * gridDim.x + blockIdx.x] (a fixed
// order: per-thread sums in grid-stride order, then a fixed shuffle / shared-memory tree), and concat_l2_fold_kernel adds
// the partials in index order into loss[0] (the total) and loss[1] (the regularization term): two runs give the same bits.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CB_MAX_ADD = 4;
constexpr int CB_MAX_SLICES = 64;
struct ConcatBwdParams {
  const float* add[CB_MAX_ADD];
  long long ld[CB_MAX_ADD];
  mm_column_slice s[CB_MAX_SLICES];
  long long B;
  int n_add;
  // L2 only
  float l2[CB_MAX_SLICES];
  const float* x0;
  long long ldx;
  float* partials;
};

template <bool L2>
__global__ void __launch_bounds__(256) concat_backward_kernel(const __grid_constant__ ConcatBwdParams q) {
  const mm_column_slice& s = q.s[blockIdx.y];
  const int Q = s.width >> 2;
  const long long total = q.B * Q;
  float sq = 0.f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long m = e / Q;
    const int c = (int)(e - m * Q) * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (int a = 0; a < q.n_add; ++a) {
      const float* src = q.add[a] + m * q.ld[a] + s.col + c;
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] += src[j];
    }
    if constexpr (L2) {
      const float two_l2 = 2.f * q.l2[blockIdx.y];
      const float* x = q.x0 + m * q.ldx + s.col + c;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xj = x[j];
        v[j] += two_l2 * xj;
        sq += xj * xj;
      }
    }
    *reinterpret_cast<float4*>(s.dst + m * s.dst_stride + c) = make_float4(v[0], v[1], v[2], v[3]);
  }
  if constexpr (L2) {
    __shared__ float red[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += red[w];
      q.partials[(long long)blockIdx.y * gridDim.x + blockIdx.x] = q.l2[blockIdx.y] * t;
    }
  }
}

__global__ void __launch_bounds__(256) concat_l2_fold_kernel(const float* __restrict__ partials, int n, float* __restrict__ loss) {
  __shared__ double red[256];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) v += partials[i];
  red[threadIdx.x] = v;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float reg = (float)red[0];
    loss[0] += reg;
    loss[1] += reg;
  }
}

}  // namespace trn
}  // namespace mm

extern "C" {

int mm_cross_backward(const float* x0, int64_t x0_stride, const float* z, int64_t z_stride, float* g, int64_t g_stride,
                      const float* p, int64_t p_stride, float* acc, int64_t acc_stride, int acc_init, int64_t B, int d, float* dz,
                      int64_t dz_stride, void* dz_split, int Kp, void* stream) {
  using namespace mm::trn;
  MM_REQUIRE(x0 && z && g && acc && dz && dz_split && B >= 0 && d >= 1, MM_ERR_ARG, "mm_cross_backward: null pointer or d < 1");
  MM_REQUIRE(Kp == mm_tc_padded_k(d), MM_ERR_ARG, "mm_cross_backward: Kp must be mm_tc_padded_k(d)=%d", mm_tc_padded_k(d));
  MM_REQUIRE(x0_stride >= d && z_stride >= d && g_stride >= d && acc_stride >= d && dz_stride >= d && (!p || p_stride >= d), MM_ERR_ARG,
             "mm_cross_backward: a row stride is < d");
  MM_REQUIRE(((x0_stride | z_stride | g_stride | acc_stride | dz_stride | (p ? p_stride : 0)) & 3) == 0, MM_ERR_ALIGN,
             "mm_cross_backward: row strides must be multiples of 4");
  MM_REQUIRE((((uintptr_t)x0 | (uintptr_t)z | (uintptr_t)g | (uintptr_t)p | (uintptr_t)acc | (uintptr_t)dz | (uintptr_t)dz_split) & 15) == 0,
             MM_ERR_ALIGN, "mm_cross_backward: every buffer must be 16-byte aligned");
  if (B == 0) return MM_OK;
  CrossBwdParams q;
  memset(&q, 0, sizeof(q));
  q.x0 = x0;
  q.z = z;
  q.g = g;
  q.p = p;
  q.acc = acc;
  q.dz = dz;
  q.dz_split = (__nv_bfloat16*)dz_split;
  q.ldx0 = x0_stride;
  q.ldz = z_stride;
  q.ldg = g_stride;
  q.ldp = p_stride;
  q.ldacc = acc_stride;
  q.lddz = dz_stride;
  q.B = B;
  q.d = d;
  q.Kp = Kp;
  q.acc_init = acc_init ? 1 : 0;
  long long blocks = (B + CB_ROWS - 1) / CB_ROWS;
  const long long cap = 16LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  cross_backward_kernel<<<(unsigned)blocks, 32 * CB_ROWS, 0, (cudaStream_t)stream>>>(q);
  return mm::check_launch("mm_cross_backward");
}

// The checks both concat backward entry points share, and their parameters; *blocks = the grid's x extent (0 when B == 0).
static int concat_backward_params(const char* fn, const float* const* addends_host, const int64_t* addend_strides_host,
                                  int n_addends, int64_t B, int d, const mm_column_slice* slices_host, int n_slices,
                                  long long max_blocks, mm::trn::ConcatBwdParams& q, long long* blocks) {
  using namespace mm::trn;
  MM_REQUIRE(addends_host && addend_strides_host && slices_host && B >= 0 && d >= 1, MM_ERR_ARG, "%s: null pointer or d < 1", fn);
  MM_REQUIRE(n_addends >= 1 && n_addends <= CB_MAX_ADD, MM_ERR_ARG, "%s: n_addends=%d outside [1, %d]", fn, n_addends, CB_MAX_ADD);
  MM_REQUIRE(n_slices >= 1 && n_slices <= CB_MAX_SLICES, MM_ERR_ARG, "%s: n_slices=%d outside [1, %d]", fn, n_slices, CB_MAX_SLICES);
  memset(&q, 0, sizeof(q));
  for (int a = 0; a < n_addends; ++a) {
    MM_REQUIRE(addends_host[a] && addend_strides_host[a] >= d, MM_ERR_ARG, "%s: addend %d: null or stride < d", fn, a);
    q.add[a] = addends_host[a];
    q.ld[a] = addend_strides_host[a];
  }
  int qmax = 0;
  for (int t = 0; t < n_slices; ++t) {
    const mm_column_slice& s = slices_host[t];
    MM_REQUIRE(s.dst && s.width >= 4 && (s.width & 3) == 0 && s.col >= 0 && (int64_t)s.col + s.width <= d, MM_ERR_ARG,
               "%s: slice %d: null destination, width not a positive multiple of 4, or columns outside [0, d)", fn, t);
    MM_REQUIRE(s.dst_stride >= s.width && (s.dst_stride & 3) == 0 && ((uintptr_t)s.dst & 15) == 0, MM_ERR_ALIGN,
               "%s: slice %d: destination must be 16-byte aligned with a row stride >= width and a multiple of 4", fn, t);
    q.s[t] = s;
    if (s.width / 4 > qmax) qmax = s.width / 4;
  }
  q.B = B;
  q.n_add = n_addends;
  *blocks = (B * qmax + 255) / 256;
  if (*blocks > max_blocks) *blocks = max_blocks;
  return MM_OK;
}

int mm_concat_backward(const float* const* addends_host, const int64_t* addend_strides_host, int n_addends, int64_t B, int d,
                       const mm_column_slice* slices_host, int n_slices, void* stream) {
  using namespace mm::trn;
  ConcatBwdParams q;
  long long blocks = 0;
  const int rc = concat_backward_params("mm_concat_backward", addends_host, addend_strides_host, n_addends, B, d, slices_host,
                                        n_slices, 4LL * mm::sm_count(), q, &blocks);
  if (rc != MM_OK) return rc;
  if (B == 0) return MM_OK;
  concat_backward_kernel<false><<<dim3((unsigned)blocks, (unsigned)n_slices), 256, 0, (cudaStream_t)stream>>>(q);
  return mm::check_launch("mm_concat_backward");
}

int mm_concat_backward_l2(const float* const* addends_host, const int64_t* addend_strides_host, int n_addends, int64_t B, int d,
                          const mm_column_slice* slices_host, int n_slices, const float* x0, int64_t x0_stride,
                          const float* l2_host, float* partials, int64_t n_partials, float* loss, void* stream) {
  using namespace mm::trn;
  ConcatBwdParams q;
  long long blocks = 0;
  const long long cap = std::min(4LL * mm::sm_count(), (long long)MM_CONCAT_L2_CTAS);
  const int rc = concat_backward_params("mm_concat_backward_l2", addends_host, addend_strides_host, n_addends, B, d, slices_host,
                                        n_slices, cap, q, &blocks);
  if (rc != MM_OK) return rc;
  MM_REQUIRE(x0 && x0_stride >= d && l2_host && partials && loss, MM_ERR_ARG,
             "mm_concat_backward_l2: null x0 / l2 / partials / loss, or x0_stride < d");
  MM_REQUIRE(n_partials >= (int64_t)n_slices * MM_CONCAT_L2_CTAS, MM_ERR_ARG,
             "mm_concat_backward_l2: partials must hold n_slices * %d = %lld floats, got %lld", MM_CONCAT_L2_CTAS,
             (long long)n_slices * MM_CONCAT_L2_CTAS, (long long)n_partials);
  for (int t = 0; t < n_slices; ++t) {
    MM_REQUIRE(l2_host[t] >= 0.f && l2_host[t] <= 3.0e38f, MM_ERR_ARG, "mm_concat_backward_l2: l2[%d] must be finite and >= 0", t);
    q.l2[t] = l2_host[t];
  }
  q.x0 = x0;
  q.ldx = x0_stride;
  q.partials = partials;
  if (B == 0) return MM_OK;
  concat_backward_kernel<true><<<dim3((unsigned)blocks, (unsigned)n_slices), 256, 0, (cudaStream_t)stream>>>(q);
  concat_l2_fold_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(partials, (int)(blocks * n_slices), loss);
  return mm::check_launch("mm_concat_backward_l2");
}

int mm_heads_fwd_bwd(const float* x, int64_t M, int K, int64_t x_stride, int H, const float* w, const float* bias,
                     const int* loss_kind, const float* loss_weight, const void* const* targets, const int* target_dtypes,
                     const float* const* sample_weights, float* logits, float* loss, float* dx, int64_t dx_stride,
                     int mask_relu, float* dw, float* db, void* stream) {
  using namespace mm::trn;
  MM_REQUIRE(x && w && loss_kind && M >= 0 && K >= 1 && x_stride >= K, MM_ERR_ARG, "mm_heads_fwd_bwd: null pointer or bad K / stride");
  MM_REQUIRE(H >= 1 && H <= HEAD_MAX, MM_ERR_UNSUPPORTED, "mm_heads_fwd_bwd: H=%d is not in 1..%d", H, HEAD_MAX);
  MM_REQUIRE(K <= HEAD_KMAX, MM_ERR_UNSUPPORTED, "mm_heads_fwd_bwd: K=%d > %d", K, HEAD_KMAX);
  const bool train = targets != nullptr;
  MM_REQUIRE(train || logits, MM_ERR_ARG, "mm_heads_fwd_bwd: forward only (targets null) needs logits");
  MM_REQUIRE(!train || (loss_weight && target_dtypes && loss), MM_ERR_ARG,
             "mm_heads_fwd_bwd: training needs loss_weight, target_dtypes and loss");
  MM_REQUIRE(!train || !dx || dx_stride >= K, MM_ERR_ARG, "mm_heads_fwd_bwd: dx_stride < K");
  HeadParams p;
  memset(&p, 0, sizeof(p));
  for (int h = 0; h < H; ++h) {
    MM_REQUIRE(loss_kind[h] == MM_LOSS_BCE || loss_kind[h] == MM_LOSS_MSE, MM_ERR_ARG, "mm_heads_fwd_bwd: head %d: bad loss kind %d",
               h, loss_kind[h]);
    p.kind[h] = loss_kind[h];
    if (train) {
      MM_REQUIRE(targets[h], MM_ERR_ARG, "mm_heads_fwd_bwd: head %d: null targets", h);
      MM_REQUIRE(target_dtypes[h] >= MM_I32 && target_dtypes[h] <= MM_F64, MM_ERR_ARG, "mm_heads_fwd_bwd: head %d: bad target dtype", h);
      p.y[h] = targets[h];
      p.y_dtype[h] = target_dtypes[h];
      p.lw[h] = loss_weight[h];
      p.sample_w[h] = sample_weights ? sample_weights[h] : nullptr;
    }
  }
  if (M == 0) return MM_OK;
  p.x = x;
  p.ldx = x_stride;
  p.M = M;
  p.K = K;
  p.w = w;
  p.bias = bias;
  p.inv_m = 1.0f / (float)M;
  p.logits = logits;
  if (train) {
    p.loss = loss;
    p.loss_heads = loss + 1;
    p.dx = dx;
    p.lddx = dx_stride;
    p.mask_relu = mask_relu;
    p.dw = dw;
    p.db = db;
  }
  run_heads(p, H, train, (cudaStream_t)stream);
  return mm::check_launch("mm_heads_fwd_bwd");
}

static int wgrad_dispatch(mm::trn::WgradParams p, void* stream) {
  using namespace mm::trn;
  cudaStream_t st = (cudaStream_t)stream;
  const int K = p.K, N = p.N;
  const int ks = K > 64 ? 128 : K > 16 ? 64 : 16;
  const int ns = N > 64 ? 128 : N > 32 ? 64 : 32;
#define MM_WG(KS_, NS_, WM, MT, WN, NT) \
  if (ks == KS_ && ns == NS_) return launch_wgrad<WM, MT, WN, NT>(p, st);
  MM_WG(128, 128, 4, 2, 4, 4) MM_WG(128, 64, 4, 2, 2, 4) MM_WG(128, 32, 4, 2, 2, 2)
  MM_WG(64, 128, 2, 2, 4, 4) MM_WG(64, 64, 2, 2, 4, 2) MM_WG(64, 32, 4, 1, 2, 2)
  MM_WG(16, 128, 1, 1, 8, 2) MM_WG(16, 64, 1, 1, 8, 1) MM_WG(16, 32, 1, 1, 4, 1)
#undef MM_WG
  return MM_ERR_UNSUPPORTED;
}

int mm_dense_wgrad(const float* x, int64_t M, int K, int64_t x_stride, const float* dz, int N, int64_t dz_stride, float* dw,
                   float* db, void* stream) {
  using namespace mm::trn;
  MM_REQUIRE(x && dz && dw && M >= 0 && K >= 1 && N >= 1 && x_stride >= K && dz_stride >= N, MM_ERR_ARG,
             "mm_dense_wgrad: null pointer or bad shape / stride");
  if (M == 0) return MM_OK;
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.x = x;
  p.ldx = x_stride;
  p.dz = dz;
  p.ldz = dz_stride;
  p.M = M;
  p.K = K;
  p.N = N;
  p.dw = dw;
  p.db = db;
  p.x_vec = ((x_stride & 3) == 0 && ((uintptr_t)x & 15) == 0) ? 1 : 0;
  p.z_vec = ((dz_stride & 3) == 0 && ((uintptr_t)dz & 15) == 0) ? 1 : 0;
  return wgrad_dispatch(p, stream);
}

int mm_dense_wgrad_split(const void* x_split, int64_t M, int K, int Kp, const float* dz, int N, int64_t dz_stride, float* dw,
                         float* db, void* stream) {
  using namespace mm::trn;
  MM_REQUIRE(x_split && dz && dw && M >= 0 && K >= 1 && N >= 1 && dz_stride >= N, MM_ERR_ARG, "mm_dense_wgrad_split: null pointer or bad shape");
  MM_REQUIRE(Kp == mm_tc_padded_k(K) && ((uintptr_t)x_split & 15) == 0, MM_ERR_ARG,
             "mm_dense_wgrad_split: Kp must be mm_tc_padded_k(K)=%d and x_split 16-byte aligned", mm_tc_padded_k(K));
  if (M == 0) return MM_OK;
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.x_split = (const __nv_bfloat16*)x_split;
  p.Kp = Kp;
  p.dz = dz;
  p.ldz = dz_stride;
  p.M = M;
  p.K = K;
  p.N = N;
  p.dw = dw;
  p.db = db;
  p.z_vec = ((dz_stride & 3) == 0 && ((uintptr_t)dz & 15) == 0) ? 1 : 0;
  return wgrad_dispatch(p, stream);
}

int mm_dense_dgrad(const float* dz, int64_t M, int N, int64_t dz_stride, const float* w, int K, const float* mask,
                   int64_t mask_stride, float* dx, int64_t dx_stride, void* stream) {
  using namespace mm::trn;
  MM_REQUIRE(dz && w && dx && M >= 0 && K >= 1 && N >= 1 && dz_stride >= N && dx_stride >= K, MM_ERR_ARG,
             "mm_dense_dgrad: null pointer or bad shape / stride");
  MM_REQUIRE(!mask || mask_stride >= K, MM_ERR_ARG, "mm_dense_dgrad: mask_stride < K");
  MM_REQUIRE(N <= 128, MM_ERR_UNSUPPORTED, "mm_dense_dgrad: N=%d > 128 (run the forward GEMM on the transposed kernel instead)", N);
  if (M == 0) return MM_OK;
  DgradParams p;
  memset(&p, 0, sizeof(p));
  p.dz = dz;
  p.ldz = dz_stride;
  p.w = w;
  p.mask = mask;
  p.ldmask = mask_stride;
  p.dx = dx;
  p.lddx = dx_stride;
  p.M = M;
  p.K = K;
  p.N = N;
  p.z_vec2 = ((dz_stride & 1) == 0 && ((uintptr_t)dz & 7) == 0) ? 1 : 0;
  p.x_vec2 = ((dx_stride & 1) == 0 && ((uintptr_t)dx & 7) == 0 && (!mask || ((mask_stride & 1) == 0 && ((uintptr_t)mask & 7) == 0))) ? 1 : 0;
  p.x_vec4 = ((dx_stride & 3) == 0 && ((uintptr_t)dx & 15) == 0 && (!mask || ((mask_stride & 3) == 0 && ((uintptr_t)mask & 15) == 0))) ? 1 : 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (N <= 32) return launch_dgrad<2>(p, st);
  if (N <= 64) return launch_dgrad<4>(p, st);
  return launch_dgrad<8>(p, st);
}

}  // extern "C"
