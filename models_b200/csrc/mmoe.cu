// MMoE gates, expert mixture and output heads (MMOEBlock, blocks/experts.py:37-208; OutputBlock, outputs/block.py:32-190).
//
//   mm_mmoe_heads_fwd_bwd  everything after the experts' last layer and the gate logits, in ONE pass over the batch:
//       p_t = softmax(L_t / T)            (E gate weights of task t)
//       m_t = sum_e p_t,e X_e             (the gate's mixture of the E expert outputs, U wide; never written)
//       z_t = m_t . w_t + b_t             (task t's Dense(1))
//     with targets: the loss and the backward
//       dz_t as mm_heads_fwd_bwd;  dm_t = dz_t w_t;  dg_t,e = <dm_t, X_e> = dz_t <w_t, X_e>
//       dL_t = p_t (dg_t - <p_t, dg_t>) / T;  dX_e = sum_t p_t,e dm_t (relu mask from X);  dW_t += m_t dz_t, db_t += dz_t
//     without: the activated predictions (the |z|-stable sigmoid of mm_heads_fwd_bwd, or z).
//   mm_mmoe_mix_fwd / mm_mmoe_mix_bwd  the same gates and mixture when task towers follow: m_t (H, B, U) and its split-bf16
//     operand are written, p (B, H E) is saved; the backward takes dm (H, B, U) to dX and dL.
//   mm_mmoe_task_heads_fwd_bwd  H Dense(K -> 1) heads where head t reads its own input x_t (its tower's output), with the
//     losses and backward of mm_heads_fwd_bwd.
//
// Layout: one warp per sample.  Lane j owns the columns j + 32 c (c < C) of every expert; the gate weights of the sample
// (H E <= 128 values) and <w_t, X_e> live in the warp's shared-memory row.  w and dw stay in registers; per CTA one
// shared-memory sum and one atomic per value, as in the heads kernel.
#include <cstring>

#include "mm_common.cuh"
#include "warp_mma.cuh"

namespace mm {
namespace moe {

constexpr int HMAX = 8;    // tasks
constexpr int EMAX = 16;   // experts
constexpr int UMAX = 256;  // expert width: 8 columns per lane
constexpr int WARPS = 8;   // 256 threads per CTA

struct Params {
  const float* x;  // (B, E U)
  long long ldx;
  const float* gl[HMAX];  // gate logits of task t: (B, E)
  long long ldgl[HMAX];
  float* dgl[HMAX];
  long long lddgl[HMAX];
  long long B;
  int E, U, H;
  float inv_t;
  const float* w;     // (U, H) Keras layout
  const float* bias;  // (H,) or null
  const void* y[HMAX];
  int y_dtype[HMAX];
  int kind[HMAX];
  float lw[HMAX];
  const float* sample_w[HMAX];
  float inv_m;
  float* logits;  // (H, B)
  float* loss;
  float* loss_heads;
  float* dx;
  long long lddx;
  int mask_relu;
  float* dw;  // (U, H) accumulated
  float* db;  // (H,) accumulated
};

// the gate soft-max of sample m into sp[t E + e] (the warp's shared row); ends with the row visible to the whole warp
__device__ __forceinline__ void gate_softmax(const float* const* gl, const long long* ldgl, long long m, int E, int H, float inv_t,
                                             float* sp, int lane) {
  for (int j = lane; j < H * E; j += 32) {
    const int t = j / E;
    sp[j] = gl[t][m * ldgl[t] + (j - t * E)] * inv_t;
  }
  __syncwarp();
  if (lane < H) {
    float* q = sp + lane * E;
    float mx = q[0];
    for (int e = 1; e < E; ++e) mx = fmaxf(mx, q[e]);
    float s = 0.0f;
    for (int e = 0; e < E; ++e) {
      q[e] = expf(q[e] - mx);
      s += q[e];
    }
    const float r = 1.0f / s;
    for (int e = 0; e < E; ++e) q[e] *= r;
  }
  __syncwarp();
}

// NH: H rounded up to a power of two (tasks t >= H are skipped at run time); C: columns per lane
template <int NH, int C, bool TRAIN>
__global__ void __launch_bounds__(32 * WARPS, 1) mmoe_heads_kernel(const Params p) {
  __shared__ float s_p[WARPS][HMAX * EMAX];  // gate weights p_t,e of the warp's sample, at t E + e
  __shared__ float s_a[WARPS][HMAX * EMAX];  // <w_t, X_e>
  __shared__ float s_dz[WARPS][HMAX];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long warp = (long long)blockIdx.x * WARPS + wid;
  const long long n_warps = (long long)gridDim.x * WARPS;
  const int E = p.E, U = p.U, H = p.H;
  float w[NH][C], dw[NH][C], b[NH], loss[NH], db[NH];
#pragma unroll
  for (int t = 0; t < NH; ++t) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const int k = lane + 32 * c;
      w[t][c] = (t < H && k < U) ? p.w[k * H + t] : 0.0f;
      dw[t][c] = 0.0f;
    }
    b[t] = (t < H && p.bias) ? p.bias[t] : 0.0f;
    loss[t] = db[t] = 0.0f;
  }
  float* sp = s_p[wid];
  float* sa = s_a[wid];
  for (long long m = warp; m < p.B; m += n_warps) {
    gate_softmax(p.gl, p.ldgl, m, E, H, p.inv_t, sp, lane);  // lane t < H normalises task t's E logits
    // mixture m_t (registers) and, for the backward, <w_t, X_e>
    float mix[NH][C];
#pragma unroll
    for (int t = 0; t < NH; ++t)
#pragma unroll
      for (int c = 0; c < C; ++c) mix[t][c] = 0.0f;
    const float* xr = p.x + m * p.ldx;
    for (int e = 0; e < E; ++e) {
      float x[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        x[c] = k < U ? __ldg(xr + e * U + k) : 0.0f;
      }
#pragma unroll
      for (int t = 0; t < NH; ++t) {
        if (t >= H) break;
        const float pe = sp[t * E + e];
        float a = 0.0f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
          mix[t][c] = fmaf(pe, x[c], mix[t][c]);
          if (TRAIN) a = fmaf(w[t][c], x[c], a);
        }
        if (TRAIN) {
          a = warp_sum(a);
          if (lane == 0) sa[t * E + e] = a;
        }
      }
    }
    // heads
#pragma unroll
    for (int t = 0; t < NH; ++t) {
      if (t >= H) break;
      float dot = 0.0f;
#pragma unroll
      for (int c = 0; c < C; ++c) dot = fmaf(mix[t][c], w[t][c], dot);
      const float z = warp_sum(dot) + b[t];
      if (!TRAIN) {
        if (lane == 0) p.logits[t * p.B + m] = head_pred(p.kind[t], z);
        continue;
      }
      const float y = load_as_f32(p.y[t], m, p.y_dtype[t]);
      const float sw = p.sample_w[t] ? p.sample_w[t][m] : 1.0f;
      float l, g;
      head_loss(p.kind[t], z, y, l, g);
      float dz = g * sw * p.inv_m;
      dz *= p.lw[t];  // exact for lambda = 1
#pragma unroll
      for (int c = 0; c < C; ++c) dw[t][c] = fmaf(mix[t][c], dz, dw[t][c]);
      if (lane == 0) {
        loss[t] += l * sw * p.inv_m;
        db[t] += dz;
        if (p.logits) p.logits[t * p.B + m] = z;
        s_dz[wid][t] = dz;
      }
    }
    if (!TRAIN) {
      __syncwarp();  // the next sample's logits overwrite sp
      continue;
    }
    __syncwarp();
    // gate backward: lane t < H, dg_t,e = dz_t <w_t, X_e>.  dg is rounded once (__fmul_rn, never contracted into an FMA)
    // so that s and dg - s see the same value: with one expert dg - s is then exactly 0, as the soft-max's gradient is.
    if (lane < H) {
      const float dz = s_dz[wid][lane];
      const float* q = sp + lane * E;
      const float* a = sa + lane * E;
      float s = 0.0f;
      for (int e = 0; e < E; ++e) s = fmaf(q[e], __fmul_rn(dz, a[e]), s);
      float* o = p.dgl[lane] + m * p.lddgl[lane];
      for (int e = 0; e < E; ++e) o[e] = q[e] * (__fmul_rn(dz, a[e]) - s) * p.inv_t;
    }
    // expert backward: dX_e = sum_t p_t,e dz_t w_t
    float dzr[NH];
#pragma unroll
    for (int t = 0; t < NH; ++t) dzr[t] = t < H ? s_dz[wid][t] : 0.0f;
    float* dxr = p.dx + m * p.lddx;
    for (int e = 0; e < E; ++e) {
      float ge[NH];
#pragma unroll
      for (int t = 0; t < NH; ++t) ge[t] = t < H ? sp[t * E + e] * dzr[t] : 0.0f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        if (k >= U) continue;
        float d = 0.0f;
#pragma unroll
        for (int t = 0; t < NH; ++t) d = fmaf(ge[t], w[t][c], d);
        if (p.mask_relu && !(__ldg(xr + e * U + k) > 0.0f)) d = 0.0f;
        dxr[e * U + k] = d;
      }
    }
    __syncwarp();  // the next sample overwrites sp / sa / s_dz
  }
  if (!TRAIN) return;
  // block-level reduction of dw / db / loss before the atomics, one task at a time
  __shared__ float red[WARPS][UMAX + 2];
#pragma unroll
  for (int t = 0; t < NH; ++t) {
    if (t >= H) break;
    if (t > 0) __syncthreads();  // the previous task's sums have been read
#pragma unroll
    for (int c = 0; c < C; ++c) red[wid][lane + 32 * c] = dw[t][c];
    if (lane == 0) {
      red[wid][UMAX] = db[t];
      red[wid][UMAX + 1] = loss[t];
    }
    __syncthreads();
    for (int k = threadIdx.x; k < UMAX + 2; k += blockDim.x) {
      if (k >= U && k < UMAX) continue;
      float s = 0.0f;
      for (int i = 0; i < WARPS; ++i) s += red[i][k];
      if (k < U) {
        if (p.dw) atomicAdd(p.dw + k * H + t, s);
      } else if (k == UMAX) {
        if (p.db) atomicAdd(p.db + t, s);
      } else {
        atomicAdd(p.loss, p.lw[t] * s);
        atomicAdd(p.loss_heads + t, s);
      }
    }
  }
}


// ---- mixture forward / backward for the task-tower path --------------------------------------------------------------
struct MixParams {
  const float* x;
  long long ldx;
  const float* gl[HMAX];
  long long ldgl[HMAX];
  float* dgl[HMAX];
  long long lddgl[HMAX];
  long long B;
  int E, U, H, Kp;
  float inv_t;
  float* p;  // (B, H E) saved gate weights
  float* m;  // (H, B, U)
  __nv_bfloat16* m_split;  // (H, B, 2 Kp) or null
  const float* dm;         // (H, B, U)
  float* dx;
  long long lddx;
  int mask_relu;
};

template <int NH, int C>
__global__ void __launch_bounds__(32 * WARPS) mmoe_mix_fwd_kernel(const MixParams q) {
  __shared__ float s_p[WARPS][HMAX * EMAX];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int E = q.E, U = q.U, H = q.H;
  float* sp = s_p[wid];
  for (long long m = (long long)blockIdx.x * WARPS + wid; m < q.B; m += (long long)gridDim.x * WARPS) {
    gate_softmax(q.gl, q.ldgl, m, E, H, q.inv_t, sp, lane);
    for (int j = lane; j < H * E; j += 32) q.p[m * H * E + j] = sp[j];
    float mix[NH][C];
#pragma unroll
    for (int t = 0; t < NH; ++t)
#pragma unroll
      for (int c = 0; c < C; ++c) mix[t][c] = 0.0f;
    const float* xr = q.x + m * q.ldx;
    for (int e = 0; e < E; ++e) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        const float xv = k < U ? __ldg(xr + e * U + k) : 0.0f;
#pragma unroll
        for (int t = 0; t < NH; ++t)
          if (t < H) mix[t][c] = fmaf(sp[t * E + e], xv, mix[t][c]);
      }
    }
#pragma unroll
    for (int t = 0; t < NH; ++t) {
      if (t >= H) break;
      float* mr = q.m + ((long long)t * q.B + m) * U;
      __nv_bfloat16* sr = q.m_split ? q.m_split + ((long long)t * q.B + m) * (2ll * q.Kp) : nullptr;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        if (k >= U) continue;
        mr[k] = mix[t][c];
        if (sr) {
          __nv_bfloat16 hi, lo;
          split_bf16(mix[t][c], hi, lo);
          sr[k] = hi;
          sr[q.Kp + k] = lo;
        }
      }
      if (sr)
        for (int k = U + lane; k < q.Kp; k += 32) sr[k] = sr[q.Kp + k] = __float2bfloat16_rn(0.0f);
    }
    __syncwarp();  // the next sample overwrites sp
  }
}

template <int NH, int C>
__global__ void __launch_bounds__(32 * WARPS) mmoe_mix_bwd_kernel(const MixParams q) {
  __shared__ float s_p[WARPS][HMAX * EMAX];
  __shared__ float s_g[WARPS][HMAX * EMAX];  // dg_t,e = <dm_t, X_e>
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int E = q.E, U = q.U, H = q.H;
  float* sp = s_p[wid];
  float* sg = s_g[wid];
  for (long long m = (long long)blockIdx.x * WARPS + wid; m < q.B; m += (long long)gridDim.x * WARPS) {
    for (int j = lane; j < H * E; j += 32) sp[j] = q.p[m * H * E + j];
    float dm[NH][C];
#pragma unroll
    for (int t = 0; t < NH; ++t)
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        dm[t][c] = (t < H && k < U) ? q.dm[((long long)t * q.B + m) * U + k] : 0.0f;
      }
    __syncwarp();
    const float* xr = q.x + m * q.ldx;
    float* dxr = q.dx + m * q.lddx;
    for (int e = 0; e < E; ++e) {
      float x[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        x[c] = k < U ? __ldg(xr + e * U + k) : 0.0f;
      }
#pragma unroll
      for (int t = 0; t < NH; ++t) {
        if (t >= H) break;
        float a = 0.0f;
#pragma unroll
        for (int c = 0; c < C; ++c) a = fmaf(dm[t][c], x[c], a);
        a = warp_sum(a);
        if (lane == 0) sg[t * E + e] = a;
      }
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        if (k >= U) continue;
        float d = 0.0f;
#pragma unroll
        for (int t = 0; t < NH; ++t)
          if (t < H) d = fmaf(sp[t * E + e], dm[t][c], d);
        if (q.mask_relu && !(x[c] > 0.0f)) d = 0.0f;
        dxr[e * U + k] = d;
      }
    }
    __syncwarp();
    if (lane < H) {
      const float* pp = sp + lane * E;
      const float* g = sg + lane * E;
      float s = 0.0f;
      for (int e = 0; e < E; ++e) s = fmaf(pp[e], g[e], s);
      float* o = q.dgl[lane] + m * q.lddgl[lane];
      for (int e = 0; e < E; ++e) o[e] = pp[e] * (g[e] - s) * q.inv_t;
    }
    __syncwarp();
  }
}

// ---- heads with one input per task --------------------------------------------------------------------------------
struct TaskHeadParams {
  const float* x[HMAX];
  long long ldx[HMAX];
  float* dx[HMAX];
  long long lddx[HMAX];
  long long B;
  int K, H;
  const float* w;     // (K, H)
  const float* bias;  // (H,) or null
  const void* y[HMAX];
  int y_dtype[HMAX];
  int kind[HMAX];
  float lw[HMAX];
  const float* sample_w[HMAX];
  float inv_m;
  float* logits;
  float* loss;
  float* loss_heads;
  int mask_relu;
  float* dw;
  float* db;
};

template <int NH, int C, bool TRAIN>
__global__ void __launch_bounds__(32 * WARPS, 1) task_heads_kernel(const TaskHeadParams p) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int K = p.K, H = p.H;
  float w[NH][C], dw[NH][C], b[NH], loss[NH], db[NH];
#pragma unroll
  for (int t = 0; t < NH; ++t) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const int k = lane + 32 * c;
      w[t][c] = (t < H && k < K) ? p.w[k * H + t] : 0.0f;
      dw[t][c] = 0.0f;
    }
    b[t] = (t < H && p.bias) ? p.bias[t] : 0.0f;
    loss[t] = db[t] = 0.0f;
  }
  for (long long m = (long long)blockIdx.x * WARPS + wid; m < p.B; m += (long long)gridDim.x * WARPS) {
#pragma unroll
    for (int t = 0; t < NH; ++t) {
      if (t >= H) break;
      float x[C];
      float dot = 0.0f;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        x[c] = k < K ? p.x[t][m * p.ldx[t] + k] : 0.0f;
        dot = fmaf(x[c], w[t][c], dot);
      }
      const float z = warp_sum(dot) + b[t];
      if (!TRAIN) {
        if (lane == 0) p.logits[t * p.B + m] = head_pred(p.kind[t], z);
        continue;
      }
      const float y = load_as_f32(p.y[t], m, p.y_dtype[t]);
      const float sw = p.sample_w[t] ? p.sample_w[t][m] : 1.0f;
      float l, g;
      head_loss(p.kind[t], z, y, l, g);
      float dz = g * sw * p.inv_m;
      dz *= p.lw[t];  // exact for lambda = 1
      if (lane == 0) {
        loss[t] += l * sw * p.inv_m;
        db[t] += dz;
        if (p.logits) p.logits[t * p.B + m] = z;
      }
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int k = lane + 32 * c;
        dw[t][c] = fmaf(x[c], dz, dw[t][c]);
        if (k < K) p.dx[t][m * p.lddx[t] + k] = (!p.mask_relu || x[c] > 0.0f) ? dz * w[t][c] : 0.0f;
      }
    }
  }
  if (!TRAIN) return;
  __shared__ float red[WARPS][UMAX + 2];
#pragma unroll
  for (int t = 0; t < NH; ++t) {
    if (t >= H) break;
    if (t > 0) __syncthreads();
#pragma unroll
    for (int c = 0; c < C; ++c) red[wid][lane + 32 * c] = dw[t][c];
    if (lane == 0) {
      red[wid][UMAX] = db[t];
      red[wid][UMAX + 1] = loss[t];
    }
    __syncthreads();
    for (int k = threadIdx.x; k < UMAX + 2; k += blockDim.x) {
      if (k >= K && k < UMAX) continue;
      float s = 0.0f;
      for (int i = 0; i < WARPS; ++i) s += red[i][k];
      if (k < K) {
        if (p.dw) atomicAdd(p.dw + k * H + t, s);
      } else if (k == UMAX) {
        if (p.db) atomicAdd(p.db + t, s);
      } else {
        atomicAdd(p.loss, p.lw[t] * s);
        atomicAdd(p.loss_heads + t, s);
      }
    }
  }
}

// dispatch on H (rounded up to a power of two) and on the columns per lane of a width n <= 256
#define MM_MOE_DISPATCH(H_, N_, LAUNCH)                                      \
  do {                                                                       \
    const int nh_ = (H_) == 1 ? 1 : (H_) == 2 ? 2 : (H_) <= 4 ? 4 : 8;       \
    const int c_ = (N_) <= 32 ? 1 : (N_) <= 64 ? 2 : (N_) <= 128 ? 4 : 8;    \
    if (nh_ == 1 && c_ == 1) LAUNCH(1, 1); else if (nh_ == 1 && c_ == 2) LAUNCH(1, 2); \
    else if (nh_ == 1 && c_ == 4) LAUNCH(1, 4); else if (nh_ == 1) LAUNCH(1, 8);       \
    else if (nh_ == 2 && c_ == 1) LAUNCH(2, 1); else if (nh_ == 2 && c_ == 2) LAUNCH(2, 2); \
    else if (nh_ == 2 && c_ == 4) LAUNCH(2, 4); else if (nh_ == 2) LAUNCH(2, 8);       \
    else if (nh_ == 4 && c_ == 1) LAUNCH(4, 1); else if (nh_ == 4 && c_ == 2) LAUNCH(4, 2); \
    else if (nh_ == 4 && c_ == 4) LAUNCH(4, 4); else if (nh_ == 4) LAUNCH(4, 8);       \
    else if (c_ == 1) LAUNCH(8, 1); else if (c_ == 2) LAUNCH(8, 2);                   \
    else if (c_ == 4) LAUNCH(8, 4); else LAUNCH(8, 8);                                 \
  } while (0)

static unsigned grid_for(long long B) {
  long long blocks = (B + WARPS - 1) / WARPS;
  const long long cap = 4LL * mm::sm_count();
  return (unsigned)(blocks > cap ? cap : blocks);
}

template <int NH, bool TRAIN>
static void launch_c(const Params& p, unsigned blocks, cudaStream_t st) {
  if (p.U <= 32) mmoe_heads_kernel<NH, 1, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
  else if (p.U <= 64) mmoe_heads_kernel<NH, 2, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
  else if (p.U <= 128) mmoe_heads_kernel<NH, 4, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
  else mmoe_heads_kernel<NH, 8, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
}

template <bool TRAIN>
static void launch(const Params& p, unsigned blocks, cudaStream_t st) {
  if (p.H == 1) launch_c<1, TRAIN>(p, blocks, st);
  else if (p.H == 2) launch_c<2, TRAIN>(p, blocks, st);
  else if (p.H <= 4) launch_c<4, TRAIN>(p, blocks, st);
  else launch_c<8, TRAIN>(p, blocks, st);
}

}  // namespace moe
}  // namespace mm

extern "C" {

int mm_mmoe_heads_fwd_bwd(const float* x, int64_t B, int E, int U, int64_t x_stride, const float* const* gate_logits_host,
                          const int64_t* gate_strides_host, int H, float temperature, const float* w, const float* bias,
                          const int* loss_kind, const float* loss_weight, const void* const* targets, const int* target_dtypes,
                          const float* const* sample_weights, float* logits, float* loss, float* dx, int64_t dx_stride,
                          int mask_relu, float* const* d_gate_logits_host, const int64_t* d_gate_strides_host, float* dw,
                          float* db, void* stream) {
  using namespace mm::moe;
  MM_REQUIRE(x && w && loss_kind && logits && gate_logits_host && gate_strides_host && B >= 0, MM_ERR_ARG,
             "mm_mmoe_heads_fwd_bwd: null pointer or B < 0");
  MM_REQUIRE(E >= 1 && E <= EMAX && U >= 1 && U <= UMAX && H >= 1 && H <= HMAX, MM_ERR_UNSUPPORTED,
             "mm_mmoe_heads_fwd_bwd: E=%d, U=%d, H=%d outside 1..%d, 1..%d, 1..%d", E, U, H, EMAX, UMAX, HMAX);
  MM_REQUIRE(temperature > 0.0f, MM_ERR_ARG, "mm_mmoe_heads_fwd_bwd: temperature must be > 0");
  MM_REQUIRE(x_stride >= (int64_t)E * U, MM_ERR_ARG, "mm_mmoe_heads_fwd_bwd: x_stride < E U");
  const bool train = targets != nullptr;
  MM_REQUIRE(!train || (loss_weight && target_dtypes && loss && dx && d_gate_logits_host && d_gate_strides_host), MM_ERR_ARG,
             "mm_mmoe_heads_fwd_bwd: training needs loss_weight, target_dtypes, loss, dx and the gate-logit gradients");
  MM_REQUIRE(!train || dx_stride >= (int64_t)E * U, MM_ERR_ARG, "mm_mmoe_heads_fwd_bwd: dx_stride < E U");
  Params p;
  memset(&p, 0, sizeof(p));
  for (int t = 0; t < H; ++t) {
    MM_REQUIRE(loss_kind[t] == MM_LOSS_BCE || loss_kind[t] == MM_LOSS_MSE, MM_ERR_ARG, "mm_mmoe_heads_fwd_bwd: task %d: bad loss kind %d",
               t, loss_kind[t]);
    MM_REQUIRE(gate_logits_host[t] && gate_strides_host[t] >= E, MM_ERR_ARG, "mm_mmoe_heads_fwd_bwd: task %d: null gate logits or stride < E", t);
    p.kind[t] = loss_kind[t];
    p.gl[t] = gate_logits_host[t];
    p.ldgl[t] = gate_strides_host[t];
    if (train) {
      MM_REQUIRE(targets[t], MM_ERR_ARG, "mm_mmoe_heads_fwd_bwd: task %d: null targets", t);
      MM_REQUIRE(target_dtypes[t] >= MM_I32 && target_dtypes[t] <= MM_F64, MM_ERR_ARG, "mm_mmoe_heads_fwd_bwd: task %d: bad target dtype", t);
      MM_REQUIRE(d_gate_logits_host[t] && d_gate_strides_host[t] >= E, MM_ERR_ARG,
                 "mm_mmoe_heads_fwd_bwd: task %d: null gate-logit gradient or stride < E", t);
      p.y[t] = targets[t];
      p.y_dtype[t] = target_dtypes[t];
      p.lw[t] = loss_weight[t];
      p.sample_w[t] = sample_weights ? sample_weights[t] : nullptr;
      p.dgl[t] = d_gate_logits_host[t];
      p.lddgl[t] = d_gate_strides_host[t];
    }
  }
  if (B == 0) return MM_OK;
  p.x = x;
  p.ldx = x_stride;
  p.B = B;
  p.E = E;
  p.U = U;
  p.H = H;
  p.inv_t = 1.0f / temperature;
  p.w = w;
  p.bias = bias;
  p.inv_m = 1.0f / (float)B;
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
  long long blocks = (B + WARPS - 1) / WARPS;
  const long long cap = 4LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  if (train) launch<true>(p, (unsigned)blocks, (cudaStream_t)stream);
  else launch<false>(p, (unsigned)blocks, (cudaStream_t)stream);
  return mm::check_launch("mm_mmoe_heads_fwd_bwd");
}

int mm_mmoe_mix_fwd(const float* x, int64_t B, int E, int U, int64_t x_stride, const float* const* gate_logits_host,
                    const int64_t* gate_strides_host, int H, float temperature, float* p, float* m, void* m_split, int Kp,
                    void* stream) {
  using namespace mm::moe;
  MM_REQUIRE(x && p && m && gate_logits_host && gate_strides_host && B >= 0, MM_ERR_ARG, "mm_mmoe_mix_fwd: null pointer or B < 0");
  MM_REQUIRE(E >= 1 && E <= EMAX && U >= 1 && U <= UMAX && H >= 1 && H <= HMAX, MM_ERR_UNSUPPORTED,
             "mm_mmoe_mix_fwd: E=%d, U=%d, H=%d outside 1..%d, 1..%d, 1..%d", E, U, H, EMAX, UMAX, HMAX);
  MM_REQUIRE(temperature > 0.0f && x_stride >= (int64_t)E * U, MM_ERR_ARG, "mm_mmoe_mix_fwd: temperature <= 0 or x_stride < E U");
  MM_REQUIRE(!m_split || (Kp == mm_tc_padded_k(U) && ((uintptr_t)m_split & 15) == 0), MM_ERR_ARG,
             "mm_mmoe_mix_fwd: Kp must be mm_tc_padded_k(U)=%d and m_split 16-byte aligned", mm_tc_padded_k(U));
  MixParams q;
  memset(&q, 0, sizeof(q));
  for (int t = 0; t < H; ++t) {
    MM_REQUIRE(gate_logits_host[t] && gate_strides_host[t] >= E, MM_ERR_ARG, "mm_mmoe_mix_fwd: task %d: null gate logits or stride < E", t);
    q.gl[t] = gate_logits_host[t];
    q.ldgl[t] = gate_strides_host[t];
  }
  if (B == 0) return MM_OK;
  q.x = x;
  q.ldx = x_stride;
  q.B = B;
  q.E = E;
  q.U = U;
  q.H = H;
  q.Kp = Kp;
  q.inv_t = 1.0f / temperature;
  q.p = p;
  q.m = m;
  q.m_split = (__nv_bfloat16*)m_split;
  const unsigned blocks = grid_for(B);
#define MM_MIX_FWD(NH, C) mmoe_mix_fwd_kernel<NH, C><<<blocks, 32 * WARPS, 0, (cudaStream_t)stream>>>(q)
  MM_MOE_DISPATCH(H, U, MM_MIX_FWD);
#undef MM_MIX_FWD
  return mm::check_launch("mm_mmoe_mix_fwd");
}

int mm_mmoe_mix_bwd(const float* x, int64_t B, int E, int U, int64_t x_stride, const float* p, int H, float temperature,
                    const float* dm, float* dx, int64_t dx_stride, int mask_relu, float* const* d_gate_logits_host,
                    const int64_t* d_gate_strides_host, void* stream) {
  using namespace mm::moe;
  MM_REQUIRE(x && p && dm && dx && d_gate_logits_host && d_gate_strides_host && B >= 0, MM_ERR_ARG,
             "mm_mmoe_mix_bwd: null pointer or B < 0");
  MM_REQUIRE(E >= 1 && E <= EMAX && U >= 1 && U <= UMAX && H >= 1 && H <= HMAX, MM_ERR_UNSUPPORTED,
             "mm_mmoe_mix_bwd: E=%d, U=%d, H=%d outside 1..%d, 1..%d, 1..%d", E, U, H, EMAX, UMAX, HMAX);
  MM_REQUIRE(temperature > 0.0f && x_stride >= (int64_t)E * U && dx_stride >= (int64_t)E * U, MM_ERR_ARG,
             "mm_mmoe_mix_bwd: temperature <= 0 or a stride < E U");
  MixParams q;
  memset(&q, 0, sizeof(q));
  for (int t = 0; t < H; ++t) {
    MM_REQUIRE(d_gate_logits_host[t] && d_gate_strides_host[t] >= E, MM_ERR_ARG,
               "mm_mmoe_mix_bwd: task %d: null gate-logit gradient or stride < E", t);
    q.dgl[t] = d_gate_logits_host[t];
    q.lddgl[t] = d_gate_strides_host[t];
  }
  if (B == 0) return MM_OK;
  q.x = x;
  q.ldx = x_stride;
  q.B = B;
  q.E = E;
  q.U = U;
  q.H = H;
  q.inv_t = 1.0f / temperature;
  q.p = const_cast<float*>(p);
  q.dm = dm;
  q.dx = dx;
  q.lddx = dx_stride;
  q.mask_relu = mask_relu;
  const unsigned blocks = grid_for(B);
#define MM_MIX_BWD(NH, C) mmoe_mix_bwd_kernel<NH, C><<<blocks, 32 * WARPS, 0, (cudaStream_t)stream>>>(q)
  MM_MOE_DISPATCH(H, U, MM_MIX_BWD);
#undef MM_MIX_BWD
  return mm::check_launch("mm_mmoe_mix_bwd");
}

int mm_mmoe_task_heads_fwd_bwd(const float* const* x_host, const int64_t* x_strides_host, int64_t B, int K, int H, const float* w,
                               const float* bias, const int* loss_kind, const float* loss_weight, const void* const* targets,
                               const int* target_dtypes, const float* const* sample_weights, float* logits, float* loss,
                               float* const* dx_host, const int64_t* dx_strides_host, int mask_relu, float* dw, float* db,
                               void* stream) {
  using namespace mm::moe;
  MM_REQUIRE(x_host && x_strides_host && w && loss_kind && logits && B >= 0, MM_ERR_ARG,
             "mm_mmoe_task_heads_fwd_bwd: null pointer or B < 0");
  MM_REQUIRE(K >= 1 && K <= UMAX && H >= 1 && H <= HMAX, MM_ERR_UNSUPPORTED, "mm_mmoe_task_heads_fwd_bwd: K=%d, H=%d outside 1..%d, 1..%d",
             K, H, UMAX, HMAX);
  const bool train = targets != nullptr;
  MM_REQUIRE(!train || (loss_weight && target_dtypes && loss && dx_host && dx_strides_host), MM_ERR_ARG,
             "mm_mmoe_task_heads_fwd_bwd: training needs loss_weight, target_dtypes, loss and dx");
  TaskHeadParams p;
  memset(&p, 0, sizeof(p));
  for (int t = 0; t < H; ++t) {
    MM_REQUIRE(loss_kind[t] == MM_LOSS_BCE || loss_kind[t] == MM_LOSS_MSE, MM_ERR_ARG,
               "mm_mmoe_task_heads_fwd_bwd: task %d: bad loss kind %d", t, loss_kind[t]);
    MM_REQUIRE(x_host[t] && x_strides_host[t] >= K, MM_ERR_ARG, "mm_mmoe_task_heads_fwd_bwd: task %d: null input or stride < K", t);
    p.kind[t] = loss_kind[t];
    p.x[t] = x_host[t];
    p.ldx[t] = x_strides_host[t];
    if (train) {
      MM_REQUIRE(targets[t] && target_dtypes[t] >= MM_I32 && target_dtypes[t] <= MM_F64, MM_ERR_ARG,
                 "mm_mmoe_task_heads_fwd_bwd: task %d: null targets or bad target dtype", t);
      MM_REQUIRE(dx_host[t] && dx_strides_host[t] >= K, MM_ERR_ARG, "mm_mmoe_task_heads_fwd_bwd: task %d: null dx or stride < K", t);
      p.y[t] = targets[t];
      p.y_dtype[t] = target_dtypes[t];
      p.lw[t] = loss_weight[t];
      p.sample_w[t] = sample_weights ? sample_weights[t] : nullptr;
      p.dx[t] = dx_host[t];
      p.lddx[t] = dx_strides_host[t];
    }
  }
  if (B == 0) return MM_OK;
  p.B = B;
  p.K = K;
  p.H = H;
  p.w = w;
  p.bias = bias;
  p.inv_m = 1.0f / (float)B;
  p.logits = logits;
  if (train) {
    p.loss = loss;
    p.loss_heads = loss + 1;
    p.mask_relu = mask_relu;
    p.dw = dw;
    p.db = db;
  }
  const unsigned blocks = grid_for(B);
#define MM_TH_T(NH, C) task_heads_kernel<NH, C, true><<<blocks, 32 * WARPS, 0, (cudaStream_t)stream>>>(p)
#define MM_TH_F(NH, C) task_heads_kernel<NH, C, false><<<blocks, 32 * WARPS, 0, (cudaStream_t)stream>>>(p)
  if (train) MM_MOE_DISPATCH(H, K, MM_TH_T);
  else MM_MOE_DISPATCH(H, K, MM_TH_F);
#undef MM_TH_T
#undef MM_TH_F
  return mm::check_launch("mm_mmoe_task_heads_fwd_bwd");
}

}  // extern "C"
