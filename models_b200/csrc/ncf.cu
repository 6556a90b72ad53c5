// Neural collaborative filtering head (NCFModel, models/benchmark.py:32-100): the GMF branch, the output heads and their
// loss, forward and backward in ONE pass over the batch.
//
//   mm_ncf_head_fwd_bwd
//       u = table_u[id_u], i = table_i[id_i]   (the GMF rows, gathered by id; the product g = u * i is never written)
//       z_t = [g | h] . w_t + b_t              (H Dense(D + U -> 1) heads, w the stacked (D + U, H) Keras kernel)
//     with targets: the losses of mm_heads_fwd_bwd and the backward
//       dz_t as mm_heads_fwd_bwd;  r = sum_t dz_t w_t[:D]
//       du = r * i + 2 l2 u,  di = r * u + 2 l2 i   (the IndexedSlices values of both tables, in sample order)
//       dh = sum_t dz_t w_t[D:]                     (zeroed where h <= 0 when relu_h)
//       dw_t += [g | h] dz_t,  db_t += dz_t,  loss += [sum_t lambda_t loss_t, loss_0 ..],  reg += l2 sum (|u|^2 + |i|^2)
//     without: the activated predictions (the |z|-stable sigmoid of mm_heads_fwd_bwd, or z) and the reg term.
//
// Layout (after mmoe.cu): one warp per sample.  Lane j owns the columns j + 32 c of u, i (c < CD) and of h (c < CU);
// the heads' kernel sits in shared memory, dw in registers; per CTA one shared-memory sum and one atomic per value.
#include <cstring>

#include "mm_common.cuh"

namespace mm {
namespace ncf {

constexpr int HMAX = 8;    // heads
constexpr int DMAX = 128;  // GMF width: 4 columns per lane
constexpr int UMAX = 256;  // MLP output: 8 columns per lane
constexpr int WARPS = 8;   // 256 threads per CTA
constexpr int KMAX = DMAX + UMAX;

struct Params {
  const float* tu;
  const float* ti;
  long long rows_u, rows_i;
  const void* ids_u;
  const void* ids_i;
  int wu, wi;  // id bytes
  const float* h;  // (B, U)
  long long ldh;
  const float* xr;  // (B, nxr) rows whose l2 |x|^2 also joins reg, or null
  long long ldxr;
  int nxr;
  long long B;
  int D, U, H;
  int relu_h;
  const float* w;     // (D + U, H) Keras layout
  const float* bias;  // (H,) or null
  const void* y[HMAX];
  int y_dtype[HMAX];
  int kind[HMAX];
  float lw[HMAX];
  const float* sample_w[HMAX];
  float inv_m;
  float l2;
  float* out;  // (H, B): logits (training) or predictions
  float* loss;
  float* loss_heads;
  float* reg;
  float* du;  // (B, D)
  float* di;
  float* dh;
  long long lddh;
  float* dw;  // (D + U, H) accumulated
  float* db;  // (H,) accumulated
  int* oob;
};

// NH: H rounded up to a power of two (heads t >= H are skipped at run time); CD / CU: columns per lane of D / U
template <int NH, int CD, int CU, bool TRAIN>
__global__ void __launch_bounds__(32 * WARPS, 1) ncf_head_kernel(const Params p) {
  // head t's kernel column at t KMAX: the D GMF rows at [0, D), the U MLP rows at [DMAX, DMAX + U), zeros elsewhere (so
  // that the padded columns of a lane add exact zeros)
  __shared__ float s_w[NH * KMAX];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int D = p.D, U = p.U, H = p.H;
  for (int j = threadIdx.x; j < NH * KMAX; j += blockDim.x) {
    const int t = j / KMAX, k = j - t * KMAX;
    float v = 0.0f;
    if (t < H && k < D) v = p.w[k * H + t];
    else if (t < H && k >= DMAX && k - DMAX < U) v = p.w[(D + k - DMAX) * H + t];
    s_w[j] = v;
  }
  float b[NH];
#pragma unroll
  for (int t = 0; t < NH; ++t) b[t] = (t < H && p.bias) ? p.bias[t] : 0.0f;
  __syncthreads();
  float dwg[NH][CD], dwh[NH][CU], loss[NH], db[NH];
#pragma unroll
  for (int t = 0; t < NH; ++t) {
#pragma unroll
    for (int c = 0; c < CD; ++c) dwg[t][c] = 0.0f;
#pragma unroll
    for (int c = 0; c < CU; ++c) dwh[t][c] = 0.0f;
    loss[t] = db[t] = 0.0f;
  }
  float rsum = 0.0f;  // this lane's share of sum |u|^2 + |i|^2 (+ |x|^2)
  const bool want_reg = p.reg != nullptr;
  for (long long m = (long long)blockIdx.x * WARPS + wid; m < p.B; m += (long long)gridDim.x * WARPS) {
    const long long iu = load_id(p.ids_u, p.wu, m), ii = load_id(p.ids_i, p.wi, m);
    const bool oku = iu >= 0 && iu < p.rows_u, oki = ii >= 0 && ii < p.rows_i;
    if (lane == 0 && p.oob) {
      if (!oku) atomicAdd(p.oob, 1);
      if (!oki) atomicAdd(p.oob, 1);
    }
    const float* ru = p.tu + (oku ? iu : 0) * D;
    const float* ri = p.ti + (oki ? ii : 0) * D;
    float u[CD], iv[CD], g[CD], hv[CU];
#pragma unroll
    for (int c = 0; c < CD; ++c) {
      const int k = lane + 32 * c;
      u[c] = (oku && k < D) ? __ldg(ru + k) : 0.0f;
      iv[c] = (oki && k < D) ? __ldg(ri + k) : 0.0f;
      g[c] = u[c] * iv[c];
    }
    const float* rh = p.h + m * p.ldh;
#pragma unroll
    for (int c = 0; c < CU; ++c) {
      const int k = lane + 32 * c;
      hv[c] = k < U ? __ldg(rh + k) : 0.0f;
    }
    if (want_reg) {
#pragma unroll
      for (int c = 0; c < CD; ++c) rsum = fmaf(u[c], u[c], fmaf(iv[c], iv[c], rsum));
      if (p.xr)
        for (int k = lane; k < p.nxr; k += 32) {
          const float x = __ldg(p.xr + m * p.ldxr + k);
          rsum = fmaf(x, x, rsum);
        }
    }
    float dz[NH];
#pragma unroll
    for (int t = 0; t < NH; ++t) {
      dz[t] = 0.0f;
      if (t >= H) continue;
      const float* wt = s_w + t * KMAX;
      float dot = 0.0f;
#pragma unroll
      for (int c = 0; c < CD; ++c) dot = fmaf(g[c], wt[lane + 32 * c], dot);
#pragma unroll
      for (int c = 0; c < CU; ++c) dot = fmaf(hv[c], wt[DMAX + lane + 32 * c], dot);
      const float z = warp_sum(dot) + b[t];
      if (!TRAIN) {
        if (lane == 0) p.out[t * p.B + m] = head_pred(p.kind[t], z);
        continue;
      }
      const float y = load_as_f32(p.y[t], m, p.y_dtype[t]);
      const float sw = p.sample_w[t] ? p.sample_w[t][m] : 1.0f;
      float l, gz;
      head_loss(p.kind[t], z, y, l, gz);
      float d = gz * sw * p.inv_m;
      d *= p.lw[t];  // exact for lambda = 1
      dz[t] = d;
#pragma unroll
      for (int c = 0; c < CD; ++c) dwg[t][c] = fmaf(g[c], d, dwg[t][c]);
#pragma unroll
      for (int c = 0; c < CU; ++c) dwh[t][c] = fmaf(hv[c], d, dwh[t][c]);
      if (lane == 0) {
        loss[t] += l * sw * p.inv_m;
        db[t] += d;
        p.out[t * p.B + m] = z;
      }
    }
    if (!TRAIN) continue;
    const float two_l2 = 2.0f * p.l2;
#pragma unroll
    for (int c = 0; c < CD; ++c) {
      const int k = lane + 32 * c;
      if (k >= D) continue;
      float r = 0.0f;
#pragma unroll
      for (int t = 0; t < NH; ++t)
        if (t < H) r = fmaf(dz[t], s_w[t * KMAX + k], r);
      p.du[m * D + k] = fmaf(two_l2, u[c], r * iv[c]);
      p.di[m * D + k] = fmaf(two_l2, iv[c], r * u[c]);
    }
    float* dhr = p.dh + m * p.lddh;
#pragma unroll
    for (int c = 0; c < CU; ++c) {
      const int k = lane + 32 * c;
      if (k >= U) continue;
      float r = 0.0f;
#pragma unroll
      for (int t = 0; t < NH; ++t)
        if (t < H) r = fmaf(dz[t], s_w[t * KMAX + DMAX + k], r);
      dhr[k] = (!p.relu_h || hv[c] > 0.0f) ? r : 0.0f;
    }
  }
  // block-level reduction before the atomics: the reg term, then dw / db / loss one head at a time
  __shared__ float red[WARPS][KMAX + 2];
  if (want_reg) {
    rsum = warp_sum(rsum);
    if (lane == 0) red[wid][0] = rsum;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.0f;
      for (int i = 0; i < WARPS; ++i) s += red[i][0];
      s *= p.l2;
      atomicAdd(p.reg, s);
      if (TRAIN) atomicAdd(p.loss, s);
    }
  }
  if (!TRAIN) return;
#pragma unroll
  for (int t = 0; t < NH; ++t) {
    if (t >= H) break;
    __syncthreads();  // the previous sums have been read
#pragma unroll
    for (int c = 0; c < CD; ++c) red[wid][lane + 32 * c] = dwg[t][c];
#pragma unroll
    for (int c = 0; c < CU; ++c) red[wid][DMAX + lane + 32 * c] = dwh[t][c];
    if (lane == 0) {
      red[wid][KMAX] = db[t];
      red[wid][KMAX + 1] = loss[t];
    }
    __syncthreads();
    for (int k = threadIdx.x; k < KMAX + 2; k += blockDim.x) {
      if ((k >= D && k < DMAX) || (k >= DMAX + U && k < KMAX)) continue;
      float s = 0.0f;
      for (int i = 0; i < WARPS; ++i) s += red[i][k];
      if (k < DMAX) {
        atomicAdd(p.dw + k * H + t, s);
      } else if (k < KMAX) {
        atomicAdd(p.dw + (D + k - DMAX) * H + t, s);
      } else if (k == KMAX) {
        if (p.db) atomicAdd(p.db + t, s);
      } else {
        atomicAdd(p.loss, p.lw[t] * s);
        atomicAdd(p.loss_heads + t, s);
      }
    }
  }
}

template <int NH, int CD, bool TRAIN>
static void launch_u(const Params& p, unsigned blocks, cudaStream_t st) {
  if (p.U <= 32) ncf_head_kernel<NH, CD, 1, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
  else if (p.U <= 64) ncf_head_kernel<NH, CD, 2, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
  else if (p.U <= 128) ncf_head_kernel<NH, CD, 4, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
  else ncf_head_kernel<NH, CD, 8, TRAIN><<<blocks, 32 * WARPS, 0, st>>>(p);
}

template <int NH, bool TRAIN>
static void launch_d(const Params& p, unsigned blocks, cudaStream_t st) {
  if (p.D <= 32) launch_u<NH, 1, TRAIN>(p, blocks, st);
  else if (p.D <= 64) launch_u<NH, 2, TRAIN>(p, blocks, st);
  else launch_u<NH, 4, TRAIN>(p, blocks, st);
}

template <bool TRAIN>
static void launch(const Params& p, unsigned blocks, cudaStream_t st) {
  if (p.H == 1) launch_d<1, TRAIN>(p, blocks, st);
  else if (p.H == 2) launch_d<2, TRAIN>(p, blocks, st);
  else if (p.H <= 4) launch_d<4, TRAIN>(p, blocks, st);
  else launch_d<8, TRAIN>(p, blocks, st);
}

}  // namespace ncf
}  // namespace mm

extern "C" {

int mm_ncf_head_fwd_bwd(const float* table_u, int64_t rows_u, const void* ids_u, int idx_bytes_u, const float* table_i,
                        int64_t rows_i, const void* ids_i, int idx_bytes_i, int D, const float* h, int64_t h_stride, int U,
                        int relu_h, int64_t B, int H, const float* w, const float* bias, const int* loss_kind,
                        const float* loss_weight, const void* const* targets, const int* target_dtypes,
                        const float* const* sample_weights, float l2, const float* x_reg, int64_t x_reg_stride, int x_reg_width,
                        float* out, float* loss, float* reg, float* du, float* di, float* dh, int64_t dh_stride, float* dw,
                        float* db, int32_t* oob_count, void* stream) {
  using namespace mm::ncf;
  static const char* who = "mm_ncf_head_fwd_bwd";
  MM_REQUIRE(table_u && table_i && h && w && loss_kind && out && B >= 0, MM_ERR_ARG, "%s: null pointer or B < 0", who);
  MM_REQUIRE(D >= 1 && D <= DMAX && U >= 1 && U <= UMAX && H >= 1 && H <= HMAX, MM_ERR_UNSUPPORTED,
             "%s: D=%d, U=%d, H=%d outside 1..%d, 1..%d, 1..%d", who, D, U, H, DMAX, UMAX, HMAX);
  if (const int rc = mm::check_id_column(who, 0, ids_u, idx_bytes_u, rows_u)) return rc;
  if (const int rc = mm::check_id_column(who, 1, ids_i, idx_bytes_i, rows_i)) return rc;
  MM_REQUIRE(h_stride >= U, MM_ERR_ARG, "%s: h_stride < U", who);
  MM_REQUIRE(l2 >= 0.0f && l2 <= 3.0e38f, MM_ERR_ARG, "%s: l2 must be finite and >= 0", who);
  MM_REQUIRE(!x_reg || (x_reg_width >= 1 && x_reg_stride >= x_reg_width), MM_ERR_ARG, "%s: x_reg needs width >= 1 and stride >= width",
             who);
  MM_REQUIRE(!x_reg || reg, MM_ERR_ARG, "%s: x_reg needs reg", who);
  const bool train = targets != nullptr;
  MM_REQUIRE(!train || (loss_weight && target_dtypes && loss && du && di && dh && dw), MM_ERR_ARG,
             "%s: training needs loss_weight, target_dtypes, loss, du, di, dh and dw", who);
  MM_REQUIRE(!train || dh_stride >= U, MM_ERR_ARG, "%s: dh_stride < U", who);
  Params p;
  memset(&p, 0, sizeof(p));
  for (int t = 0; t < H; ++t) {
    MM_REQUIRE(loss_kind[t] == MM_LOSS_BCE || loss_kind[t] == MM_LOSS_MSE, MM_ERR_ARG, "%s: head %d: bad loss kind %d", who, t,
               loss_kind[t]);
    p.kind[t] = loss_kind[t];
    if (train) {
      MM_REQUIRE(targets[t] && target_dtypes[t] >= MM_I32 && target_dtypes[t] <= MM_F64, MM_ERR_ARG,
                 "%s: head %d: null targets or bad target dtype", who, t);
      p.y[t] = targets[t];
      p.y_dtype[t] = target_dtypes[t];
      p.lw[t] = loss_weight[t];
      p.sample_w[t] = sample_weights ? sample_weights[t] : nullptr;
    }
  }
  if (B == 0) return MM_OK;
  p.tu = table_u;
  p.ti = table_i;
  p.rows_u = rows_u;
  p.rows_i = rows_i;
  p.ids_u = ids_u;
  p.ids_i = ids_i;
  p.wu = idx_bytes_u;
  p.wi = idx_bytes_i;
  p.h = h;
  p.ldh = h_stride;
  p.xr = x_reg;
  p.ldxr = x_reg_stride;
  p.nxr = x_reg ? x_reg_width : 0;
  p.B = B;
  p.D = D;
  p.U = U;
  p.H = H;
  p.relu_h = relu_h;
  p.w = w;
  p.bias = bias;
  p.inv_m = 1.0f / (float)B;
  p.l2 = l2;
  p.out = out;
  p.reg = reg;
  p.oob = oob_count;
  if (train) {
    p.loss = loss;
    p.loss_heads = loss + 1;
    p.du = du;
    p.di = di;
    p.dh = dh;
    p.lddh = dh_stride;
    p.dw = dw;
    p.db = db;
  }
  long long blocks = (B + WARPS - 1) / WARPS;
  const long long cap = 4LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  if (train) launch<true>(p, (unsigned)blocks, (cudaStream_t)stream);
  else launch<false>(p, (unsigned)blocks, (cudaStream_t)stream);
  return mm::check_launch(who);
}

}  // extern "C"
