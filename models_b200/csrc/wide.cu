// Wide&Deep head (WideAndDeepModel, models/ranking.py:276-570; CategoryEncoding, transforms/features.py:473-612).
//
//   mm_wide_deep_head_fwd_bwd  everything after the deep tower's last hidden layer, in ONE pass over the batch:
//       wide[b] = sum over one-hot blocks W[off + id] + sum over bag blocks of W[off + id] over the bag's ids
//                 (multi_hot: each distinct id once, Keras' bincount(binary_output=True); count: every occurrence) + bw
//       u[b]    = h[b] . w_dl + b_dl,  deep[b] = act_dl(u)            (the deep branch's MLPBlock([1]) Dense)
//       s = wide + deep;  z = s w_out + b_out                         (element-wise sum, then the output's Dense(1))
//     with targets: the loss and the backward (ds, dh, the Dense gradients); without: out[b] = act(z).
//   mm_wide_bag_grad  one bag block's gradient as nnz (id, value) pairs for mm_wide_rows_apply.
//
// Layout of the head: a group of G = 16 lanes owns one sample (two samples per warp).  The lanes of a group read h[b]
// as float4 (lane j: columns 4 (j + 16 c) .. +3), stride the one-hot blocks and each bag's positions, and reduce with
// four shuffles inside the group.  dw_dl stays in registers; per CTA one shared-memory sum and one atomic per value.
#include <cstring>

#include "mm_common.cuh"

namespace mm {
namespace wide {

constexpr int MAX_ONEHOT = 64;
constexpr int MAX_BAGS = 32;
constexpr int G = 16;            // lanes per sample
constexpr int MAX_U = 64 * 8;    // 8 float4 per lane
constexpr int WARPS = 8;         // 256 threads per CTA
constexpr int NS = 8;            // scalar sums per CTA: loss, dw_out, db_out, db_dl, d_wide_bias

struct OneHot {
  const void* ids;
  long long rows;
  long long off;
  int idb;
};
struct Bag {
  const void* values;
  const void* offsets;  // (B + 1,) or null: fixed length L
  long long rows;
  long long off;
  long long nnz;
  int idb;
  int off_dtype;
  int L;
  int mode;
};

struct HeadParams {
  OneHot oh[MAX_ONEHOT];
  Bag bag[MAX_BAGS];
  int n_oh, n_bag;
  const float* wide;
  const float* wide_bias;
  const float* h;
  long long ldh;
  int U;
  int vec;  // h, dh, w_dl 16-byte aligned with strides and U multiples of 4
  int mask_h;
  const float* w_dl;
  const float* b_dl;
  int act_dl;
  const float* out_w;
  const float* out_b;
  int out_act;
  int kind;
  const void* y;
  int y_dtype;
  const float* sw;
  float inv_m;
  float* out;  // logits with targets, act(z) without
  float* loss;
  float* ds;
  float* dh;
  long long lddh;
  float* dw_out;
  float* db_out;
  float* dw_dl;
  float* db_dl;
  float* dbw;
  int* oob;
  long long B;
};

__device__ __forceinline__ long long load_offset(const void* p, int dtype, long long i) {
  return dtype == MM_I64 ? reinterpret_cast<const long long*>(p)[i] : (long long)reinterpret_cast<const int32_t*>(p)[i];
}

// [start, end) of sample b's bag: offsets clamped to [0, nnz], an end below the start is an empty bag; fixed length: b L.
__device__ __forceinline__ void bag_range(const Bag& q, long long b, long long& start, long long& end) {
  if (!q.offsets) {
    start = b * q.L;
    end = start + q.L;
    return;
  }
  start = load_offset(q.offsets, q.off_dtype, b);
  end = load_offset(q.offsets, q.off_dtype, b + 1);
  start = start < 0 ? 0 : (start > q.nnz ? q.nnz : start);
  end = end < start ? start : (end > q.nnz ? q.nnz : end);
}

// True when position p holds the first occurrence of `id` in [start, p): the multi_hot encoding counts each distinct id of
// a bag once.  A linear scan of the earlier positions (bags are short; the cost is quadratic in the bag length).
__device__ __forceinline__ bool first_occurrence(const void* values, int idb, long long start, long long p, long long id) {
  for (long long j = start; j < p; ++j)
    if (load_id(values, idb, j) == id) return false;
  return true;
}

__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float4 load4(const float* row, int k, int U, bool vec) {
  if (vec) return k < U ? *reinterpret_cast<const float4*>(row + k) : make_float4(0.f, 0.f, 0.f, 0.f);
  return make_float4(k < U ? row[k] : 0.f, k + 1 < U ? row[k + 1] : 0.f, k + 2 < U ? row[k + 2] : 0.f, k + 3 < U ? row[k + 3] : 0.f);
}

__device__ __forceinline__ void store4(float* row, int k, int U, bool vec, float4 v) {
  if (vec) {
    if (k < U) *reinterpret_cast<float4*>(row + k) = v;
    return;
  }
  if (k < U) row[k] = v.x;
  if (k + 1 < U) row[k + 1] = v.y;
  if (k + 2 < U) row[k + 2] = v.z;
  if (k + 3 < U) row[k + 3] = v.w;
}

// this lane's share of sample b's wide term (the group's lanes stride the one-hot blocks and each bag's positions)
__device__ __forceinline__ float wide_partial(const HeadParams& p, long long b, int gl) {
  float acc = 0.0f;
  int n_bad = 0;
  for (int f = gl; f < p.n_oh; f += G) {
    const OneHot& o = p.oh[f];
    const unsigned long long id = (unsigned long long)load_id(o.ids, o.idb, b);
    if (id < (unsigned long long)o.rows) acc += __ldg(p.wide + o.off + (long long)id);
    else ++n_bad;
  }
  for (int q = 0; q < p.n_bag; ++q) {
    const Bag& g = p.bag[q];
    long long start, end;
    bag_range(g, b, start, end);
    for (long long i = start + gl; i < end; i += G) {
      const long long id = load_id(g.values, g.idb, i);
      if ((unsigned long long)id >= (unsigned long long)g.rows) {
        ++n_bad;
        continue;
      }
      if (g.mode == MM_WIDE_MULTI_HOT && !first_occurrence(g.values, g.idb, start, i, id)) continue;
      acc += __ldg(p.wide + g.off + id);
    }
  }
  if (n_bad && p.oob) atomicAdd(p.oob, n_bad);
  return acc;
}

template <int UC>  // float4 chunks of h per lane: U <= 64 UC
__global__ void __launch_bounds__(256, 1) wide_deep_head_kernel(const __grid_constant__ HeadParams p) {
  const int lane = threadIdx.x & 31, gl = lane & (G - 1), wid = threadIdx.x >> 5;
  const long long grp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const long long n_grp = ((long long)gridDim.x * blockDim.x) / G;
  const bool vec = p.vec != 0, deep = p.h != nullptr, train = p.y != nullptr;
  float4 wdl[UC], dwl[UC];
#pragma unroll
  for (int c = 0; c < UC; ++c) {
    wdl[c] = deep ? load4(p.w_dl, 4 * (gl + G * c), p.U, vec) : make_float4(0.f, 0.f, 0.f, 0.f);
    dwl[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float wo = p.out_w[0], bo = p.out_b ? p.out_b[0] : 0.0f;
  const float bw = p.wide_bias ? p.wide_bias[0] : 0.0f, bdl = p.b_dl ? p.b_dl[0] : 0.0f;
  const bool relu_dl = p.act_dl == MM_ACT_RELU;
  float a_loss = 0.f, a_dwo = 0.f, a_dbo = 0.f, a_dbdl = 0.f, a_dbw = 0.f;
  // every lane of a warp runs the same number of laps (the shuffles need the whole warp)
  const long long laps = (p.B + n_grp - 1) / n_grp;
  for (long long lap = 0; lap < laps; ++lap) {
    const long long b = grp + lap * n_grp;
    const bool valid = b < p.B;
    const long long bb = valid ? b : 0;
    const float w = group_sum(valid ? wide_partial(p, bb, gl) : 0.0f);
    float4 hv[UC];
    float u = 0.0f;
    if (deep) {
      const float* hr = p.h + bb * p.ldh;
#pragma unroll
      for (int c = 0; c < UC; ++c) {
        hv[c] = valid ? load4(hr, 4 * (gl + G * c), p.U, vec) : make_float4(0.f, 0.f, 0.f, 0.f);
        u = fmaf(hv[c].x, wdl[c].x, u);
        u = fmaf(hv[c].y, wdl[c].y, u);
        u = fmaf(hv[c].z, wdl[c].z, u);
        u = fmaf(hv[c].w, wdl[c].w, u);
      }
      u = group_sum(u) + bdl;
    }
    if (!valid) continue;
    const float s = w + bw + (deep ? (relu_dl ? fmaxf(u, 0.0f) : u) : 0.0f);
    const float z = fmaf(s, wo, bo);
    if (!train) {
      if (gl == 0) p.out[b] = apply_act(z, p.out_act);
      continue;
    }
    const float y = load_as_f32(p.y, b, p.y_dtype);
    const float sw = p.sw ? p.sw[b] : 1.0f;
    float l, g;
    head_loss(p.kind, z, y, l, g);
    const float delta = g * sw * p.inv_m;
    const float dsv = delta * wo;
    const float du = (relu_dl && !(u > 0.0f)) ? 0.0f : dsv;
    if (gl == 0) {
      a_loss += l * sw * p.inv_m;
      a_dwo = fmaf(delta, s, a_dwo);
      a_dbo += delta;
      a_dbdl += du;
      a_dbw += dsv;
      p.out[b] = z;
      p.ds[b] = dsv;
    }
    if (deep) {
      float* dr = p.dh + b * p.lddh;
#pragma unroll
      for (int c = 0; c < UC; ++c) {
        const int k = 4 * (gl + G * c);
        const float4 h4 = hv[c], w4 = wdl[c];
        dwl[c].x = fmaf(du, h4.x, dwl[c].x);
        dwl[c].y = fmaf(du, h4.y, dwl[c].y);
        dwl[c].z = fmaf(du, h4.z, dwl[c].z);
        dwl[c].w = fmaf(du, h4.w, dwl[c].w);
        const bool m = p.mask_h != 0;
        float4 d;
        d.x = (!m || h4.x > 0.0f) ? du * w4.x : 0.0f;
        d.y = (!m || h4.y > 0.0f) ? du * w4.y : 0.0f;
        d.z = (!m || h4.z > 0.0f) ? du * w4.z : 0.0f;
        d.w = (!m || h4.w > 0.0f) ? du * w4.w : 0.0f;
        store4(dr, k, p.U, vec, d);
      }
    }
  }
  if (!train) return;
  // the warp's two groups hold the same columns: fold them, then one row per warp in shared memory
  __shared__ __align__(16) float red[WARPS][MAX_U + NS];
  const auto fold = [](float v) { return v + __shfl_xor_sync(0xffffffffu, v, G); };
#pragma unroll
  for (int c = 0; c < UC; ++c) {
    const float4 v = make_float4(fold(dwl[c].x), fold(dwl[c].y), fold(dwl[c].z), fold(dwl[c].w));
    if (lane < G) *reinterpret_cast<float4*>(&red[wid][4 * (gl + G * c)]) = v;
  }
  a_loss = fold(a_loss);
  a_dwo = fold(a_dwo);
  a_dbo = fold(a_dbo);
  a_dbdl = fold(a_dbdl);
  a_dbw = fold(a_dbw);
  if (lane == 0) {
    red[wid][MAX_U + 0] = a_loss;
    red[wid][MAX_U + 1] = a_dwo;
    red[wid][MAX_U + 2] = a_dbo;
    red[wid][MAX_U + 3] = a_dbdl;
    red[wid][MAX_U + 4] = a_dbw;
  }
  __syncthreads();
  const int nw = blockDim.x >> 5;
  for (int k = threadIdx.x; k < MAX_U + 5; k += blockDim.x) {
    if (k < MAX_U && (!deep || k >= p.U)) continue;
    float s = 0.0f;
    for (int i = 0; i < nw; ++i) s += red[i][k];
    switch (k - MAX_U) {
      case 0:
        if (p.loss) {
          atomicAdd(p.loss, s);  // loss (2,): [total, the one output's]
          atomicAdd(p.loss + 1, s);
        }
        break;
      case 1: if (p.dw_out) atomicAdd(p.dw_out, s); break;
      case 2: if (p.db_out) atomicAdd(p.db_out, s); break;
      case 3: if (p.db_dl) atomicAdd(p.db_dl, s); break;
      case 4: if (p.dbw) atomicAdd(p.dbw, s); break;
      default: if (p.dw_dl) atomicAdd(p.dw_dl + k, s); break;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// mm_wide_bag_grad: one thread per position i of the bag block.  Its sample is i / L (fixed length) or the last b with
// offsets[b] <= i (binary search; the position must then lie in b's clamped range, else no bag covers it).
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) wide_bag_grad_kernel(const __grid_constant__ Bag q, long long B, const float* __restrict__ ds,
                                                            long long* __restrict__ out_ids, float* __restrict__ out_vals) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < q.nnz; i += (long long)gridDim.x * blockDim.x) {
    long long b = B;  // no sample
    if (!q.offsets) {
      b = i / q.L;
    } else if (B > 0) {
      long long lo = 0, hi = B;  // invariant for non-decreasing offsets: offsets[lo] <= i < offsets[hi]
      while (hi - lo > 1) {
        const long long mid = (lo + hi) >> 1;
        if (load_offset(q.offsets, q.off_dtype, mid) <= i) lo = mid;
        else hi = mid;
      }
      b = lo;
    }
    long long start = 0, end = 0;
    if (b < B) bag_range(q, b, start, end);
    long long id = -1;
    float v = 0.0f;
    if (i >= start && i < end) {
      const long long x = load_id(q.values, q.idb, i);
      if ((unsigned long long)x < (unsigned long long)q.rows &&
          (q.mode == MM_WIDE_COUNT || first_occurrence(q.values, q.idb, start, i, x))) {
        id = x;
        v = ds[b];
      }
    }
    out_ids[i] = id;
    out_vals[i] = v;
  }
}

}  // namespace wide
}  // namespace mm

namespace {

int fill_bag(const char* who, int i, const mm_wide_bag& s, int64_t B, mm::wide::Bag& q) {
  MM_REQUIRE(s.values && s.offset >= 0 && s.nnz >= 0 && (s.mode == MM_WIDE_MULTI_HOT || s.mode == MM_WIDE_COUNT), MM_ERR_ARG,
             "%s: bag block %d: null values, negative offset or nnz, or unknown mode", who, i);
  if (const int rc = mm::check_id_column(who, i, s.values, s.idx_bytes, s.rows)) return rc;
  if (s.offsets) {
    MM_REQUIRE(s.off_dtype == MM_I32 || s.off_dtype == MM_I64, MM_ERR_ARG, "%s: bag block %d: offsets must be int32 or int64", who, i);
    MM_REQUIRE(((uintptr_t)s.offsets & (s.off_dtype == MM_I64 ? 7 : 3)) == 0, MM_ERR_ALIGN, "%s: bag block %d: misaligned offsets", who, i);
  } else {
    MM_REQUIRE(s.length >= 1 && s.nnz == B * (int64_t)s.length, MM_ERR_ARG,
               "%s: bag block %d: a fixed-length block needs length >= 1 and nnz = B * length", who, i);
  }
  q.values = s.values;
  q.offsets = s.offsets;
  q.rows = s.rows;
  q.off = s.offset;
  q.nnz = s.nnz;
  q.idb = s.idx_bytes;
  q.off_dtype = s.off_dtype;
  q.L = s.offsets ? 0 : s.length;
  q.mode = s.mode;
  return MM_OK;
}

}  // namespace

extern "C" {

int mm_wide_deep_head_fwd_bwd(const mm_wide_block* onehot_host, int n_onehot, const mm_wide_bag* bags_host, int n_bags,
                              const float* wide_kernel, const float* wide_bias, const float* h, int64_t h_stride, int units,
                              int mask_h, const float* w_dl, const float* b_dl, int act_dl, const float* out_w, const float* out_b,
                              int out_act, int loss_kind, const void* targets, int target_dtype, const float* sample_weight,
                              int64_t B, float* out, float* loss, float* ds, float* dh, int64_t dh_stride, float* dw_out,
                              float* db_out, float* dw_dl, float* db_dl, float* d_wide_bias, int32_t* oob_count, void* stream) {
  using namespace mm::wide;
  const char* who = "mm_wide_deep_head_fwd_bwd";
  MM_REQUIRE(out_w && out && B >= 0, MM_ERR_ARG, "%s: null out_w / out or negative B", who);
  MM_REQUIRE(n_onehot >= 0 && n_onehot <= MAX_ONEHOT && n_bags >= 0 && n_bags <= MAX_BAGS, MM_ERR_UNSUPPORTED,
             "%s: 0..%d one-hot and 0..%d bag blocks", who, MAX_ONEHOT, MAX_BAGS);
  MM_REQUIRE((n_onehot == 0 || onehot_host) && (n_bags == 0 || bags_host), MM_ERR_ARG, "%s: blocks without descriptors", who);
  MM_REQUIRE(n_onehot + n_bags == 0 || wide_kernel, MM_ERR_ARG, "%s: wide blocks without a wide kernel", who);
  MM_REQUIRE(h || n_onehot + n_bags > 0, MM_ERR_ARG, "%s: neither a wide nor a deep part", who);
  if (h) {
    MM_REQUIRE(w_dl && units >= 1 && units <= MAX_U && h_stride >= units, MM_ERR_UNSUPPORTED,
               "%s: deep part needs w_dl, 1 <= units <= %d and h_stride >= units (units=%d)", who, MAX_U, units);
    MM_REQUIRE(act_dl == MM_ACT_LINEAR || act_dl == MM_ACT_RELU, MM_ERR_UNSUPPORTED, "%s: deep-logit activation must be linear or relu", who);
  }
  if (targets) {
    MM_REQUIRE(ds && (!h || (dh && dh_stride >= units)), MM_ERR_ARG, "%s: training needs ds and (deep part) dh with dh_stride >= units", who);
    MM_REQUIRE(loss_kind == MM_LOSS_BCE || loss_kind == MM_LOSS_MSE, MM_ERR_ARG, "%s: bad loss kind %d", who, loss_kind);
    MM_REQUIRE(target_dtype >= MM_I32 && target_dtype <= MM_F64, MM_ERR_ARG, "%s: bad target dtype", who);
  } else {
    MM_REQUIRE(out_act >= MM_ACT_LINEAR && out_act <= MM_ACT_GELU, MM_ERR_ARG, "%s: unknown activation", who);
  }
  HeadParams p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < n_onehot; ++i) {
    const mm_wide_block& t = onehot_host[i];
    MM_REQUIRE(t.offset >= 0, MM_ERR_ARG, "%s: one-hot block %d: negative offset", who, i);
    if (const int rc = mm::check_id_column(who, i, t.indices, t.idx_bytes, t.rows)) return rc;
    p.oh[i] = OneHot{t.indices, t.rows, t.offset, t.idx_bytes};
  }
  for (int i = 0; i < n_bags; ++i)
    if (const int rc = fill_bag(who, i, bags_host[i], B, p.bag[i])) return rc;
  p.n_oh = n_onehot;
  p.n_bag = n_bags;
  if (B == 0) return MM_OK;
  p.wide = wide_kernel;
  p.wide_bias = wide_bias;
  p.h = h;
  p.ldh = h_stride;
  p.U = h ? units : 0;
  p.vec = h && units % 4 == 0 && h_stride % 4 == 0 && ((uintptr_t)h & 15) == 0 && ((uintptr_t)w_dl & 15) == 0 &&
          (!targets || (dh_stride % 4 == 0 && ((uintptr_t)dh & 15) == 0));
  p.mask_h = mask_h ? 1 : 0;
  p.w_dl = w_dl;
  p.b_dl = b_dl;
  p.act_dl = act_dl;
  p.out_w = out_w;
  p.out_b = out_b;
  p.out_act = out_act;
  p.kind = loss_kind;
  p.y = targets;
  p.y_dtype = target_dtype;
  p.sw = sample_weight;
  p.inv_m = 1.0f / (float)B;
  p.out = out;
  p.loss = loss;
  p.ds = ds;
  p.dh = dh;
  p.lddh = dh_stride;
  p.dw_out = dw_out;
  p.db_out = db_out;
  p.dw_dl = dw_dl;
  p.db_dl = db_dl;
  p.dbw = d_wide_bias;
  p.oob = oob_count;
  p.B = B;
  const long long per_cta = 256 / G;
  long long blocks = (B + per_cta - 1) / per_cta;
  const long long cap = 8LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  const int uc = p.U <= 64 ? 1 : p.U <= 128 ? 2 : p.U <= 256 ? 4 : 8;
  cudaStream_t st = (cudaStream_t)stream;
  switch (uc) {
    case 1: wide_deep_head_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(p); break;
    case 2: wide_deep_head_kernel<2><<<(unsigned)blocks, 256, 0, st>>>(p); break;
    case 4: wide_deep_head_kernel<4><<<(unsigned)blocks, 256, 0, st>>>(p); break;
    default: wide_deep_head_kernel<8><<<(unsigned)blocks, 256, 0, st>>>(p); break;
  }
  return mm::check_launch(who);
}

int mm_wide_bag_grad(const mm_wide_bag* bag_host, int64_t B, const float* ds, int64_t* out_ids, float* out_values, void* stream) {
  using namespace mm::wide;
  const char* who = "mm_wide_bag_grad";
  MM_REQUIRE(bag_host && ds && out_ids && out_values && B >= 0, MM_ERR_ARG, "%s: null pointer or negative B", who);
  Bag q;
  memset(&q, 0, sizeof(q));
  if (const int rc = fill_bag(who, 0, *bag_host, B, q)) return rc;
  if (q.nnz == 0) return MM_OK;
  long long blocks = (q.nnz + 255) / 256;
  const long long cap = 16LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  wide_bag_grad_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(q, (long long)B, ds, (long long*)out_ids, out_values);
  return mm::check_launch(who);
}

}  // extern "C"
