// Factorization-machine heads (merlin/models/tf/blocks/interaction.py:205-332, models/ranking.py:171-279 DeepFMModel).
//
//   mm_fm_pairwise   FMPairwiseInteraction.call on a (B, A, K) tensor: 0.5 * ((sum_a x)^2 - sum_a x^2) -> (B, K)
//   mm_deepfm_head   what DeepFMModel evaluates after its deep tower, in ONE pass over the batch:
//       pairwise[b] = sum_f 0.5 * ((sum_d e_f[d])^2 - sum_d e_f[d]^2)
//           FMBlock stacks the F embeddings with StackFeatures(axis=-1) -> (B, D, F) and FMPairwiseInteraction reduces
//           axis 1, so the reference's "pairwise" term is taken over the D components of EACH feature and then summed over
//           the features (interaction.py:323-328); restated as written, not as the textbook FM.
//       wide[b]     = sum_f Wk[off_f + id_f] + sum_c Wk[off_c] * x_c + bw
//           = Dense(1) over concat(one-hot(categorical), continuous) (CategoryEncoding + MLPBlock([1]), :307-316): the
//           one-hot matmul is a row lookup in the (sum of cardinalities + n_cont, 1) Keras kernel.
//       z = pairwise + wide + deep[b]         (ParallelBlock "element-wise-sum" of the fm and deep towers)
//       out[b] = act(z * w_out + b_out)       (BinaryOutput's Dense(1, sigmoid) on the 1-wide sum; optional)
//   One warp per sample: lanes stride the D components of a row (coalesced), the per-feature sum needs one warp
//   reduction, the squares are reduced once per sample.  The embedding rows are read once (F x D x 4 bytes per sample).
//   mm_deepfm_head_fwd_bwd  the training counterpart: forward, loss and backward of the head in one pass (below)
//   mm_fm_concat_backward   the FM term's gradient into the embedding rows, summed with the deep tower's input gradient
#include <cstring>

#include "mm_common.cuh"

namespace mm {
namespace fm {

constexpr int MAX_T = MM_LOOKUP_MAX_ROWS;

struct Params {
  const float* w[MAX_T];
  const void* ids[MAX_T];
  long long rows[MAX_T];
  long long woff[MAX_T];  // row of the feature's block in the wide kernel
  unsigned char idb[MAX_T];
  int T;
  const void* csrc[MAX_T];
  long long cstride[MAX_T];
  long long coff[MAX_T];
  int cdtype[MAX_T];
  int C;
  const float* wide;
  const float* wide_bias;
  const float* addend;
  long long addend_stride;
  const float* out_w;
  const float* out_b;
  int out_act;
  float* out;
  int* oob;
  long long B;
  int D;
};

__global__ void __launch_bounds__(256) deepfm_head_kernel(const __grid_constant__ Params p) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long b = warp; b < p.B; b += n_warps) {
    float pair = 0.0f, sq = 0.0f, wide = 0.0f;
    for (int f = 0; f < p.T; ++f) {
      const unsigned long long id = (unsigned long long)load_id(p.ids[f], p.idb[f], b);
      const bool ok = id < (unsigned long long)p.rows[f];
      if (!ok && lane == 0 && p.oob) atomicAdd(p.oob, 1);
      float s = 0.0f;
      if (ok) {
        const float* row = p.w[f] + id * p.D;
        for (int d = lane; d < p.D; d += 32) {
          const float e = __ldg(row + d);
          s += e;
          sq = fmaf(e, e, sq);
        }
        if (lane == 0) wide += __ldg(p.wide + p.woff[f] + (long long)id);
      }
      s = warp_sum(s);
      pair = fmaf(s, s, pair);
    }
    sq = warp_sum(sq);
    if (lane == 0) {
      for (int c = 0; c < p.C; ++c) wide = fmaf(__ldg(p.wide + p.coff[c]), load_as_f32(p.csrc[c], b * p.cstride[c], p.cdtype[c]), wide);
      float z = 0.5f * (pair - sq) + wide + (p.wide_bias ? p.wide_bias[0] : 0.0f);
      if (p.addend) z += p.addend[b * p.addend_stride];
      if (p.out_w) z = apply_act(fmaf(z, p.out_w[0], p.out_b ? p.out_b[0] : 0.0f), p.out_act);
      p.out[b] = z;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Training: the head's forward, loss and backward in one pass (mm_deepfm_head_fwd_bwd).  One warp per sample, as the
// forward: the embedding rows are read from the gathered x0 (B, d) at each feature's column (no second lookup), lanes
// stride D; lane f < T reads feature f's id and wide scalar, lane c < C continuous column c; lanes stride the units of h
// (held in registers: h is read once).  Per-CTA sums of the parameter gradients, then one atomic per CTA and quantity.
// ---------------------------------------------------------------------------------------------------------------
constexpr int HB_MAX_U = 512;  // units of h (16 per lane)

struct HeadBwdParams {
  const float* x0;
  long long ldx;
  long long col[MAX_T];  // column of feature f's row in x0
  const void* ids[MAX_T];
  long long rows[MAX_T];
  long long woff[MAX_T];
  unsigned char idb[MAX_T];
  int T;
  const void* csrc[MAX_T];
  long long cstride[MAX_T];
  long long coff[MAX_T];
  int cdtype[MAX_T];
  int C;
  const float* wide;
  const float* wide_bias;
  const float* h;
  long long ldh;
  int U;
  int mask_h;
  const float* w_dl;
  const float* b_dl;
  int act_dl;
  const float* out_w;
  const float* out_b;
  int kind;
  const void* y;
  int y_dtype;
  const float* sw;
  float inv_m;
  float* logits;
  float* loss;  // (2,): [total, the output's loss], accumulated
  float* ds;
  float* dh;
  long long lddh;
  float* dw_out;
  float* db_out;
  float* dw_dl;
  float* db_dl;
  float* dbw;
  float* dcont;
  int* oob;
  long long B;
  int D;
};

__global__ void __launch_bounds__(256) deepfm_head_fwd_bwd_kernel(const __grid_constant__ HeadBwdParams p) {
  constexpr int UC = HB_MAX_U / 32;
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  float wdl[UC], dwl[UC];
#pragma unroll
  for (int c = 0; c < UC; ++c) {
    const int k = lane + 32 * c;
    wdl[c] = k < p.U ? p.w_dl[k] : 0.0f;
    dwl[c] = 0.0f;
  }
  const float wo = p.out_w[0], bo = p.out_b ? p.out_b[0] : 0.0f;
  const float bw = p.wide_bias ? p.wide_bias[0] : 0.0f, bdl = p.b_dl ? p.b_dl[0] : 0.0f;
  const float wc = lane < p.C ? p.wide[p.coff[lane]] : 0.0f;
  float a_loss = 0.f, a_dwo = 0.f, a_dbo = 0.f, a_dbdl = 0.f, a_dbw = 0.f, a_dc = 0.f;
  for (long long b = warp; b < p.B; b += n_warps) {
    const float* xr = p.x0 + b * p.ldx;
    float pair = 0.0f, sq = 0.0f;
    for (int f = 0; f < p.T; ++f) {
      const float* e = xr + p.col[f];
      float s = 0.0f;
      for (int d = lane; d < p.D; d += 32) {
        const float v = e[d];
        s += v;
        sq = fmaf(v, v, sq);
      }
      s = warp_sum(s);
      pair = fmaf(s, s, pair);
    }
    sq = warp_sum(sq);
    float wide = 0.0f, xc = 0.0f;
    if (lane < p.T) {
      const unsigned long long id = (unsigned long long)load_id(p.ids[lane], p.idb[lane], b);
      if (id < (unsigned long long)p.rows[lane]) wide = p.wide[p.woff[lane] + (long long)id];
      else if (p.oob) atomicAdd(p.oob, 1);
    }
    if (lane < p.C) {
      xc = load_as_f32(p.csrc[lane], b * p.cstride[lane], p.cdtype[lane]);
      wide = fmaf(wc, xc, wide);
    }
    wide = warp_sum(wide);
    float hv[UC], u = 0.0f;
#pragma unroll
    for (int c = 0; c < UC; ++c) {
      const int k = lane + 32 * c;
      hv[c] = k < p.U ? p.h[b * p.ldh + k] : 0.0f;
      u = fmaf(hv[c], wdl[c], u);
    }
    u = warp_sum(u) + bdl;
    const bool relu_dl = p.act_dl == MM_ACT_RELU;
    const float s = 0.5f * (pair - sq) + wide + bw + (relu_dl ? fmaxf(u, 0.0f) : u);
    const float z = fmaf(s, wo, bo);
    const float y = load_as_f32(p.y, b, p.y_dtype);
    const float sw = p.sw ? p.sw[b] : 1.0f;
    float l, g;
    head_loss(p.kind, z, y, l, g);
    const float delta = g * sw * p.inv_m;
    const float dsv = delta * wo;
    const float du = (relu_dl && !(u > 0.0f)) ? 0.0f : dsv;
    if (lane == 0) {
      a_loss += l * sw * p.inv_m;
      a_dwo = fmaf(delta, s, a_dwo);
      a_dbo += delta;
      a_dbdl += du;
      a_dbw += dsv;
      p.logits[b] = z;
      p.ds[b] = dsv;
    }
    a_dc = fmaf(dsv, xc, a_dc);
#pragma unroll
    for (int c = 0; c < UC; ++c) {
      const int k = lane + 32 * c;
      if (k < p.U) {
        dwl[c] = fmaf(du, hv[c], dwl[c]);
        p.dh[b * p.lddh + k] = (!p.mask_h || hv[c] > 0.0f) ? du * wdl[c] : 0.0f;
      }
    }
  }
  // per-CTA sums, then one atomic per quantity
  constexpr int NQ = HB_MAX_U + 32 + 5;
  __shared__ float red[8][NQ];
  const int wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int c = 0; c < UC; ++c) red[wid][lane + 32 * c] = dwl[c];
  red[wid][HB_MAX_U + lane] = a_dc;
  if (lane == 0) {
    red[wid][HB_MAX_U + 32] = a_loss;
    red[wid][HB_MAX_U + 33] = a_dwo;
    red[wid][HB_MAX_U + 34] = a_dbo;
    red[wid][HB_MAX_U + 35] = a_dbdl;
    red[wid][HB_MAX_U + 36] = a_dbw;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < NQ; k += blockDim.x) {
    const bool used = k < p.U || (k >= HB_MAX_U && k < HB_MAX_U + p.C) || k >= HB_MAX_U + 32;
    if (!used) continue;
    float s = 0.0f;
    for (int i = 0; i < nw; ++i) s += red[i][k];
    if (k < HB_MAX_U) {
      if (p.dw_dl) atomicAdd(p.dw_dl + k, s);
    } else if (k < HB_MAX_U + 32) {
      if (p.dcont) atomicAdd(p.dcont + (k - HB_MAX_U), s);
    } else if (k == HB_MAX_U + 32) {
      if (p.loss) {
        atomicAdd(p.loss, s);
        atomicAdd(p.loss + 1, s);
      }
    } else if (k == HB_MAX_U + 33) {
      if (p.dw_out) atomicAdd(p.dw_out, s);
    } else if (k == HB_MAX_U + 34) {
      if (p.db_out) atomicAdd(p.db_out, s);
    } else if (k == HB_MAX_U + 35) {
      if (p.db_dl) atomicAdd(p.db_dl, s);
    } else if (p.dbw) {
      atomicAdd(p.dbw, s);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// FM input backward (mm_fm_concat_backward): slice_f[b, :] = sum_a addend_a[b, col_f : col_f + D] + ds[b] (S_f,b - e_f,b)
// with e_f,b = x0[b, col_f : col_f + D] and S_f,b its sum — mm_concat_backward with the FM term as one more addend computed
// from x0, written straight into each table's (B, D) slice.  G lanes (a power of two <= 32) own one row; a warp takes
// 32 / G rows per lap; blockIdx.y = slice.  Columns are arbitrary (continuous columns interleave), so reads are scalar.
// ---------------------------------------------------------------------------------------------------------------
constexpr int FB_MAX_ADD = 4;
constexpr int FB_MAX_SLICES = 64;
struct FmBwdParams {
  const float* add[FB_MAX_ADD];
  long long ld[FB_MAX_ADD];
  int n_add;
  const float* x0;
  long long ldx;
  const float* ds;
  mm_column_slice s[FB_MAX_SLICES];
  long long B;
  int lgG;
};

__global__ void __launch_bounds__(256) fm_concat_backward_kernel(const __grid_constant__ FmBwdParams q) {
  const mm_column_slice& sl = q.s[blockIdx.y];
  const int lane = threadIdx.x & 31, G = 1 << q.lgG, c = lane & (G - 1), sub = lane >> q.lgG, R = 32 >> q.lgG;
  const int D = sl.width;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long base = warp * R; base < q.B; base += n_warps * R) {  // uniform per warp: every lane reaches the shuffles
    const long long b = base + sub;
    const bool valid = b < q.B;
    float e[4], S = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int d = c + j * G;
      e[j] = (valid && d < D) ? q.x0[b * q.ldx + sl.col + d] : 0.0f;
      S += e[j];
    }
    for (int o = G >> 1; o > 0; o >>= 1) S += __shfl_xor_sync(0xffffffffu, S, o);
    if (!valid) continue;
    const float g = q.ds[b];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int d = c + j * G;
      if (d < D) {
        float v = g * (S - e[j]);
        for (int a = 0; a < q.n_add; ++a) v += q.add[a][b * q.ld[a] + sl.col + d];
        sl.dst[b * sl.dst_stride + d] = v;
      }
    }
  }
}

// (B, A, K) -> (B, K): one thread per output element, A strided reads (K contiguous across threads)
__global__ void fm_pairwise_kernel(const float* __restrict__ x, long long B, int A, int K, float* __restrict__ out) {
  const long long total = B * K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / K;
    const int k = (int)(i - b * K);
    const float* base = x + b * A * K + k;
    float s = 0.0f, q = 0.0f;
    for (int a = 0; a < A; ++a) {
      const float v = base[(long long)a * K];
      s += v;
      q = fmaf(v, v, q);
    }
    out[i] = 0.5f * (s * s - q);
  }
}

}  // namespace fm
}  // namespace mm

extern "C" {

int mm_fm_pairwise(const float* x, int64_t B, int A, int K, float* out, void* stream) {
  MM_REQUIRE(x && out && B >= 0 && A >= 1 && K >= 1, MM_ERR_ARG, "mm_fm_pairwise: null pointer or bad shape");
  if (B == 0) return MM_OK;
  long long blocks = (B * K + 255) / 256;
  const long long cap = 16LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  mm::fm::fm_pairwise_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, (long long)B, A, K, out);
  return mm::check_launch("mm_fm_pairwise");
}

int mm_deepfm_head(const mm_lookup_table* tables_host, const int64_t* wide_offsets_host, int n_tables, int64_t B, int D,
                   const mm_concat_piece* cont_host, const int64_t* cont_offsets_host, int n_cont, const float* wide_kernel,
                   const float* wide_bias, const float* addend, int64_t addend_stride, const float* out_w, const float* out_b,
                   int out_act, float* out, int32_t* oob_count, void* stream) {
  using namespace mm::fm;
  MM_REQUIRE(tables_host && wide_offsets_host && wide_kernel && out && B >= 0 && D >= 1, MM_ERR_ARG, "mm_deepfm_head: null pointer or bad shape");
  MM_REQUIRE(n_tables >= 1 && n_tables <= MAX_T && n_cont >= 0 && n_cont <= MAX_T, MM_ERR_UNSUPPORTED,
             "mm_deepfm_head: 1..%d categorical and 0..%d continuous features", MAX_T, MAX_T);
  MM_REQUIRE(n_cont == 0 || (cont_host && cont_offsets_host), MM_ERR_ARG, "mm_deepfm_head: continuous columns without descriptors");
  MM_REQUIRE(out_act >= MM_ACT_LINEAR && out_act <= MM_ACT_GELU, MM_ERR_ARG, "mm_deepfm_head: unknown activation");
  if (B == 0) return MM_OK;
  Params p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < n_tables; ++i) {
    const mm_lookup_table& t = tables_host[i];
    MM_REQUIRE(t.weights && wide_offsets_host[i] >= 0, MM_ERR_ARG, "mm_deepfm_head: table %d: null weights or negative wide offset", i);
    if (const int rc = mm::check_id_column("mm_deepfm_head", i, t.indices, t.idx_bytes, t.rows)) return rc;
    MM_REQUIRE(!t.peer_weights_host, MM_ERR_UNSUPPORTED, "mm_deepfm_head: row-sharded tables are not supported");
    p.w[i] = t.weights;
    p.ids[i] = t.indices;
    p.rows[i] = t.rows;
    p.idb[i] = (unsigned char)t.idx_bytes;
    p.woff[i] = wide_offsets_host[i];
  }
  p.T = n_tables;
  for (int c = 0; c < n_cont; ++c) {
    const mm_concat_piece& pc = cont_host[c];
    MM_REQUIRE(pc.src && pc.width == 1 && pc.src_stride >= 1 && pc.dtype >= MM_I32 && pc.dtype <= MM_F64 && cont_offsets_host[c] >= 0, MM_ERR_ARG,
               "mm_deepfm_head: continuous column %d: null source, width != 1 or bad dtype", c);
    p.csrc[c] = pc.src;
    p.cstride[c] = pc.src_stride;
    p.cdtype[c] = pc.dtype;
    p.coff[c] = cont_offsets_host[c];
  }
  p.C = n_cont;
  p.wide = wide_kernel;
  p.wide_bias = wide_bias;
  p.addend = addend;
  p.addend_stride = addend_stride;
  p.out_w = out_w;
  p.out_b = out_b;
  p.out_act = out_act;
  p.out = out;
  p.oob = oob_count;
  p.B = B;
  p.D = D;
  long long blocks = (B + 7) / 8;
  const long long cap = 8LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  deepfm_head_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(p);
  return mm::check_launch("mm_deepfm_head");
}

int mm_deepfm_head_fwd_bwd(const float* x0, int64_t x0_stride, const int64_t* emb_cols_host, int D, const mm_wide_block* tables_host,
                           int n_tables, const mm_concat_piece* cont_host, const int64_t* cont_offsets_host, int n_cont,
                           const float* wide_kernel, const float* wide_bias, const float* h, int64_t h_stride, int units, int mask_h,
                           const float* w_dl, const float* b_dl, int act_dl, const float* out_w, const float* out_b, int loss_kind,
                           const void* targets, int target_dtype, const float* sample_weight, int64_t B, float* logits, float* loss,
                           float* ds, float* dh, int64_t dh_stride, float* dw_out, float* db_out, float* dw_dl, float* db_dl,
                           float* d_wide_bias, float* d_cont, int32_t* oob_count, void* stream) {
  using namespace mm::fm;
  MM_REQUIRE(x0 && emb_cols_host && tables_host && wide_kernel && h && w_dl && out_w && targets && logits && ds && dh && B >= 0,
             MM_ERR_ARG, "mm_deepfm_head_fwd_bwd: null pointer or negative B");
  MM_REQUIRE(n_tables >= 1 && n_tables <= MAX_T && n_cont >= 0 && n_cont <= MAX_T, MM_ERR_UNSUPPORTED,
             "mm_deepfm_head_fwd_bwd: 1..%d categorical and 0..%d continuous features", MAX_T, MAX_T);
  MM_REQUIRE(n_cont == 0 || (cont_host && cont_offsets_host), MM_ERR_ARG, "mm_deepfm_head_fwd_bwd: continuous columns without descriptors");
  MM_REQUIRE(D >= 1 && units >= 1 && units <= HB_MAX_U, MM_ERR_UNSUPPORTED, "mm_deepfm_head_fwd_bwd: D=%d, units=%d (needs D >= 1, 1 <= units <= %d)",
             D, units, HB_MAX_U);
  MM_REQUIRE(h_stride >= units && dh_stride >= units, MM_ERR_ARG, "mm_deepfm_head_fwd_bwd: h / dh row stride < units");
  MM_REQUIRE(act_dl == MM_ACT_LINEAR || act_dl == MM_ACT_RELU, MM_ERR_UNSUPPORTED, "mm_deepfm_head_fwd_bwd: deep-logit activation must be linear or relu");
  MM_REQUIRE(loss_kind == MM_LOSS_BCE || loss_kind == MM_LOSS_MSE, MM_ERR_ARG, "mm_deepfm_head_fwd_bwd: bad loss kind %d", loss_kind);
  MM_REQUIRE(target_dtype >= MM_I32 && target_dtype <= MM_F64, MM_ERR_ARG, "mm_deepfm_head_fwd_bwd: bad target dtype");
  HeadBwdParams p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < n_tables; ++i) {
    const mm_wide_block& t = tables_host[i];
    MM_REQUIRE(t.offset >= 0 && emb_cols_host[i] >= 0 && emb_cols_host[i] + D <= x0_stride, MM_ERR_ARG,
               "mm_deepfm_head_fwd_bwd: table %d: negative wide offset or its columns outside the x0 row", i);
    if (const int rc = mm::check_id_column("mm_deepfm_head_fwd_bwd", i, t.indices, t.idx_bytes, t.rows)) return rc;
    p.col[i] = emb_cols_host[i];
    p.ids[i] = t.indices;
    p.rows[i] = t.rows;
    p.idb[i] = (unsigned char)t.idx_bytes;
    p.woff[i] = t.offset;
  }
  p.T = n_tables;
  for (int c = 0; c < n_cont; ++c) {
    const mm_concat_piece& pc = cont_host[c];
    MM_REQUIRE(pc.src && pc.width == 1 && pc.src_stride >= 1 && pc.dtype >= MM_I32 && pc.dtype <= MM_F64 && cont_offsets_host[c] >= 0, MM_ERR_ARG,
               "mm_deepfm_head_fwd_bwd: continuous column %d: null source, width != 1 or bad dtype", c);
    p.csrc[c] = pc.src;
    p.cstride[c] = pc.src_stride;
    p.cdtype[c] = pc.dtype;
    p.coff[c] = cont_offsets_host[c];
  }
  p.C = n_cont;
  if (B == 0) return MM_OK;
  p.x0 = x0;
  p.ldx = x0_stride;
  p.wide = wide_kernel;
  p.wide_bias = wide_bias;
  p.h = h;
  p.ldh = h_stride;
  p.U = units;
  p.mask_h = mask_h ? 1 : 0;
  p.w_dl = w_dl;
  p.b_dl = b_dl;
  p.act_dl = act_dl;
  p.out_w = out_w;
  p.out_b = out_b;
  p.kind = loss_kind;
  p.y = targets;
  p.y_dtype = target_dtype;
  p.sw = sample_weight;
  p.inv_m = 1.0f / (float)B;
  p.logits = logits;
  p.loss = loss;
  p.ds = ds;
  p.dh = dh;
  p.lddh = dh_stride;
  p.dw_out = dw_out;
  p.db_out = db_out;
  p.dw_dl = dw_dl;
  p.db_dl = db_dl;
  p.dbw = d_wide_bias;
  p.dcont = d_cont;
  p.oob = oob_count;
  p.B = B;
  p.D = D;
  long long blocks = (B + 7) / 8;
  const long long cap = 8LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  deepfm_head_fwd_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(p);
  return mm::check_launch("mm_deepfm_head_fwd_bwd");
}

int mm_fm_concat_backward(const float* const* addends_host, const int64_t* addend_strides_host, int n_addends, int64_t B, int d,
                          const float* x0, int64_t x0_stride, const float* ds, const mm_column_slice* slices_host, int n_slices,
                          void* stream) {
  using namespace mm::fm;
  MM_REQUIRE(x0 && ds && slices_host && B >= 0 && d >= 1 && x0_stride >= d && (n_addends == 0 || (addends_host && addend_strides_host)),
             MM_ERR_ARG, "mm_fm_concat_backward: null pointer, d < 1 or x0_stride < d");
  MM_REQUIRE(n_addends >= 0 && n_addends <= FB_MAX_ADD, MM_ERR_ARG, "mm_fm_concat_backward: n_addends=%d outside [0, %d]", n_addends, FB_MAX_ADD);
  MM_REQUIRE(n_slices >= 1 && n_slices <= FB_MAX_SLICES, MM_ERR_ARG, "mm_fm_concat_backward: n_slices=%d outside [1, %d]", n_slices, FB_MAX_SLICES);
  FmBwdParams q;
  memset(&q, 0, sizeof(q));
  for (int a = 0; a < n_addends; ++a) {
    MM_REQUIRE(addends_host[a] && addend_strides_host[a] >= d, MM_ERR_ARG, "mm_fm_concat_backward: addend %d: null or stride < d", a);
    q.add[a] = addends_host[a];
    q.ld[a] = addend_strides_host[a];
  }
  const int D = slices_host[0].width;
  for (int t = 0; t < n_slices; ++t) {
    const mm_column_slice& s = slices_host[t];
    MM_REQUIRE(s.dst && s.width == D && D >= 1 && D <= 128 && s.col >= 0 && (int64_t)s.col + s.width <= d, MM_ERR_ARG,
               "mm_fm_concat_backward: slice %d: null destination, width != %d (1..128, one width for all) or columns outside [0, d)", t, D);
    MM_REQUIRE(s.dst_stride >= s.width, MM_ERR_ARG, "mm_fm_concat_backward: slice %d: destination row stride < width", t);
    q.s[t] = s;
  }
  q.n_add = n_addends;
  q.x0 = x0;
  q.ldx = x0_stride;
  q.ds = ds;
  q.B = B;
  int G = 4;
  while (G < 32 && G < D) G <<= 1;
  while ((1 << q.lgG) < G) ++q.lgG;
  if (B == 0) return MM_OK;
  const long long rows_per_cta = 8LL * (32 / G);
  long long blocks = (B + rows_per_cta - 1) / rows_per_cta;
  long long cap = 16LL * mm::sm_count() / n_slices;
  if (cap < 1) cap = 1;
  if (blocks > cap) blocks = cap;
  fm_concat_backward_kernel<<<dim3((unsigned)blocks, (unsigned)n_slices), 256, 0, (cudaStream_t)stream>>>(q);
  return mm::check_launch("mm_fm_concat_backward");
}

}  // extern "C"
