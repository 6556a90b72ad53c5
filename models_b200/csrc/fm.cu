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

}  // extern "C"
