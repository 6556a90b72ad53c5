// Pairwise dot-product interaction (DLRM), standalone and fused with the embedding gather.
// Replaces tf.matmul(x, x^T) + band_part + boolean_mask (merlin/models/tf/blocks/interaction.py:
// 86-116), StackFeatures (core/aggregation.py:101-108) and the [bottom | interactions] concat
// (blocks/dlrm.py:126-130).  HBM-bound by design: every input row is read once (cp.async into
// shared memory, no register staging), the (B,F,F) Gram matrix never exists, the output row is
// assembled in shared memory and written with coalesced 128-bit stores.
#include <cstring>

#include "mm_common.cuh"

namespace mm {

bool use_imma_v1();

namespace imma2 {  // interaction_v2.cu: second-generation warp-per-sample kernel (packed ids, sharded tables)
template <int MODE>
int launch(const float* x, int64_t x_stride, const LookupParams& lk, const float* prefix, int64_t prefix_stride, int P,
           int bottom_slot, int64_t B, int F, int D, float* out_f32, int64_t out_stride, void* out_split, int out_Kp,
           int32_t* oob, cudaStream_t st, const char* who, bool presplit);
}
namespace imma {  // interaction_mma.cu: warp-level mma.sync path (F <= 32, D in {16,32,64,128})
template <int MODE, typename IdxT>
int launch(const float* x, int64_t x_stride, const GatherParams& gp, const float* prefix, int64_t prefix_stride,
           int P, int bottom_slot, int64_t B, int F, int D, float* out_f32, int64_t out_stride, void* out_split,
           int out_Kp, int32_t* oob, cudaStream_t st, const char* who);
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// index of pair (i,j), i<j (or i<=j with self interaction), row-major over the upper triangle
__device__ __forceinline__ int pair_index(int i, int j, int F, int self) {
  return self ? i * F - (i * (i - 1)) / 2 + (j - i) : i * (2 * F - i - 1) / 2 + (j - i - 1);
}

// Shared-memory plan (floats): xs[G][F][DS] | os[G][OWP] | (fused) idx as long long [G][T]
// Compute: 3x3 register blocks over the upper triangle of the FxF Gram matrix; a task is
// (sample g, block pair bp); tasks are flattened over the CTA so all lanes stay busy.
template <int MODE /*0 = x from HBM stack, 1 = gather rows from tables*/, typename IdxT>
__global__ void __launch_bounds__(128)
interact_kernel(const float* __restrict__ x, long long x_stride, const __grid_constant__ GatherParams p,
                const float* __restrict__ prefix, long long prefix_stride, int P, int bottom_slot,
                long long B, int F, int D, int G, int self_inter, float* __restrict__ out,
                long long out_stride, int* __restrict__ oob_count) {
  extern __shared__ __align__(16) float smem[];
  const int DS = D + 4;
  const int npairs = self_inter ? F * (F + 1) / 2 : F * (F - 1) / 2;
  const int OW = P + npairs;
  const int OWP = (OW + 3) & ~3;
  float* xs = smem;
  float* os = xs + (size_t)G * F * DS;
  long long* idx_s = reinterpret_cast<long long*>(os + (size_t)G * OWP);
  const int nb = (F + 2) / 3;
  const int nbp = nb * (nb + 1) / 2;
  const int V = D >> 2;
  const int tid = threadIdx.x, nth = blockDim.x;

  for (long long b0 = (long long)blockIdx.x * G; b0 < B; b0 += (long long)gridDim.x * G) {
    const int gcount = (int)((B - b0) < G ? (B - b0) : G);
    // ---- load phase -------------------------------------------------------------------
    if (MODE == 0) {
      const int total = gcount * F * V;
      for (int e = tid; e < total; e += nth) {
        const int v = e % V, f = (e / V) % F, g = e / (V * F);
        cp_async16(xs + ((size_t)g * F + f) * DS + v * 4, x + (b0 + g) * x_stride + (size_t)f * D + v * 4);
      }
    } else {
      const int T = p.n_tables;
      for (int e = tid; e < gcount * T; e += nth) {
        const int g = e % gcount, t = e / gcount;  // consecutive threads -> consecutive samples
        long long id = (long long)reinterpret_cast<const IdxT*>(p.t[t].indices)[b0 + g];
        if (id < 0 || id >= p.t[t].rows) {
          id = -1;
          if (oob_count) atomicAdd(oob_count, 1);
        }
        idx_s[g * T + t] = id;
      }
      __syncthreads();
      const int total = gcount * T * V;
      for (int e = tid; e < total; e += nth) {
        const int v = e % V, t = (e / V) % T, g = e / (V * T);
        const long long id = idx_s[g * T + t];
        const int slot = p.t[t].out_col / D;
        float* dst = xs + ((size_t)g * F + slot) * DS + v * 4;
        if (id >= 0) cp_async16(dst, p.t[t].weights + id * D + v * 4);
        else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (bottom_slot >= 0) {
        for (int e = tid; e < gcount * V; e += nth) {
          const int v = e % V, g = e / V;
          cp_async16(xs + ((size_t)g * F + bottom_slot) * DS + v * 4,
                     prefix + (b0 + g) * prefix_stride + v * 4);
        }
      }
    }
    // prefix (shortcut branch) goes to the head of the output row
    if (P > 0) {
      for (int e = tid; e < gcount * P; e += nth) {
        const int c = e % P, g = e / P;
        os[(size_t)g * OWP + c] = prefix[(b0 + g) * prefix_stride + c];
      }
    }
    cp_async_commit_wait_all();
    __syncthreads();

    // ---- compute phase ----------------------------------------------------------------
    const int tasks = gcount * nbp;
    for (int task = tid; task < tasks; task += nth) {
      const int g = task / nbp;
      int bp = task % nbp;
      // decode (bi <= bj) from bp, rows of the block-pair triangle have nb, nb-1, ... entries
      int bi = 0, rowlen = nb;
      while (bp >= rowlen) {
        bp -= rowlen;
        ++bi;
        --rowlen;
      }
      const int bj = bi + bp;
      const float* xg = xs + (size_t)g * F * DS;
      int ri[3], rj[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        ri[a] = min(3 * bi + a, F - 1);
        rj[a] = min(3 * bj + a, F - 1);
      }
      float acc[3][3];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[a][c] = 0.0f;
      for (int v = 0; v < V; ++v) {
        float4 av[3], bv[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          av[a] = *reinterpret_cast<const float4*>(xg + ri[a] * DS + v * 4);
          bv[a] = *reinterpret_cast<const float4*>(xg + rj[a] * DS + v * 4);
        }
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            acc[a][c] = fmaf(av[a].x, bv[c].x, acc[a][c]);
            acc[a][c] = fmaf(av[a].y, bv[c].y, acc[a][c]);
            acc[a][c] = fmaf(av[a].z, bv[c].z, acc[a][c]);
            acc[a][c] = fmaf(av[a].w, bv[c].w, acc[a][c]);
          }
      }
      float* og = os + (size_t)g * OWP + P;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int i = 3 * bi + a, j = 3 * bj + c;
          if (i < F && j < F && (i < j || (self_inter && i == j)))
            og[pair_index(i, j, F, self_inter)] = acc[a][c];
        }
    }
    __syncthreads();

    // ---- store phase: coalesced row writes ----------------------------------------------
    if ((out_stride & 3) == 0 && ((uintptr_t)out & 15) == 0) {
      const int OW4 = OW >> 2;
      for (int e = tid; e < gcount * OW4; e += nth) {
        const int c = e % OW4, g = e / OW4;
        stg_stream(reinterpret_cast<float4*>(out + (b0 + g) * out_stride) + c,
                   *reinterpret_cast<const float4*>(os + (size_t)g * OWP + c * 4));
      }
      const int rem = OW & 3;
      for (int e = tid; e < gcount * rem; e += nth) {
        const int c = OW4 * 4 + e % rem, g = e / rem;
        out[(b0 + g) * out_stride + c] = os[(size_t)g * OWP + c];
      }
    } else {
      for (int e = tid; e < gcount * OW; e += nth) {
        const int c = e % OW, g = e / OW;
        out[(b0 + g) * out_stride + c] = os[(size_t)g * OWP + c];
      }
    }
    __syncthreads();  // smem is reused by the next tile
  }
}

static size_t interact_smem(int G, int F, int D, int OW, int T) {
  const int OWP = (OW + 3) & ~3;
  return ((size_t)G * F * (D + 4) + (size_t)G * OWP) * sizeof(float) + (size_t)G * T * sizeof(long long);
}

template <int MODE, typename IdxT>
static int launch_interact(const float* x, int64_t x_stride, const GatherParams& p,
                           const float* prefix, int64_t prefix_stride, int P, int bottom_slot,
                           int64_t B, int F, int D, int self_inter, float* out, int64_t out_stride,
                           int32_t* oob, cudaStream_t st, const char* who) {
  const int npairs = self_inter ? F * (F + 1) / 2 : F * (F - 1) / 2;
  const int OW = P + npairs;
  const int T = MODE ? p.n_tables : 0;
  // samples per CTA: fill ~56 KB so that 3-4 CTAs are resident per SM (load/compute overlap)
  int G = 1;
  while (G < 16 && interact_smem(G + 1, F, D, OW, T) <= 56 * 1024) ++G;
  const size_t smem = interact_smem(G, F, D, OW, T);
  MM_REQUIRE(smem <= 200 * 1024, MM_ERR_UNSUPPORTED,
             "%s: F=%d D=%d needs %zu B of shared memory per sample (> 200 KB)", who, F, D, smem);
  auto kern = interact_kernel<MODE, IdxT>;
  static size_t smem_set = 0;  // per template instantiation
  if (smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute(200 KB smem) failed: %s", who, cudaGetErrorString(e));
      return (int)e;
    }
    smem_set = 200 * 1024;
  }
  long long tiles = (B + G - 1) / G;
  const long long cap = (long long)sm_count() * 4 * 8;
  const unsigned blocks = (unsigned)(tiles < cap ? tiles : cap);
  kern<<<blocks, 128, smem, st>>>(x, x_stride, p, prefix, prefix_stride, P, bottom_slot, B, F, D, G,
                                  self_inter, out, out_stride, oob);
  return check_launch(who);
}

bool use_imma_v1() {  // MM_IMMA_V1=1: first-generation kernel (interaction_mma.cu), kept for A/B measurements
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("MM_IMMA_V1");
    v = (e && e[0] == '1') ? 1 : 0;
  }
  return v == 1;
}

}  // namespace mm

extern "C" {

int mm_dlrm_lookup_interact(const mm_lookup_table* tables_host, int n_tables, int64_t B, int D, int rank, int world,
                            const float* bottom, int64_t bottom_stride, int bottom_slot, float* out,
                            int64_t out_stride, void* out_split, int out_Kp, int32_t* oob_count, int row_format,
                            void* stream) {
  const char* who = "mm_dlrm_lookup_interact";
  MM_REQUIRE(row_format == MM_ROWS_F32 || row_format == MM_ROWS_OPERAND, MM_ERR_ARG, "%s: bad row_format", who);
  MM_REQUIRE(row_format == MM_ROWS_F32 || (out_split && !out), MM_ERR_ARG,
             "%s: operand-format rows need the split-bf16 output (the fp32 prefix cannot be rebuilt exactly)", who);
  MM_REQUIRE(tables_host && n_tables > 0 && (out || out_split) && B >= 0, MM_ERR_ARG, "%s: bad table list / null out / B<0", who);
  MM_REQUIRE(!(out && out_split), MM_ERR_ARG, "%s: give either out or out_split", who);
  MM_REQUIRE(D == 16 || D == 32 || D == 64 || D == 128, MM_ERR_UNSUPPORTED, "%s: D must be 16, 32, 64 or 128", who);
  MM_REQUIRE(world >= 1 && world <= mm::MM_LOOKUP_MAX_WORLD && rank >= 0 && rank < world, MM_ERR_ARG,
             "%s: world must be 1..%d and 0 <= rank < world", who, mm::MM_LOOKUP_MAX_WORLD);
  const int F = n_tables + (bottom ? 1 : 0);
  MM_REQUIRE(F >= 2 && F <= mm::MM_LOOKUP_MAX_ROWS, MM_ERR_UNSUPPORTED, "%s: 2..%d feature slots", who, mm::MM_LOOKUP_MAX_ROWS);
  MM_REQUIRE(!bottom || (bottom_slot >= 0 && bottom_slot < F && bottom_stride >= D && bottom_stride % 4 == 0 &&
                         ((uintptr_t)bottom % 16) == 0),
             MM_ERR_ARG, "%s: bad bottom slot / stride / alignment", who);
  mm::LookupParams lk;
  memset(&lk, 0, sizeof(lk));
  lk.world = world;
  lk.log2_world = -1;
  for (int b = 0; b < 4; ++b)
    if ((1 << b) == world) lk.log2_world = b;
  unsigned seen = bottom ? (1u << bottom_slot) : 0u;
  for (int t = 0; t < n_tables; ++t) {
    const mm_lookup_table& tb = tables_host[t];
    const int r = tb.slot;
    MM_REQUIRE(tb.weights && tb.indices && tb.rows > 0 && r >= 0 && r < F && ((uintptr_t)tb.weights % 16) == 0, MM_ERR_ARG,
               "%s: table %d: null pointer, rows <= 0, bad slot or misaligned weights", who, t);
    MM_REQUIRE(!(seen & (1u << r)), MM_ERR_ARG, "%s: slot %d used twice", who, r);
    seen |= 1u << r;
    const int w = tb.idx_bytes;
    MM_REQUIRE(w == 1 || w == 2 || w == 3 || w == 4 || w == 8, MM_ERR_ARG, "%s: table %d: idx_bytes must be 1, 2, 3, 4 or 8", who, t);
    MM_REQUIRE(w >= 4 || tb.rows <= (1ll << (8 * w)), MM_ERR_ARG, "%s: table %d: %lld rows do not fit %d-byte ids", who, t,
               (long long)tb.rows, w);
    MM_REQUIRE((w != 4 && w != 8) || ((uintptr_t)tb.indices % w) == 0, MM_ERR_ALIGN, "%s: table %d: misaligned ids", who, t);
    lk.weights[r] = tb.weights;
    lk.indices[r] = tb.indices;
    lk.rows[r] = tb.rows;
    lk.idx_bytes[r] = (unsigned char)w;
    if (tb.peer_weights_host) {
      MM_REQUIRE(world > 1, MM_ERR_ARG, "%s: table %d is sharded but world == 1", who, t);
      lk.sharded[r] = 1;
      for (int k = 0; k < world; ++k) {
        MM_REQUIRE(tb.peer_weights_host[k] && ((uintptr_t)tb.peer_weights_host[k] % 16) == 0, MM_ERR_ARG,
                   "%s: table %d: null / misaligned shard pointer of rank %d", who, t, k);
        lk.peers[r * world + k] = tb.peer_weights_host[k];
      }
      MM_REQUIRE(tb.peer_weights_host[rank] == tb.weights, MM_ERR_ARG, "%s: table %d: peer_weights_host[rank] != weights", who, t);
    }
  }
  const int P = bottom ? D : 0;
  MM_REQUIRE(!out || out_stride >= P + F * (F - 1) / 2, MM_ERR_ARG, "%s: out_stride too small", who);
  MM_REQUIRE(!out_split || (out_Kp % 64 == 0 && out_Kp >= P + F * (F - 1) / 2 && ((uintptr_t)out_split % 16) == 0), MM_ERR_ARG,
             "%s: out_Kp must be a multiple of 64 >= the row width, out_split 16-B aligned", who);
  if (B == 0) return MM_OK;
  const int rc = mm::imma2::launch<1>(nullptr, 0, lk, bottom, bottom_stride, P, bottom ? bottom_slot : -1, B, F, D, out,
                                      out_stride, out_split, out_Kp, oob_count, (cudaStream_t)stream, who,
                                      row_format == MM_ROWS_OPERAND);
  MM_REQUIRE(rc != MM_ERR_UNSUPPORTED, MM_ERR_UNSUPPORTED, "%s: shape outside the fused kernel (F=%d, D=%d)", who, F, D);
  return rc;
}

int mm_dot_interaction(const float* x, int64_t B, int F, int D, int64_t x_stride,
                       const float* prefix, int P, int64_t prefix_stride, int self_interaction,
                       float* out, int64_t out_stride, void* out_split, int out_Kp, void* stream) {
  MM_REQUIRE(x && (out || out_split) && B >= 0 && F >= 1 && D >= 4, MM_ERR_ARG,
             "mm_dot_interaction: null pointer, B<0, F<1 or D<4");
  MM_REQUIRE(!(out && out_split), MM_ERR_ARG, "mm_dot_interaction: give either out or out_split");
  MM_REQUIRE(D % 4 == 0 && x_stride % 4 == 0 && ((uintptr_t)x % 16) == 0, MM_ERR_ALIGN,
             "mm_dot_interaction: D and x_stride must be multiples of 4 floats and x 16-B aligned");
  MM_REQUIRE(x_stride >= (int64_t)F * D, MM_ERR_ARG, "mm_dot_interaction: x_stride < F*D");
  MM_REQUIRE((P == 0) || (prefix != nullptr && prefix_stride >= P), MM_ERR_ARG,
             "mm_dot_interaction: P>0 requires a prefix pointer with stride >= P");
  const int npairs = self_interaction ? F * (F + 1) / 2 : F * (F - 1) / 2;
  MM_REQUIRE(!out || out_stride >= P + npairs, MM_ERR_ARG, "mm_dot_interaction: out_stride %lld < %d",
             (long long)out_stride, P + npairs);
  MM_REQUIRE(!out_split || (out_Kp % 64 == 0 && out_Kp >= P + npairs && ((uintptr_t)out_split % 16) == 0), MM_ERR_ARG,
             "mm_dot_interaction: out_Kp must be a multiple of 64 >= %d and out_split 16-B aligned", P + npairs);
  if (B == 0) return MM_OK;
  mm::GatherParams p;
  memset(&p, 0, sizeof(p));
  if (!self_interaction && !mm::use_imma_v1()) {
    mm::LookupParams lk;
    memset(&lk, 0, sizeof(lk));
    lk.world = 1;
    const int rc2 = mm::imma2::launch<0>(x, x_stride, lk, prefix, prefix_stride, P, -1, B, F, D, out, out_stride, out_split,
                                         out_Kp, nullptr, (cudaStream_t)stream, "mm_dot_interaction", false);
    if (rc2 != MM_ERR_UNSUPPORTED) return rc2;
  }
  if (!self_interaction) {
    const int rc = mm::imma::launch<0, int32_t>(x, x_stride, p, prefix, prefix_stride, P, -1, B, F, D, out, out_stride,
                                                out_split, out_Kp, nullptr, (cudaStream_t)stream, "mm_dot_interaction");
    if (rc != MM_ERR_UNSUPPORTED) return rc;
  }
  MM_REQUIRE(out != nullptr, MM_ERR_UNSUPPORTED,
             "mm_dot_interaction: split-bf16 output needs the tensor-core path (F<=32, D%%16==0, P in {0,D})");
  return mm::launch_interact<0, int32_t>(x, x_stride, p, prefix, prefix_stride, P, -1, B, F, D,
                                         self_interaction ? 1 : 0, out, out_stride, nullptr,
                                         (cudaStream_t)stream, "mm_dot_interaction");
}

int mm_dlrm_gather_interact(const mm_gather_table* tables_host, int n_tables, int idx_dtype,
                            int64_t B, int D, const float* bottom, int64_t bottom_stride,
                            int bottom_slot, float* out, int64_t out_stride, void* out_split,
                            int out_Kp, int32_t* oob_count, void* stream) {
  MM_REQUIRE(tables_host && n_tables > 0 && n_tables <= MM_MAX_TABLES && (out || out_split) && B >= 0, MM_ERR_ARG,
             "mm_dlrm_gather_interact: bad table list / null out / B<0");
  MM_REQUIRE(!(out && out_split), MM_ERR_ARG, "mm_dlrm_gather_interact: give either out or out_split");
  MM_REQUIRE(D >= 4 && D % 4 == 0, MM_ERR_ALIGN, "mm_dlrm_gather_interact: D must be a multiple of 4");
  MM_REQUIRE(idx_dtype == MM_I32 || idx_dtype == MM_I64, MM_ERR_ARG,
             "mm_dlrm_gather_interact: bad idx_dtype");
  const int F = n_tables + (bottom ? 1 : 0);
  MM_REQUIRE(F <= 64, MM_ERR_UNSUPPORTED, "mm_dlrm_gather_interact: at most 64 feature slots");
  MM_REQUIRE(!bottom || (bottom_slot >= 0 && bottom_slot < F && bottom_stride >= D &&
                         bottom_stride % 4 == 0 && ((uintptr_t)bottom % 16) == 0),
             MM_ERR_ARG, "mm_dlrm_gather_interact: bad bottom slot / stride / alignment");
  unsigned long long seen = 0;
  if (bottom) seen |= 1ull << bottom_slot;
  for (int t = 0; t < n_tables; ++t) {
    const mm_gather_table& tb = tables_host[t];
    MM_REQUIRE(tb.weights && tb.indices && tb.rows > 0 && tb.dim == D && tb.out_col % D == 0 &&
                   tb.out_col / D < F && ((uintptr_t)tb.weights % 16) == 0,
               MM_ERR_ARG, "mm_dlrm_gather_interact: table %d: dim != D, bad slot or misaligned", t);
    MM_REQUIRE(!(seen & (1ull << (tb.out_col / D))), MM_ERR_ARG,
               "mm_dlrm_gather_interact: slot %d used twice", tb.out_col / D);
    seen |= 1ull << (tb.out_col / D);
  }
  const int P = bottom ? D : 0;
  MM_REQUIRE(!out || out_stride >= P + F * (F - 1) / 2, MM_ERR_ARG,
             "mm_dlrm_gather_interact: out_stride too small");
  MM_REQUIRE(!out_split || (out_Kp % 64 == 0 && out_Kp >= P + F * (F - 1) / 2 && ((uintptr_t)out_split % 16) == 0),
             MM_ERR_ARG, "mm_dlrm_gather_interact: out_Kp must be a multiple of 64 >= the row width, out_split 16-B aligned");
  if (B == 0) return MM_OK;
  mm::GatherParams p;
  memset(&p, 0, sizeof(p));
  p.n_tables = n_tables;
  for (int t = 0; t < n_tables; ++t) p.t[t] = tables_host[t];
  cudaStream_t st = (cudaStream_t)stream;
  if (!mm::use_imma_v1() && F <= mm::MM_LOOKUP_MAX_ROWS) {
    mm::LookupParams lk;
    memset(&lk, 0, sizeof(lk));
    lk.world = 1;
    for (int t = 0; t < n_tables; ++t) {
      const int r = tables_host[t].out_col / D;
      lk.weights[r] = tables_host[t].weights;
      lk.indices[r] = tables_host[t].indices;
      lk.rows[r] = tables_host[t].rows;
      lk.idx_bytes[r] = idx_dtype == MM_I32 ? 4 : 8;
    }
    const int rc2 = mm::imma2::launch<1>(nullptr, 0, lk, bottom, bottom_stride, P, bottom ? bottom_slot : -1, B, F, D, out,
                                         out_stride, out_split, out_Kp, oob_count, st, "mm_dlrm_gather_interact", false);
    if (rc2 != MM_ERR_UNSUPPORTED) return rc2;
  }
  {
    const int bs = bottom ? bottom_slot : -1;
    const int rc = idx_dtype == MM_I32
                       ? mm::imma::launch<1, int32_t>(nullptr, 0, p, bottom, bottom_stride, P, bs, B, F, D, out, out_stride,
                                                      out_split, out_Kp, oob_count, st, "mm_dlrm_gather_interact")
                       : mm::imma::launch<1, int64_t>(nullptr, 0, p, bottom, bottom_stride, P, bs, B, F, D, out, out_stride,
                                                      out_split, out_Kp, oob_count, st, "mm_dlrm_gather_interact");
    if (rc != MM_ERR_UNSUPPORTED) return rc;
  }
  MM_REQUIRE(out != nullptr, MM_ERR_UNSUPPORTED,
             "mm_dlrm_gather_interact: split-bf16 output needs the tensor-core path (F<=32, D%%16==0)");
  return idx_dtype == MM_I32
             ? mm::launch_interact<1, int32_t>(nullptr, 0, p, bottom, bottom_stride, P,
                                               bottom ? bottom_slot : -1, B, F, D, 0, out,
                                               out_stride, oob_count, st, "mm_dlrm_gather_interact")
             : mm::launch_interact<1, int64_t>(nullptr, 0, p, bottom, bottom_stride, P,
                                               bottom ? bottom_slot : -1, B, F, D, 0, out,
                                               out_stride, oob_count, st, "mm_dlrm_gather_interact");
}

}  // extern "C"
