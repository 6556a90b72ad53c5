// In-batch losses over the (B, N) query x negative scores without materialising them: a flash-attention-style pass that
// recomputes every 128x128 score tile from the split-bf16 operands the forward read and, in registers, either reduces it
// into per-row statistics or turns it into the gradient tile G and multiplies G straight into the operand tile still
// resident in shared memory.  One CTA body, templated on the loss and on what it computes (MODE):
//
//   DQ   one CTA per 128 queries (resident), streams the negatives:   S = Q N^T,   dQ += G N
//   DN   one CTA per 128 negatives (resident), streams the queries:   S^T = N Q^T, dN += G^T Q
//   FWD  pairwise losses only: one CTA per 128 queries, streams the negatives: per-row statistics [row loss, dloss/dsp,
//        lse, A]; the -max kinds stream the negatives twice (pass 1: the row's log-sum-exp, which the eps0 decision of
//        pass 2 needs)
//
// The losses:
//   SoftmaxCE       backward of the in-batch soft-max cross-entropy (mm_inbatch_softmax_ce): G = c (softmax - onehot) / T
//                   from the forward's logQ, id mask, temperature and log-sum-exp, so exp(s - lse) is consistent with its
//                   statistics
//   Pairwise<KIND>  BPR, BPR-max, TOP1, TOP1-v2, TOP1-max, logistic, hinge (the reference's losses/pairwise.py; element
//                   functions in pairwise.cuh): G = c / T dloss/ds with c = 1 / (B N) (Keras' SUM_OVER_BATCH_SIZE over
//                   the (B, N) per-element losses; top1_v2's per-row mean over N and batch mean over B give the same c)
//   CatalogCE       backward of the full-catalog soft-max cross-entropy (CategoricalOutput over a weight-tied table): the
//                   queries are x / T, the streamed "negatives" are the catalog rows, the tempered bias b / T is a column
//                   value and the one-hot compares the column index with the row's label in registers.  DQ: G = c / T
//                   (softmax - onehot), dX = G E; DN: G = c (softmax - onehot), dE = G^T (x / T), db = 1 / T sum_b G.
//                   DQ may split the catalog over gridDim.y CTAs per query tile (partial dX, summed in a fixed order)
//   SmoothedCatalogCE  CatalogCE against the label-smoothed target (1 - eps) onehot + eps / N: the one-hot weighs 1 - eps
//                   and the uniform part's rank-one terms are added in the epilogue from fixed-order column sums
// and inbatch_loss_kernel adds any of the losses from the per-row statistics in a fixed order (one CTA).
//
// Two warpgroups (64 resident rows each) over a TMA ring of streamed tiles: the forward catalog kernel's structure
// (catalog_tc.cu) without its producer warp.  The scores use the forward's 3-pass split-bf16 products.  The second product
// takes G as the register A operand (split hi / lo, 3 passes) and the streamed tile as an MN-major B operand (wgmma's
// transpose bit for 16-bit types), so no transposed copy of either operand exists.  Every output row is owned by one CTA:
// no atomics, bit-reproducible.
#include <type_traits>

#include "pairwise.cuh"
#include "tc_common.cuh"

extern "C" int mm_tc_padded_k(int K);

namespace mm {
namespace flash {

using namespace mm::tc;

constexpr int BM = 128, BN = 128, BLOCK_K = 64, MMA_K = 16;
constexpr int kThreads = 256;  // two warpgroups of 64 resident rows each; thread 0 also issues the TMA loads
constexpr uint32_t TILE_BYTES = 128 * BLOCK_K * 2;  // one 128-row x 64-col bf16 tile = 16 KB
constexpr float LOG2E = 1.4426950408889634f;
constexpr int FWD = 0, DQ = 1, DN = 2;
constexpr int kColVals = 3;        // per-tile column values staged in shared memory (at most; the loss says how many)
constexpr int kColStride = 2 * BN;  // floats between two column values of one column (each double-buffered)

struct Params {
  long long M, I;  // resident rows, streamed rows
  int D, stages, n_tiles;
  const void* row_ids;  // ids of the resident rows / streamed rows (null: no down-scoring)
  const void* col_ids;
  int id_is64;
  float inv_temp;
  float masked_score, lambda, c;  // pairwise: a down-scored column's score (already / T), reg_lambda, 1 / (B N)
  const float* neg_prob;          // soft-max: (N,) sampling probabilities (logQ) or null
  const float* row_scale;         // soft-max: (B,) or one float c
  int scale_is_scalar;
  const float* pos_logit;  // pairwise: (B,) the positive scores sp (already / T)
  float* stats;            // soft-max: (B, 3) [max, lse, positive logit]; pairwise: (B, 4) [row loss, dloss/dsp, lse, A]
  const float* q;          // (B, D) fp32
  const float* pos;        // (B, D) fp32
  float* out;              // dq (B, D) or dneg (N, D)
  float* dpos;             // dq kernel: dpos when it is its own buffer; dn kernel: non-null = dpos aliases dneg (add g0 q)
  // catalog soft-max only (null / unused for the other losses)
  const void* labels;   // (B,) class ids, id_is64 wide
  const float* bias;    // (N,) the tempered bias b / T, or null
  float* db;            // dn kernel: (N,) bias gradient, or null
  int tiles_per_split;  // dq kernel: streamed tiles per CTA of a query tile (gridDim.y CTAs share one)
  int* oob;             // dq kernel: labels outside [0, N) are counted here (null: not counted)
  // label-smoothed catalog soft-max only (SmoothedCatalogCE)
  float keep;           // 1 - eps: the one-hot's weight in the smoothed target
  const float* ls_e;    // [kAux]: (eps / N) sum_j e_j per column, (eps / N) sum_j b_j / T at kAuxExtra
  const float* ls_x;    // [kAux]: (eps / N) sum_b c_b x_b / T per column, (eps / N) sum_b c_b at kAuxExtra
};

// the label-smoothing vectors: 128 columns and one extra sum at kAuxExtra, padded to kAux floats
constexpr int kAux = 160, kAuxExtra = 128;

// The catalog kernels stream up to N / 128 tiles into one wgmma fp32 accumulator, which loses magnitude over millions of
// additions (dx of a 10 M catalog in 4 splits came out 0.2 % small).  Every kFlushTiles tiles a CTA adds its accumulator
// into its own output rows (read, add, write: each row has one owner) and restarts it from zero.
constexpr int kFlushTiles = 256;

__device__ __forceinline__ long long id_at(const void* p, long long i, int is64) {
  return is64 ? reinterpret_cast<const long long*>(p)[i] : (long long)reinterpret_cast<const int*>(p)[i];
}

// ---- the losses: what the body reads per resident row (`row_vals`, kept in registers) and per streamed column
// (`col_vals`, staged in shared memory per tile, `cols` of them), the score of an element, its gradient and the
// epilogue's g0 (the gradient of the row's positive score).  Column value k of the element's column is
// c[k * kColStride]. ----

struct SoftmaxCE {
  static constexpr bool kTwoPass = false;
  static constexpr bool kCatalog = false;
  static constexpr bool kSmooth = false;
  __device__ __forceinline__ static float logq_bias(const float* prob, long long n) {  // the forward's -log(p + 1e-16)
    return prob ? -logf(prob[n] + 1e-16f) : 0.0f;
  }
  __device__ __forceinline__ static float scale_of(const Params& p, long long b) {  // c[b] / T
    return (p.scale_is_scalar ? p.row_scale[0] : p.row_scale[b]) * p.inv_temp;
  }
  template <int MODE>
  static constexpr int cols() {
    return MODE == DN ? 2 : 1;
  }
  // DQ: the query's [lse, c/T]; DN: the negative's [logQ bias]
  template <int MODE>
  __device__ __forceinline__ static void row_vals(const Params& p, long long r, float (&v)[3]) {
    if (MODE == DN) {
      v[0] = logq_bias(p.neg_prob, r);
    } else {
      v[0] = p.stats[r * 3 + 1];
      v[1] = scale_of(p, r);
    }
  }
  // DQ: the negative's [logQ bias]; DN: the query's [lse, c/T]
  template <int MODE>
  __device__ __forceinline__ static void col_vals(const Params& p, long long c, float (&v)[3]) {
    if (MODE == DN) {
      v[0] = p.stats[c * 3 + 1];
      v[1] = scale_of(p, c);
    } else {
      v[0] = logq_bias(p.neg_prob, c);
    }
  }
  template <int MODE>
  __device__ __forceinline__ static float score(const Params& p, float a, const float (&r)[3], const float* c) {
    return (a + (MODE == DN ? r[0] : c[0])) * p.inv_temp;
  }
  // c/T softmax
  template <int MODE>
  __device__ __forceinline__ static float grad(const Params& p, float s, const float (&r)[3], const float* c) {
    const float lse = MODE == DN ? c[0] : r[0];
    const float sc = MODE == DN ? c[kColStride] : r[1];
    return sc * ex2_approx((s - lse) * LOG2E);
  }
  // g[b, 0] = c[b] (p[b, 0] - 1) / T
  __device__ __forceinline__ static float g0(const Params& p, long long b) {
    const float lse = p.stats[b * 3 + 1];
    return scale_of(p, b) * (ex2_approx((p.stats[b * 3 + 2] - lse) * LOG2E) - 1.0f);
  }
};

template <int KIND>
struct Pairwise {
  static constexpr int kKind = KIND;
  static constexpr bool kTwoPass = pw::is_max<KIND>::value;  // the forward's lse pass
  static constexpr bool kCatalog = false;
  static constexpr bool kSmooth = false;
  template <int MODE>
  static constexpr int cols() {
    return MODE == DN ? 3 : 0;
  }
  // FWD: the query's [sp] (the -max kinds' lse goes to v[1] after pass 1); DQ: the query's [sp, lse, A]
  template <int MODE>
  __device__ __forceinline__ static void row_vals(const Params& p, long long r, float (&v)[3]) {
    if (MODE != DN) v[0] = p.pos_logit[r];
    if (MODE == DQ) {
      v[1] = p.stats[r * 4 + 2];
      v[2] = p.stats[r * 4 + 3];
    }
  }
  // DN: the query's [sp, lse, A]
  template <int MODE>
  __device__ __forceinline__ static void col_vals(const Params& p, long long c, float (&v)[3]) {
    if (MODE == DN) {
      v[0] = p.pos_logit[c];
      v[1] = p.stats[c * 4 + 2];
      v[2] = p.stats[c * 4 + 3];
    }
  }
  template <int MODE>
  __device__ __forceinline__ static float score(const Params& p, float a, const float (&)[3], const float*) {
    return a * p.inv_temp;
  }
  // c / T dloss/ds of an unmasked element
  template <int MODE>
  __device__ __forceinline__ static float grad(const Params& p, float s, const float (&r)[3], const float* c) {
    const float g = MODE == DN ? pw::bwd_elem<KIND>(s, c[0], c[kColStride], c[2 * kColStride], p.lambda)
                               : pw::bwd_elem<KIND>(s, r[0], r[1], r[2], p.lambda);
    return p.c * p.inv_temp * g;
  }
  __device__ __forceinline__ static float g0(const Params& p, long long b) { return p.c * p.inv_temp * p.stats[b * 4 + 1]; }
};

// Integer values (a label, a row or column index) travel through the float row / column slots bit for bit.  A label
// outside [0, N) becomes -1, which matches no column: its row keeps the soft-max term and loses the one-hot.
struct CatalogCE {
  static constexpr bool kTwoPass = false;
  static constexpr bool kCatalog = true;
  static constexpr bool kSmooth = false;
  __device__ __forceinline__ static float label_of(const Params& p, long long b, long long n_classes) {
    const long long y = id_at(p.labels, b, p.id_is64);
    return __int_as_float(y >= 0 && y < n_classes ? (int)y : -1);
  }
  __device__ __forceinline__ static float bias_of(const Params& p, long long n) { return p.bias ? p.bias[n] : 0.0f; }
  template <int MODE>
  static constexpr int cols() {
    return MODE == DN ? 3 : 2;
  }
  // DQ: the query's [lse, c/T, label]; DN: the catalog row's [b/T, its index]
  template <int MODE>
  __device__ __forceinline__ static void row_vals(const Params& p, long long r, float (&v)[3]) {
    if (MODE == DN) {
      v[0] = bias_of(p, r);
      v[1] = __int_as_float((int)r);
    } else {
      v[0] = p.stats[r * 3 + 1];
      v[1] = (p.scale_is_scalar ? p.row_scale[0] : p.row_scale[r]) * p.inv_temp;
      v[2] = label_of(p, r, p.I);
    }
  }
  // DQ: the catalog row's [b/T, its index]; DN: the query's [lse, c, label]
  template <int MODE>
  __device__ __forceinline__ static void col_vals(const Params& p, long long c, float (&v)[3]) {
    if (MODE == DN) {
      v[0] = p.stats[c * 3 + 1];
      v[1] = p.scale_is_scalar ? p.row_scale[0] : p.row_scale[c];
      v[2] = label_of(p, c, p.M);
    } else {
      v[0] = bias_of(p, c);
      v[1] = __int_as_float((int)c);
    }
  }
  // the forward's logit: (x / T) . e + b / T, the same fp32 add mm_catalog_score does
  template <int MODE>
  __device__ __forceinline__ static float score(const Params&, float a, const float (&r)[3], const float* c) {
    return a + (MODE == DN ? r[0] : c[0]);
  }
  // DQ: c/T (softmax - onehot); DN: c (softmax - onehot)
  template <int MODE>
  __device__ __forceinline__ static float grad(const Params&, float s, const float (&r)[3], const float* c) {
    const float lse = MODE == DN ? c[0] : r[0];
    const float sc = MODE == DN ? c[kColStride] : r[1];
    const bool hit = MODE == DN ? __float_as_int(c[2 * kColStride]) == __float_as_int(r[1])
                                : __float_as_int(r[2]) == __float_as_int(c[kColStride]);
    return sc * (ex2_approx((s - lse) * LOG2E) - (hit ? 1.0f : 0.0f));
  }
  __device__ __forceinline__ static float g0(const Params&, long long) { return 0.0f; }
};

// CatalogCE against the label-smoothed target (1 - eps) onehot + eps / N.  The tile keeps G = c (softmax - (1 - eps)
// onehot); the uniform part -c eps / N is the same for every column, so its products are rank-one and come from the
// column sums in ls_e / ls_x, added where each output row is written: dx -= c / T ls_e, dE -= ls_x, db -= ls_x[extra] / T.
struct SmoothedCatalogCE : CatalogCE {
  static constexpr bool kSmooth = true;
  template <int MODE>
  __device__ __forceinline__ static float grad(const Params& p, float s, const float (&r)[3], const float* c) {
    const float lse = MODE == DN ? c[0] : r[0];
    const float sc = MODE == DN ? c[kColStride] : r[1];
    const bool hit = MODE == DN ? __float_as_int(c[2 * kColStride]) == __float_as_int(r[1])
                                : __float_as_int(r[2]) == __float_as_int(c[kColStride]);
    return sc * (ex2_approx((s - lse) * LOG2E) - (hit ? p.keep : 0.0f));
  }
};

// wgmma with the A operand from registers and an MN-major (transposed) B operand: D[64 x n] += A[64 x 16] . B[16 x n]
__device__ __forceinline__ void wgmma_rs_tb_n64(float (&d)[64], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
__device__ __forceinline__ void wgmma_rs_tb_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, "
      "%68, 1, 1, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <int KP>
__device__ __forceinline__ void wgmma_rs_tb(float (&d)[64], const uint32_t (&a)[4], uint64_t b) {
  if (KP == 64)
    wgmma_rs_tb_n64(d, a, b);
  else
    wgmma_rs_tb_n128(d, a, b);
}
// MN-major SWIZZLE_128B descriptor over the streamed tile as TMA wrote it: 128-B rows of 64 feature columns, one row per
// streamed item (the K dimension of G . X), 8-row groups 1024 B apart (SBO); the next 64 feature columns sit one 16 KB
// tile further (LBO).  A k-step of 16 items advances the start by 16 rows = 2048 B.
__device__ __forceinline__ uint64_t make_desc_sw128_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(TILE_BYTES >> 4) << 16;  // LBO: next 64 columns of the MN (feature) dimension
  d |= (uint64_t)(1024 >> 4) << 32;        // SBO: next 8 rows of the K (item) dimension
  d |= (uint64_t)1 << 62;                  // SWIZZLE_128B
  return d;
}

// Loss: SoftmaxCE or Pairwise<KIND>.  MODE: FWD (pairwise only), DQ (resident rows are queries, streamed rows negatives)
// or DN (resident rows are negatives, streamed rows queries).  KP = padded feature width (64 or 128): the n of the second
// product.
template <class Loss, int MODE, int KP>
__global__ void __launch_bounds__(kThreads, 1)
inbatch_flash_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Params p) {
  constexpr bool TRANS = MODE == DN;
  constexpr int PASSES = MODE == FWD && Loss::kTwoPass ? 2 : 1;
  constexpr int NCOL = Loss::template cols<MODE>();
  constexpr int KB = KP / BLOCK_K;
  constexpr uint32_t A_BYTES = 2u * KB * TILE_BYTES;      // [hi kb0..][lo kb0..]
  constexpr uint32_t STAGE_BYTES = 2u * KB * TILE_BYTES;  // one streamed tile, all k-blocks, hi + lo
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + (size_t)p.stages * STAGE_BYTES);
  uint64_t* full_bar = bars;           // [stages]
  uint64_t* a_full = bars + p.stages;  // [1]
  // per streamed tile, double-buffered: the loss's column values [kColVals][2][128] (0 past the end), the column ids
  float* col_v = reinterpret_cast<float*>(bars + p.stages + 2);
  int* ids_lo = reinterpret_cast<int*>(col_v + kColVals * kColStride);  // [2][128]
  int* ids_hi = ids_lo + 2 * BN;                                        // [2][128]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long m0 = (long long)blockIdx.x * BM;
  // the catalog loss's dq kernel streams only its split's tiles t_base .. t_base + total - 1
  const int t_base = Loss::kCatalog ? (int)blockIdx.y * p.tiles_per_split : 0;
  const int total = Loss::kCatalog ? min(p.n_tiles - t_base, p.tiles_per_split) : PASSES * p.n_tiles;
  // Thread 0 issues every TMA load.  The two warpgroups meet at a named barrier at the start of each tile; by then both
  // have waited for their MMAs of the previous tile, so its stage is free and is refilled right there.  No producer warp:
  // a ninth warp would share a register sub-partition with two consumer warps and cap every thread at 168 registers.
  auto load_tile = [&](int t) {
    const int stage = t % p.stages;
    const int tile = t_base + (PASSES == 1 ? t : t % p.n_tiles);
    const uint32_t fb = smem_u32(full_bar + stage);
    uint8_t* st = smem_b + (size_t)stage * STAGE_BYTES;
    mbar_expect_tx(fb, STAGE_BYTES);
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      tma_load_2d(smem_u32(st + kb * TILE_BYTES), &tmB, fb, kb * BLOCK_K, tile * BN);
      tma_load_2d(smem_u32(st + (KB + kb) * TILE_BYTES), &tmB, fb, KP + kb * BLOCK_K, tile * BN);
    }
  };
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < p.stages; ++s) mbar_init(smem_u32(full_bar + s), 1);
    mbar_init(smem_u32(a_full), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(smem_u32(a_full), A_BYTES);
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      tma_load_2d(smem_u32(smem_a + kb * TILE_BYTES), &tmA, smem_u32(a_full), kb * BLOCK_K, (int)m0);
      tma_load_2d(smem_u32(smem_a + (KB + kb) * TILE_BYTES), &tmA, smem_u32(a_full), KP + kb * BLOCK_K, (int)m0);
    }
    for (int t = 0; t < p.stages && t < total; ++t) load_tile(t);
  }

  // ===================== consumers =====================
  const int wg = warp >> 2;
  const int part = lane & 3;
  const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // tile row of fragment row 0 (row 1 is 8 further)
  const bool do_mask = p.row_ids != nullptr;
  long long row[2], my_id[2] = {0, 0};
  bool rvalid[2];
  float rv[2][3] = {{0.0f, 0.0f, 0.0f}, {0.0f, 0.0f, 0.0f}};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row[h] = m0 + frow + 8 * h;
    rvalid[h] = row[h] < p.M;
    if (rvalid[h]) {
      Loss::template row_vals<MODE>(p, row[h], rv[h]);
      if (do_mask) my_id[h] = id_at(p.row_ids, row[h], p.id_is64);
      if constexpr (Loss::kCatalog && MODE == DQ) {  // one count per row: the quad's lane 0 of the first split
        if (p.oob && part == 0 && blockIdx.y == 0 && __float_as_int(rv[h][2]) < 0) atomicAdd(p.oob, 1);
      }
    }
  }
  // forward: per row, this thread's partials over the columns it sees (the four lanes of a quad share a row)
  pw::RowAcc racc[2];
  float run_m[2] = {-INFINITY, -INFINITY}, run_s[2] = {0.0f, 0.0f};
  float dacc[64];
  float dbacc[2] = {0.0f, 0.0f};  // catalog dn kernel: this thread's part of the row's bias gradient sum_b G
  if (MODE != FWD) {
#pragma unroll
    for (int i = 0; i < 64; ++i) dacc[i] = 0.0f;
  }
  // the catalog dq kernel writes its split's partial dX (gridDim.y > 1) or dX itself
  float* out = p.out;
  if constexpr (Loss::kCatalog) out += (long long)blockIdx.y * p.M * p.D;
  int stage = 0, buf = 0;
  uint32_t phase = 0;
  mbar_wait(smem_u32(a_full), 0);
  const uint32_t a_base = smem_u32(smem_a) + (uint32_t)wg * (TILE_BYTES / 2);
  for (int t = 0; t < total; ++t) {
    const int pass = PASSES == 1 ? 0 : t / p.n_tiles;
    const long long n0 = (long long)(t_base + t - pass * p.n_tiles) * BN;
    float* cv = col_v + buf * BN;
    int* cl = ids_lo + buf * BN;
    int* chh = ids_hi + buf * BN;
    buf ^= 1;
    // per-tile column data -> shared memory (the buffer of tile t-2 is free: its readers passed bar 1 of t-1)
    named_bar(1, kThreads);
    // every warp has finished tile t-1: refill its stage with tile t-1+stages
    if (threadIdx.x == 0 && t > 0 && t - 1 + p.stages < total) load_tile(t - 1 + p.stages);
    for (int i = threadIdx.x; i < BN; i += kThreads) {
      const long long c = n0 + i;
      const bool in = c < p.I;
      if (NCOL > 0) {
        float v[3] = {0.0f, 0.0f, 0.0f};
        if (in) Loss::template col_vals<MODE>(p, c, v);
#pragma unroll
        for (int k = 0; k < NCOL; ++k) cv[k * kColStride + i] = v[k];
      }
      if (do_mask) {
        const long long cid = in ? id_at(p.col_ids, c, p.id_is64) : 0;
        cl[i] = (int)cid;
        chh[i] = (int)(cid >> 32);
      }
    }
    named_bar(1, kThreads);

    // ---- S: 64 x 128 scores of this warpgroup (the forward's 3-pass split-bf16 product) ----
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
    mbar_wait(smem_u32(full_bar + stage), phase);
    const uint32_t b_base = smem_u32(smem_b + (size_t)stage * STAGE_BYTES);
    wgmma_fence_acc(acc);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      const uint32_t a_hi = a_base + kb * TILE_BYTES, a_lo = a_base + (KB + kb) * TILE_BYTES;
      const uint32_t b_hi = b_base + kb * TILE_BYTES, b_lo = b_base + (KB + kb) * TILE_BYTES;
#pragma unroll
      for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss_n128(acc, make_desc_sw128(a_hi + k * 32), make_desc_sw128(b_lo + k * 32));
#pragma unroll
      for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss_n128(acc, make_desc_sw128(a_lo + k * 32), make_desc_sw128(b_hi + k * 32));
#pragma unroll
      for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss_n128(acc, make_desc_sw128(a_hi + k * 32), make_desc_sw128(b_hi + k * 32));
    }
    wgmma_commit();
    wgmma_wait_all();
    wgmma_fence_acc(acc);

    // acc[4 j + 2 h + e]: row h, column 8 j + 2 part + e.  The element code is compiled twice: only a ragged last tile
    // runs the copy with the column bound test, so full tiles carry no per-element bound predicate.
    auto elements = [&](auto ragged_tile) {
      constexpr bool RAGGED = decltype(ragged_tile)::value;
      if constexpr (MODE == FWD) {
        if (PASSES == 2 && pass == 0) {
          // ---- pass 1 of the -max kinds: running max and sum of exp over the row's negatives ----
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float cmax = -INFINITY;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int c = 8 * j + 2 * part + e;
                const int i = 4 * j + 2 * h + e;
                float s = Loss::template score<MODE>(p, acc[i], rv[h], cv + c);
                if (do_mask && cl[c] == (int)my_id[h] && chh[c] == (int)(my_id[h] >> 32)) s = p.masked_score;
                if (RAGGED && n0 + c >= p.I) s = -INFINITY;
                acc[i] = s;
                cmax = fmaxf(cmax, s);
              }
            }
            if (cmax > -INFINITY) {
              const float m_new = fmaxf(run_m[h], cmax);
              float sum = run_s[h] * expf(run_m[h] - m_new);
#pragma unroll
              for (int j = 0; j < 16; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) sum += expf(acc[4 * j + 2 * h + e] - m_new);
              }
              run_m[h] = m_new;
              run_s[h] = sum;
            }
          }
        } else {
          // ---- the per-element losses of this tile into the row sums ----
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int c = 8 * j + 2 * part + e;
                const int i = 4 * j + 2 * h + e;
                const bool valid = rvalid[h] && !(RAGGED && n0 + c >= p.I);
                float s = Loss::template score<MODE>(p, acc[i], rv[h], cv + c);
                if (do_mask && cl[c] == (int)my_id[h] && chh[c] == (int)(my_id[h] >> 32)) s = p.masked_score;
                pw::fwd_elem<Loss::kKind>(valid, s, rv[h][0], rv[h][1], p.lambda, racc[h]);
              }
            }
          }
        }
      } else {
        // ---- G, zero where masked (a constant score) or outside the matrix ----
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * j + 2 * part + e;
              const int i = 4 * j + 2 * h + e;
              bool ok = rvalid[h] && !(RAGGED && n0 + c >= p.I);
              if (do_mask && cl[c] == (int)my_id[h] && chh[c] == (int)(my_id[h] >> 32)) ok = false;
              const float s = Loss::template score<MODE>(p, acc[i], rv[h], cv + c);
              const float g = Loss::template grad<MODE>(p, s, rv[h], cv + c);
              acc[i] = ok ? g : 0.0f;
              if constexpr (Loss::kCatalog && MODE == DN) dbacc[h] += acc[i];
            }
          }
        }
      }
    };
    if (n0 + BN > p.I)
      elements(std::true_type());
    else
      elements(std::false_type());
    if constexpr (MODE == FWD) {
      if (PASSES == 2 && pass == 0 && t == p.n_tiles - 1) {
        // the row's log-sum-exp: merge the quad's four partials (same order in every lane)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, run_m[h], o);
            const float os = __shfl_xor_sync(0xffffffffu, run_s[h], o);
            const float m_new = fmaxf(run_m[h], om);
            const float a = run_m[h] > -INFINITY ? run_s[h] * expf(run_m[h] - m_new) : 0.0f;
            const float b = om > -INFINITY ? os * expf(om - m_new) : 0.0f;
            run_s[h] = (o & lane) ? b + a : a + b;
            run_m[h] = m_new;
          }
          rv[h][1] = run_m[h] + logf(run_s[h]);
        }
      }
    } else {
      // k-step ks of the second product = columns 16 ks .. 16 ks + 15 = fragment words 4 ks .. 4 ks + 3
      uint32_t ghi[32], glo[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) split_pair(acc[2 * i], acc[2 * i + 1], ghi[i], glo[i]);

      // ---- dX += G . X_tile: 3-pass split (G_hi X_lo + G_lo X_hi + G_hi X_hi), X as the MN-major B operand ----
      const uint32_t x_hi = b_base, x_lo = b_base + KB * TILE_BYTES;
      wgmma_fence_acc(dacc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BN / MMA_K; ++ks) {
        const uint32_t f[4] = {ghi[4 * ks], ghi[4 * ks + 1], ghi[4 * ks + 2], ghi[4 * ks + 3]};
        wgmma_rs_tb<KP>(dacc, f, make_desc_sw128_mn(x_lo + ks * 2048));
      }
#pragma unroll
      for (int ks = 0; ks < BN / MMA_K; ++ks) {
        const uint32_t f[4] = {glo[4 * ks], glo[4 * ks + 1], glo[4 * ks + 2], glo[4 * ks + 3]};
        wgmma_rs_tb<KP>(dacc, f, make_desc_sw128_mn(x_hi + ks * 2048));
      }
#pragma unroll
      for (int ks = 0; ks < BN / MMA_K; ++ks) {
        const uint32_t f[4] = {ghi[4 * ks], ghi[4 * ks + 1], ghi[4 * ks + 2], ghi[4 * ks + 3]};
        wgmma_rs_tb<KP>(dacc, f, make_desc_sw128_mn(x_hi + ks * 2048));
      }
      wgmma_commit();
      wgmma_wait_all();
      wgmma_fence_acc(dacc);
      if constexpr (Loss::kCatalog) {
        if ((t + 1) % kFlushTiles == 0 && t + 1 < total) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int j = 0; j < KP / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int c = 8 * j + 2 * part + e;
                if (rvalid[h] && c < p.D) {
                  const long long o = row[h] * p.D + c;
                  out[o] = t + 1 > kFlushTiles ? out[o] + dacc[4 * j + 2 * h + e] : dacc[4 * j + 2 * h + e];
                }
                dacc[4 * j + 2 * h + e] = 0.0f;
              }
            }
          }
        }
      }
    }
    if (++stage == p.stages) {
      stage = 0;
      phase ^= 1;
    }
  }

  if constexpr (MODE == FWD) {
    // ---- the row's statistics: the quad's four partials summed in the same order in every lane ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      pw::RowAcc& a = racc[h];
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        const float ol = __shfl_xor_sync(0xffffffffu, a.loss, o), og = __shfl_xor_sync(0xffffffffu, a.gp, o);
        const float oc = __shfl_xor_sync(0xffffffffu, a.cnt, o), oq = __shfl_xor_sync(0xffffffffu, a.sq, o);
        const bool hi = (o & lane) != 0;
        a.loss = hi ? ol + a.loss : a.loss + ol;
        a.gp = hi ? og + a.gp : a.gp + og;
        a.cnt = hi ? oc + a.cnt : a.cnt + oc;
        a.sq = hi ? oq + a.sq : a.sq + oq;
      }
      if (rvalid[h] && part == 0) {
        const float A = pw::fwd_row<Loss::kKind>(rv[h][0], p.lambda, a);
        float4 v = make_float4(a.loss, a.gp, rv[h][1], A);
        *reinterpret_cast<float4*>(p.stats + row[h] * 4) = v;
      }
    }
  } else {
    if constexpr (Loss::kCatalog && MODE == DN) {
      // ---- the row's bias gradient: the quad's four partials summed in the same order in every lane ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, dbacc[h], o);
          dbacc[h] = (o & lane) ? ov + dbacc[h] : dbacc[h] + ov;
        }
        if constexpr (Loss::kSmooth) dbacc[h] -= p.ls_x[kAuxExtra];
        if (p.db && rvalid[h] && part == 0) p.db[row[h]] = dbacc[h] * p.inv_temp;
      }
    }
    // ---- epilogue: dacc[4 j + 2 h + e] is output row h, feature column 8 j + 2 part + e ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!rvalid[h]) continue;
      const long long r = row[h];
      // dQ: + g0[b] pos[b] (and dpos = g0[b] q[b] in its own buffer); dN with dpos aliasing dneg: + g0[n] q[n]
      const bool add = Loss::kCatalog ? false : TRANS ? p.dpos != nullptr : true;
      const float g0 = add ? Loss::g0(p, r) : 0.0f;
      const float* addend = TRANS ? p.q : p.pos;
#pragma unroll
      for (int j = 0; j < KP / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + 2 * part + e;
          if (c < p.D) {
            const long long o = r * p.D + c;
            float v = dacc[4 * j + 2 * h + e];
            if (add) v = fmaf(g0, addend[o], v);
            if (Loss::kCatalog && total > kFlushTiles) v = out[o] + v;  // after the flushed chunks
            if constexpr (Loss::kSmooth) {  // the uniform target's term, in the first split's partial only
              if (TRANS)
                v -= p.ls_x[c];
              else if (blockIdx.y == 0)
                v = fmaf(-rv[h][1], p.ls_e[c], v);
            }
            out[o] = v;
            if (!TRANS && p.dpos) p.dpos[o] = g0 * p.q[o];
          }
        }
      }
    }
  }
}

// loss[0] += factor sum_b w[b] (stats[b, col] - stats[b, sub]), w[b] = row_scale[b] (or row_scale[0], or 1 when null),
// no subtrahend when sub < 0: one CTA, fixed summation order (double per thread, then a tree)
__global__ void inbatch_loss_kernel(long long B, const float* __restrict__ stats, int stride, int col, int sub,
                                    const float* __restrict__ row_scale, int scale_is_scalar, double factor,
                                    float* __restrict__ loss) {
  __shared__ double part[1024];
  double s = 0.0;
  for (long long b = threadIdx.x; b < B; b += blockDim.x) {
    const double v = (double)stats[b * stride + col];
    const double d = sub >= 0 ? v - (double)stats[b * stride + sub] : v;
    s = row_scale ? fma((double)(scale_is_scalar ? row_scale[0] : row_scale[b]), d, s) : s + d;
  }
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] += (float)(factor * part[0]);
}

// out[i] = sum_s part[s n + i] over the S partial dX of the catalog dq kernel's splits, in split order
__global__ void split_sum_kernel(long long n, int S, const float* __restrict__ part, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float s = part[i];
    for (int k = 1; k < S; ++k) s += part[(long long)k * n + i];
    out[i] = s;
  }
}

// ---- label smoothing: column sums of a split operand, in a fixed order ----
// The rows are cut into chunks (at most kSumChunks, a function of the row count only); warp w of a chunk's CTA adds rows
// w, w + 8, ... of the chunk in row order, in double, and the CTA adds its warps in warp order into the chunk's partial
// (kPartStride doubles: the columns, then the extra sum at kAuxExtra).  colsum_finish_kernel adds the partials in chunk
// order.  The extra sum is sum_r extra[r] (the bias), or sum_r w[r] (the row weights c) when extra is null.
constexpr int kSumWarps = 8, kSumChunks = 1024, kPartStride = 130;

static long long sum_chunks(long long R) {
  const long long c = (R + 255) / 256;
  return c < kSumChunks ? c : kSumChunks;
}

template <int KB>
__global__ void __launch_bounds__(kSumWarps * 32)
colsum_partial_kernel(const __nv_bfloat16* __restrict__ split, long long R, int D, long long per_chunk, const float* __restrict__ w,
                      int w_scalar, const float* __restrict__ extra, double* __restrict__ part) {
  constexpr int KP = 64 * KB;
  __shared__ double sm[kSumWarps][kPartStride];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r0 = (long long)blockIdx.x * per_chunk, r1 = min(R, r0 + per_chunk);
  double acc[2 * KB] = {}, ex = 0.0;
  for (long long r = r0 + warp; r < r1; r += kSumWarps) {
    const __nv_bfloat16* row = split + r * 2 * KP;
    const float wr = w ? w[w_scalar ? 0 : r] : 1.0f;
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      const int c = 64 * k + 2 * lane;
      const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + c));
      const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + KP + c));
      acc[2 * k] += (double)(wr * (hi.x + lo.x));
      acc[2 * k + 1] += (double)(wr * (hi.y + lo.y));
    }
    if (lane == 0) ex += extra ? (double)extra[r] : w ? (double)wr : 0.0;
  }
#pragma unroll
  for (int k = 0; k < KB; ++k) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = 64 * k + 2 * lane + e;
      sm[warp][c] = c < D ? acc[2 * k + e] : 0.0;
    }
  }
  if (lane == 0) sm[warp][kAuxExtra] = ex;
  __syncthreads();
  for (int c = threadIdx.x; c <= kAuxExtra; c += blockDim.x) {
    double s = 0.0;
    if (c < KP || c == kAuxExtra) {
      for (int i = 0; i < kSumWarps; ++i) s += sm[i][c];
    }
    part[blockIdx.x * (long long)kPartStride + c] = s;
  }
}

// out[c] = scale sum_chunk part[chunk][c] in chunk order, c in [0, kAux) (zero past the sums)
__global__ void colsum_finish_kernel(const double* __restrict__ part, int chunks, double scale, float* __restrict__ out) {
  for (int c = threadIdx.x; c < kAux; c += blockDim.x) {
    double s = 0.0;
    if (c <= kAuxExtra) {
      for (int i = 0; i < chunks; ++i) s += part[(long long)i * kPartStride + c];
    }
    out[c] = (float)(scale * s);
  }
}

// out[b] = x_split[b] . aux[0:Kp] + aux[kAuxExtra]: one warp per row, the lanes' products added in a fixed butterfly
template <int KB>
__global__ void __launch_bounds__(256) row_dot_kernel(const __nv_bfloat16* __restrict__ split, long long B, int D,
                                                      const float* __restrict__ aux, float* __restrict__ out) {
  constexpr int KP = 64 * KB;
  const int lane = threadIdx.x & 31;
  const long long b = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const __nv_bfloat16* row = split + b * 2 * KP;
  float s = 0.0f;
#pragma unroll
  for (int k = 0; k < KB; ++k) {
    const int c = 64 * k + 2 * lane;
    const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + c));
    const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + KP + c));
    if (c < D) s = fmaf(hi.x + lo.x, aux[c], s);
    if (c + 1 < D) s = fmaf(hi.y + lo.y, aux[c + 1], s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(0xffffffffu, s, o);
    s = (o & lane) ? v + s : s + v;
  }
  if (lane == 0) out[b] = s + aux[kAuxExtra];
}

// loss[0] += sum_b c[b] (stats[b,1] - keep stats[b,2] - u[b]): the smoothed loss with u[b] = eps mean_j z[b,j]; one CTA,
// the fixed order of inbatch_loss_kernel
__global__ void smoothed_loss_kernel(long long B, const float* __restrict__ stats, float keep, const float* __restrict__ u,
                                     const float* __restrict__ row_scale, int scale_is_scalar, float* __restrict__ loss) {
  __shared__ double part[1024];
  double s = 0.0;
  for (long long b = threadIdx.x; b < B; b += blockDim.x) {
    const double d = (double)stats[b * 3 + 1] - (double)keep * (double)stats[b * 3 + 2] - (double)u[b];
    s = fma((double)(scale_is_scalar ? row_scale[0] : row_scale[b]), d, s);
  }
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] += (float)part[0];
}

// scale * (column sums of split (R, 2*Kp), extra sum) -> out[kAux]: two launches, part holds sum_chunks(R) partials
static int colsum(const char* who, const void* split, long long R, int D, int Kp, const float* w, int w_scalar, const float* extra,
                  double scale, double* part, float* out, cudaStream_t st) {
  const long long chunks = sum_chunks(R), per = (R + chunks - 1) / chunks;
  const __nv_bfloat16* s = (const __nv_bfloat16*)split;
  if (Kp == 64)
    colsum_partial_kernel<1><<<(unsigned)chunks, kSumWarps * 32, 0, st>>>(s, R, D, per, w, w_scalar, extra, part);
  else
    colsum_partial_kernel<2><<<(unsigned)chunks, kSumWarps * 32, 0, st>>>(s, R, D, per, w, w_scalar, extra, part);
  int rc = mm::check_launch(who);
  if (rc) return rc;
  colsum_finish_kernel<<<1, kAux, 0, st>>>(part, (int)chunks, scale, out);
  return mm::check_launch(who);
}

static int row_dot(const char* who, const void* split, long long B, int D, int Kp, const float* aux, float* out, cudaStream_t st) {
  const unsigned blocks = (unsigned)((B + 7) / 8);
  const __nv_bfloat16* s = (const __nv_bfloat16*)split;
  if (Kp == 64)
    row_dot_kernel<1><<<blocks, 256, 0, st>>>(s, B, D, aux, out);
  else
    row_dot_kernel<2><<<blocks, 256, 0, st>>>(s, B, D, aux, out);
  return mm::check_launch(who);
}

// The smoothing workspace after the dq splits' partials (256-B aligned): the E and X column partials, ls_e, ls_x, u (B,)
struct SmoothLayout {
  double *part_e, *part_x;
  float *ls_e, *ls_x, *u;
  int64_t end;
};
static int64_t align256(int64_t n) { return (n + 255) & ~(int64_t)255; }

// The catalog dq kernel's splits per query tile: one query tile per CTA leaves SMs idle while ceil(B / 128) is below the
// SM count (B = 4096 is 32 CTAs), so each query tile's catalog is split over floor(SMs / query tiles) CTAs (one CTA
// fits per SM: one wave), at most one per catalog tile and with no empty split.  The workspace is S B D floats with
// S B <= 128 SMs whatever the catalog size.
static int catalog_splits(long long B, long long N) {
  const long long m_blocks = (B + BM - 1) / BM, n_tiles = (N + BN - 1) / BN;
  long long S = sm_count() / m_blocks;
  if (S > n_tiles) S = n_tiles;
  if (S < 1) S = 1;
  const long long per = (n_tiles + S - 1) / S;
  return (int)((n_tiles + per - 1) / per);
}

static int64_t split_bytes(int64_t B, int64_t N, int D) {
  const int S = catalog_splits(B, N);
  return S > 1 ? (int64_t)S * B * D * (int64_t)sizeof(float) : 0;
}

static SmoothLayout smooth_layout(int64_t B, int64_t N, int D, void* ws) {
  uint8_t* base = (uint8_t*)ws;
  SmoothLayout l{};
  int64_t o = align256(split_bytes(B, N, D));
  l.part_e = (double*)(base + o);
  o += align256(sum_chunks(N) * kPartStride * (int64_t)sizeof(double));
  l.part_x = (double*)(base + o);
  o += align256(sum_chunks(B) * kPartStride * (int64_t)sizeof(double));
  l.ls_e = (float*)(base + o);
  l.ls_x = l.ls_e + kAux;
  o += align256(2 * kAux * (int64_t)sizeof(float));
  l.u = (float*)(base + o);
  l.end = o + align256(B * (int64_t)sizeof(float));
  return l;
}

typedef void (*Kernel)(const CUtensorMap, const CUtensorMap, const Params);

// one CTA per 128 of the p.M resident rows (times `splits` for the catalog dq kernel), streaming the p.I others through
// as many stages as fit (at most 4)
static int launch(const char* who, Kernel kern, int Kp, const CUtensorMap& tmA, const CUtensorMap& tmB, Params p,
                  cudaStream_t st, int splits = 1) {
  const size_t tile_bytes = 2ull * (Kp / BLOCK_K) * TILE_BYTES;  // the resident tile and one stage are the same size
  const size_t extra = (kColVals + 2) * 2 * BN * sizeof(float);  // per-tile column data: the values and two id words
  const size_t fixed = 1024 + tile_bytes + 8 * sizeof(uint64_t) + extra;
  int stages = (int)((227 * 1024 - fixed) / tile_bytes);
  if (stages > 4) stages = 4;
  MM_REQUIRE(stages >= 2, MM_ERR_UNSUPPORTED, "%s: tiles do not fit two pipeline stages", who);
  p.stages = stages;
  p.n_tiles = (int)((p.I + BN - 1) / BN);
  p.tiles_per_split = (p.n_tiles + splits - 1) / splits;
  const size_t smem = 1024 + tile_bytes + stages * tile_bytes + (stages + 2) * sizeof(uint64_t) + extra;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    mm::set_error("%s: cudaFuncSetAttribute failed: %s", who, cudaGetErrorString(e));
    return (int)e;
  }
  kern<<<dim3((unsigned)((p.M + BM - 1) / BM), (unsigned)splits), kThreads, smem, st>>>(tmA, tmB, p);
  return mm::check_launch(who);
}

// The backward from the query-side parameters p (resident queries, streamed negatives): the dq kernel, which also
// writes dpos unless it is dneg's buffer, then the dn kernel with the roles swapped, which adds g0[n] q[n] when dpos
// aliases dneg (the negatives are the positives).
static int launch_bwd(const char* who, Kernel dq_kern, Kernel dn_kern, int Kp, const CUtensorMap& tmQ, const CUtensorMap& tmN,
                      const Params& p, float* dq, float* dpos, float* dneg, cudaStream_t st) {
  Params pq = p;
  pq.out = dq;
  pq.dpos = dpos == dneg ? nullptr : dpos;
  int rc = launch(who, dq_kern, Kp, tmQ, tmN, pq, st);
  if (rc) return rc;
  Params pn = p;
  pn.M = p.I;
  pn.I = p.M;
  pn.row_ids = p.col_ids;
  pn.col_ids = p.row_ids;
  pn.out = dneg;
  pn.dpos = dpos == dneg ? dpos : nullptr;
  return launch(who, dn_kern, Kp, tmN, tmQ, pn, st);
}

// The argument rules every entry point shares (dq / dpos / dneg: the backward's gradients, which its caller has checked
// for null; null in the forward), then, for B > 0, the tensor maps of the split operands and the query-side parameters.
// The entry points check their own rules first: no rule may lose to a driver error.
static int prepare(const char* who, const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                   const void* neg_ids, int id_dtype, int downscore, float temperature, const float* dq, const float* dpos,
                   const float* dneg, int* Kp, CUtensorMap* tmQ, CUtensorMap* tmN, Params* p) {
  MM_REQUIRE(q_split && neg_split, MM_ERR_ARG, "%s: null pointer (the split operands are required)", who);
  MM_REQUIRE(B >= 0 && N > 0 && D > 0, MM_ERR_ARG, "%s: bad size (B >= 0, N > 0, D > 0)", who);
  MM_REQUIRE(temperature > 0.0f, MM_ERR_ARG, "%s: temperature must be positive", who);
  MM_REQUIRE(!downscore || (pos_ids && neg_ids), MM_ERR_ARG, "%s: down-scoring needs positive and negative ids", who);
  MM_REQUIRE(id_dtype == MM_I32 || id_dtype == MM_I64, MM_ERR_ARG, "%s: bad id dtype", who);
  if (dq) {
    MM_REQUIRE(dpos != dneg || N == B, MM_ERR_ARG, "%s: dpos may alias dneg only when the negatives are the positives (N == B)",
               who);
    MM_REQUIRE(dq != dpos && dq != dneg, MM_ERR_ARG, "%s: dq must not alias dpos / dneg", who);
  }
  *Kp = mm_tc_padded_k(D);
  MM_REQUIRE(*Kp <= 128, MM_ERR_UNSUPPORTED, "%s: D up to 128 (the resident tile is kept in shared memory)", who);
  MM_REQUIRE(B < (1ll << 31) && N < (1ll << 31), MM_ERR_UNSUPPORTED, "%s: sizes exceed 32-bit TMA coordinates", who);
  MM_REQUIRE(((uintptr_t)q_split % 16) == 0 && ((uintptr_t)neg_split % 16) == 0, MM_ERR_ALIGN,
             "%s: split operands must be 16-B aligned", who);
  if (B == 0) return MM_OK;
  int rc = make_map(tmQ, q_split, (uint64_t)B, (uint64_t)2 * *Kp, BM);
  if (rc) return rc;
  rc = make_map(tmN, neg_split, (uint64_t)N, (uint64_t)2 * *Kp, BN);
  if (rc) return rc;
  p->M = B;
  p->I = N;
  p->D = D;
  p->row_ids = downscore ? pos_ids : nullptr;
  p->col_ids = downscore ? neg_ids : nullptr;
  p->id_is64 = id_dtype == MM_I64;
  p->inv_temp = 1.0f / temperature;
  return MM_OK;
}

// the rules of the two pairwise entry points, and their parameters
static int prepare_pairwise(const char* who, int kind, float reg_lambda, float false_neg_score, float temperature, int64_t B,
                            int64_t N, const float* pos_logit, const float* stats, Params* p) {
  MM_REQUIRE(pos_logit && stats, MM_ERR_ARG, "%s: null pointer (pos_logit and stats are required)", who);
  MM_REQUIRE(kind >= 0 && kind < pw::N_KINDS, MM_ERR_ARG, "%s: unknown loss kind %d", who, kind);
  MM_REQUIRE(reg_lambda == reg_lambda && reg_lambda < INFINITY && reg_lambda > -INFINITY, MM_ERR_ARG, "%s: reg_lambda must be finite",
             who);
  MM_REQUIRE(((uintptr_t)stats % 16) == 0, MM_ERR_ALIGN, "%s: stats must be 16-B aligned (float4 rows)", who);
  MM_REQUIRE(((uintptr_t)pos_logit % 4) == 0, MM_ERR_ALIGN, "%s: fp32 buffers must be 4-B aligned", who);
  p->masked_score = false_neg_score * (1.0f / temperature);  // the forward's order: rescore, then divide by T
  p->lambda = reg_lambda;
  p->c = (float)(1.0 / ((double)B * (double)N));
  p->pos_logit = pos_logit;
  p->stats = const_cast<float*>(stats);
  return MM_OK;
}

template <int MODE, int KP>
static Kernel pick_kind(int kind) {
  using namespace mm::pw;
  switch (kind) {
    case BPR: return inbatch_flash_kernel<Pairwise<BPR>, MODE, KP>;
    case BPR_MAX: return inbatch_flash_kernel<Pairwise<BPR_MAX>, MODE, KP>;
    case TOP1: return inbatch_flash_kernel<Pairwise<TOP1>, MODE, KP>;
    case TOP1_V2: return inbatch_flash_kernel<Pairwise<TOP1_V2>, MODE, KP>;
    case TOP1_MAX: return inbatch_flash_kernel<Pairwise<TOP1_MAX>, MODE, KP>;
    case LOGISTIC: return inbatch_flash_kernel<Pairwise<LOGISTIC>, MODE, KP>;
    default: return inbatch_flash_kernel<Pairwise<HINGE>, MODE, KP>;
  }
}
template <int MODE>
static Kernel pick_pairwise(int Kp, int kind) {
  return Kp == 64 ? pick_kind<MODE, 64>(kind) : pick_kind<MODE, 128>(kind);
}
template <int MODE>
static Kernel pick_ce(int Kp) {
  return Kp == 64 ? inbatch_flash_kernel<SoftmaxCE, MODE, 64> : inbatch_flash_kernel<SoftmaxCE, MODE, 128>;
}
template <class Loss, int MODE>
static Kernel pick_catalog(int Kp) {
  return Kp == 64 ? inbatch_flash_kernel<Loss, MODE, 64> : inbatch_flash_kernel<Loss, MODE, 128>;
}

// mm_catalog_softmax_ce_backward (eps == 0: the CatalogCE kernels) and its label-smoothed form (eps > 0: the column sums,
// then the SmoothedCatalogCE kernels and the smoothed loss)
static int catalog_backward(const char* who, const void* x_split, const void* e_split, int64_t B, int64_t N, int D,
                            const float* bias, const void* labels, int label_dtype, float temperature, float eps,
                            const float* stats, const float* row_scale, int row_scale_is_scalar, float* dx, float* de, float* db,
                            float* loss, int* oob_count, void* workspace, int64_t workspace_bytes, void* stream) {
  MM_REQUIRE(labels && stats && row_scale && dx && de, MM_ERR_ARG,
             "%s: null pointer (labels, stats, row_scale, dx and de are required)", who);
  MM_REQUIRE(((uintptr_t)stats | (uintptr_t)row_scale | (uintptr_t)dx | (uintptr_t)de | (uintptr_t)(bias ? bias : stats) |
              (uintptr_t)(db ? db : stats) | (uintptr_t)(loss ? loss : stats)) % 4 == 0,
             MM_ERR_ALIGN, "%s: fp32 buffers must be 4-B aligned", who);
  MM_REQUIRE(((uintptr_t)workspace % 16) == 0 && ((uintptr_t)oob_count % 4) == 0, MM_ERR_ALIGN,
             "%s: workspace must be 16-B and oob_count 4-B aligned", who);
  int Kp = 0;
  CUtensorMap tmX, tmE;
  Params p{};
  int rc = prepare(who, x_split, e_split, B, N, D, nullptr, nullptr, label_dtype, 0, temperature, dx, nullptr, de, &Kp, &tmX, &tmE,
                   &p);
  if (rc) return rc;
  const int64_t need = B <= 0 ? 0 : eps > 0.0f ? smooth_layout(B, N, D, nullptr).end : split_bytes(B, N, D);
  MM_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), MM_ERR_ARG, "%s: workspace too small (%lld < %lld)", who,
             (long long)workspace_bytes, (long long)need);
  if (B == 0) return MM_OK;
  p.labels = labels;
  p.bias = bias;
  p.stats = const_cast<float*>(stats);
  p.row_scale = row_scale;
  p.scale_is_scalar = row_scale_is_scalar != 0;
  cudaStream_t st = (cudaStream_t)stream;
  const bool smooth = eps > 0.0f;
  SmoothLayout sl{};
  if (smooth) {
    // (eps / N) sum_j e_j and sum_j b_j / T; (eps / N) sum_b c_b x_b / T and sum_b c_b; u[b] = eps mean_j z[b, j]
    sl = smooth_layout(B, N, D, workspace);
    const double en = (double)eps / (double)N;
    rc = colsum(who, e_split, N, D, Kp, nullptr, 0, bias, en, sl.part_e, sl.ls_e, st);
    if (rc == MM_OK) rc = colsum(who, x_split, B, D, Kp, row_scale, p.scale_is_scalar, nullptr, en, sl.part_x, sl.ls_x, st);
    if (rc == MM_OK && loss) rc = row_dot(who, x_split, B, D, Kp, sl.ls_e, sl.u, st);
    if (rc) return rc;
    p.keep = 1.0f - eps;
    p.ls_e = sl.ls_e;
    p.ls_x = sl.ls_x;
  }
  Params pq = p;
  pq.oob = oob_count;
  // dX: one CTA per (query tile, catalog split); the splits' partials are summed in split order
  const int S = catalog_splits(B, N);
  pq.out = S > 1 ? (float*)workspace : dx;
  rc = launch(who, smooth ? pick_catalog<SmoothedCatalogCE, DQ>(Kp) : pick_catalog<CatalogCE, DQ>(Kp), Kp, tmX, tmE, pq, st, S);
  if (rc) return rc;
  if (S > 1) {
    const long long n = B * (long long)D;
    long long blocks = (n + 255) / 256;
    const long long cap = (long long)mm::sm_count() * 8;
    split_sum_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, st>>>(n, S, (const float*)workspace, dx);
    rc = mm::check_launch(who);
    if (rc) return rc;
  }
  // dE and db: one CTA per 128 catalog rows streaming the queries
  Params pn = p;
  pn.M = N;
  pn.I = B;
  pn.out = de;
  pn.db = db;
  rc = launch(who, smooth ? pick_catalog<SmoothedCatalogCE, DN>(Kp) : pick_catalog<CatalogCE, DN>(Kp), Kp, tmE, tmX, pn, st);
  if (rc == MM_OK && loss) {
    if (smooth)
      smoothed_loss_kernel<<<1, 1024, 0, st>>>(B, stats, p.keep, sl.u, row_scale, row_scale_is_scalar != 0, loss);
    else
      inbatch_loss_kernel<<<1, 1024, 0, st>>>(B, stats, 3, 1, 2, row_scale, row_scale_is_scalar != 0, 1.0, loss);
    rc = mm::check_launch(who);
  }
  return rc;
}

}  // namespace flash
}  // namespace mm

extern "C" {

int mm_inbatch_softmax_ce_backward(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                                   const void* neg_ids, int id_dtype, int downscore, float false_neg_score, const float* neg_prob,
                                   float temperature, const float* stats, const float* q, const float* pos, const float* row_scale,
                                   int row_scale_is_scalar, float* dq, float* dpos, float* dneg, float* loss, void* stream) {
  const char* who = "mm_inbatch_softmax_ce_backward";
  using namespace mm::flash;
  MM_REQUIRE(stats && q && pos && row_scale && dq && dpos && dneg, MM_ERR_ARG,
             "%s: null pointer (stats, q, pos, row_scale and the three gradients are required)", who);
  MM_REQUIRE(((uintptr_t)stats | (uintptr_t)q | (uintptr_t)pos | (uintptr_t)row_scale | (uintptr_t)dq | (uintptr_t)dpos |
              (uintptr_t)dneg | (uintptr_t)(loss ? loss : stats)) % 4 == 0,
             MM_ERR_ALIGN, "%s: fp32 buffers must be 4-B aligned", who);
  (void)false_neg_score;  // a masked logit is the constant false_neg_score / T: its gradient is zero whatever the score
  int Kp = 0;
  CUtensorMap tmQ, tmN;
  Params p{};
  int rc = prepare(who, q_split, neg_split, B, N, D, pos_ids, neg_ids, id_dtype, downscore, temperature, dq, dpos, dneg, &Kp, &tmQ,
                   &tmN, &p);
  if (rc || B == 0) return rc;
  p.neg_prob = neg_prob;
  p.stats = const_cast<float*>(stats);
  p.row_scale = row_scale;
  p.scale_is_scalar = row_scale_is_scalar != 0;
  p.q = q;
  p.pos = pos;
  cudaStream_t st = (cudaStream_t)stream;
  rc = launch_bwd(who, pick_ce<DQ>(Kp), pick_ce<DN>(Kp), Kp, tmQ, tmN, p, dq, dpos, dneg, st);
  if (rc == MM_OK && loss) {
    inbatch_loss_kernel<<<1, 1024, 0, st>>>(B, stats, 3, 1, 2, row_scale, row_scale_is_scalar != 0, 1.0, loss);
    rc = mm::check_launch(who);
  }
  return rc;
}

int mm_inbatch_pairwise_fwd(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                            const void* neg_ids, int id_dtype, int downscore, float false_neg_score, float temperature, int kind,
                            float reg_lambda, const float* pos_logit, float* stats, float* loss, void* stream) {
  const char* who = "mm_inbatch_pairwise_fwd";
  using namespace mm::flash;
  MM_REQUIRE(((uintptr_t)loss % 4) == 0, MM_ERR_ALIGN, "%s: loss must be 4-B aligned", who);
  int Kp = 0;
  CUtensorMap tmQ, tmN;
  Params p{};
  int rc = prepare_pairwise(who, kind, reg_lambda, false_neg_score, temperature, B, N, pos_logit, stats, &p);
  if (rc == MM_OK)
    rc = prepare(who, q_split, neg_split, B, N, D, pos_ids, neg_ids, id_dtype, downscore, temperature, nullptr, nullptr, nullptr,
                 &Kp, &tmQ, &tmN, &p);
  if (rc || B == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = launch(who, pick_pairwise<FWD>(Kp, kind), Kp, tmQ, tmN, p, st);
  if (rc == MM_OK && loss) {
    inbatch_loss_kernel<<<1, 1024, 0, st>>>(B, stats, 4, 0, -1, nullptr, 0, 1.0 / ((double)B * (double)N), loss);
    rc = mm::check_launch(who);
  }
  return rc;
}

int mm_inbatch_pairwise_bwd(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                            const void* neg_ids, int id_dtype, int downscore, float false_neg_score, float temperature, int kind,
                            float reg_lambda, const float* pos_logit, const float* stats, const float* q, const float* pos,
                            float* dq, float* dpos, float* dneg, void* stream) {
  const char* who = "mm_inbatch_pairwise_bwd";
  using namespace mm::flash;
  MM_REQUIRE(q && pos && dq && dpos && dneg, MM_ERR_ARG, "%s: null pointer (q, pos and the three gradients are required)", who);
  MM_REQUIRE(((uintptr_t)q | (uintptr_t)pos | (uintptr_t)dq | (uintptr_t)dpos | (uintptr_t)dneg) % 4 == 0, MM_ERR_ALIGN,
             "%s: fp32 buffers must be 4-B aligned", who);
  int Kp = 0;
  CUtensorMap tmQ, tmN;
  Params p{};
  int rc = prepare_pairwise(who, kind, reg_lambda, false_neg_score, temperature, B, N, pos_logit, stats, &p);
  if (rc == MM_OK)
    rc = prepare(who, q_split, neg_split, B, N, D, pos_ids, neg_ids, id_dtype, downscore, temperature, dq, dpos, dneg, &Kp, &tmQ,
                 &tmN, &p);
  if (rc || B == 0) return rc;
  p.q = q;
  p.pos = pos;
  return launch_bwd(who, pick_pairwise<DQ>(Kp, kind), pick_pairwise<DN>(Kp, kind), Kp, tmQ, tmN, p, dq, dpos, dneg,
                    (cudaStream_t)stream);
}

int64_t mm_catalog_softmax_ce_workspace_bytes(int64_t B, int64_t N, int D) {
  if (B <= 0 || N <= 0 || D <= 0) return 0;
  return mm::flash::split_bytes(B, N, D);
}

int mm_catalog_softmax_ce_backward(const void* x_split, const void* e_split, int64_t B, int64_t N, int D, const float* bias,
                                   const void* labels, int label_dtype, float temperature, const float* stats,
                                   const float* row_scale, int row_scale_is_scalar, float* dx, float* de, float* db, float* loss,
                                   int* oob_count, void* workspace, int64_t workspace_bytes, void* stream) {
  return mm::flash::catalog_backward("mm_catalog_softmax_ce_backward", x_split, e_split, B, N, D, bias, labels, label_dtype,
                                     temperature, 0.0f, stats, row_scale, row_scale_is_scalar, dx, de, db, loss, oob_count,
                                     workspace, workspace_bytes, stream);
}

int64_t mm_catalog_smoothed_ce_workspace_bytes(int64_t B, int64_t N, int D) {
  if (B <= 0 || N <= 0 || D <= 0) return 0;
  return mm::flash::smooth_layout(B, N, D, nullptr).end;
}

int mm_catalog_smoothed_ce_backward(const void* x_split, const void* e_split, int64_t B, int64_t N, int D, const float* bias,
                                    const void* labels, int label_dtype, float temperature, float label_smoothing,
                                    const float* stats, const float* row_scale, int row_scale_is_scalar, float* dx, float* de,
                                    float* db, float* loss, int* oob_count, void* workspace, int64_t workspace_bytes,
                                    void* stream) {
  const char* who = "mm_catalog_smoothed_ce_backward";
  MM_REQUIRE(label_smoothing >= 0.0f && label_smoothing < 1.0f, MM_ERR_ARG, "%s: label_smoothing must be in [0, 1)", who);
  return mm::flash::catalog_backward(who, x_split, e_split, B, N, D, bias, labels, label_dtype, temperature, label_smoothing,
                                     stats, row_scale, row_scale_is_scalar, dx, de, db, loss, oob_count, workspace,
                                     workspace_bytes, stream);
}

int64_t mm_catalog_mean_logit_workspace_bytes(int64_t N) {
  using namespace mm::flash;
  if (N <= 0) return 0;
  return align256(sum_chunks(N) * kPartStride * (int64_t)sizeof(double)) + kAux * (int64_t)sizeof(float);
}

int mm_catalog_mean_logit(const void* x_split, const void* e_split, int64_t B, int64_t N, int D, const float* bias, float* out,
                          void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "mm_catalog_mean_logit";
  using namespace mm::flash;
  MM_REQUIRE(x_split && e_split && out, MM_ERR_ARG, "%s: null pointer (x_split, e_split and out are required)", who);
  MM_REQUIRE(B >= 0 && N > 0 && D > 0, MM_ERR_ARG, "%s: bad size (B >= 0, N > 0, D > 0)", who);
  const int Kp = mm_tc_padded_k(D);
  MM_REQUIRE(Kp <= 128, MM_ERR_UNSUPPORTED, "%s: D up to 128", who);
  MM_REQUIRE(((uintptr_t)x_split % 16) == 0 && ((uintptr_t)e_split % 16) == 0 && ((uintptr_t)workspace % 16) == 0 &&
                 ((uintptr_t)out | (uintptr_t)(bias ? bias : out)) % 4 == 0,
             MM_ERR_ALIGN, "%s: split operands and workspace must be 16-B, fp32 buffers 4-B aligned", who);
  const int64_t need = mm_catalog_mean_logit_workspace_bytes(N);
  MM_REQUIRE(workspace_bytes >= need && workspace, MM_ERR_ARG, "%s: workspace too small (%lld < %lld)", who,
             (long long)workspace_bytes, (long long)need);
  if (B == 0) return MM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  // [E's chunk partials][the (1 / N) column sums and bias sum]
  double* part = (double*)workspace;
  float* aux = (float*)((uint8_t*)workspace + align256(sum_chunks(N) * kPartStride * (int64_t)sizeof(double)));
  int rc = colsum(who, e_split, N, D, Kp, nullptr, 0, bias, 1.0 / (double)N, part, aux, st);
  return rc ? rc : row_dot(who, x_split, B, D, Kp, aux, out, st);
}

}  // extern "C"
