// Backward of the in-batch soft-max cross-entropy (mm_inbatch_softmax_ce) without materialising the (B, 1+N) logits:
// a flash-attention-style pass that recomputes every 128x128 logits tile from the split-bf16 operands the forward read,
// turns it into the gradient tile G = c (softmax - onehot) / T with the forward's log-sum-exp, and multiplies G straight
// out of registers into the operand tile still resident in shared memory.
//
//   inbatch_ce_dq_kernel  one CTA per 128 queries (resident), streams the negatives:  S = Q N^T, dQ += G N
//   inbatch_ce_dn_kernel  one CTA per 128 negatives (resident), streams the queries:  S^T = N Q^T, dN += G^T Q
//   inbatch_ce_loss_kernel  loss += sum_b c[b] (lse[b] - s[b,0]) in a fixed order (one CTA)
//
// Both GEMM kernels are one template: two warpgroups (64 resident rows each) over a TMA ring of streamed tiles, the
// forward catalog kernel's structure (catalog_tc.cu) without its producer warp.  The logits use the forward's 3-pass split-bf16 products, logQ, id mask and
// temperature, so exp(s - lse) is consistent with its statistics.  The second product takes G as the register A operand
// (split hi / lo, 3 passes) and the streamed tile as an MN-major B operand (wgmma's transpose bit for 16-bit types), so
// no transposed copy of either operand exists.  Every output row is owned by one CTA: no atomics, bit-reproducible.
#include <cstring>

#include "tc_common.cuh"

namespace mm {
namespace ibw {

using namespace mm::tc;

constexpr int BM = 128, BN = 128, BLOCK_K = 64, MMA_K = 16;
constexpr int kThreads = 256;  // two warpgroups of 64 resident rows each; thread 0 also issues the TMA loads
constexpr uint32_t TILE_BYTES = 128 * BLOCK_K * 2;   // one 128-row x 64-col bf16 tile = 16 KB
constexpr float LOG2E = 1.4426950408889634f;

struct Params {
  long long M, I;  // resident rows, streamed rows
  int D, stages, n_tiles;
  const void* row_ids;  // ids of the resident rows / streamed rows (null: no down-scoring)
  const void* col_ids;
  int id_is64;
  float inv_temp;
  const float* neg_prob;   // (N,) sampling probabilities (logQ) or null
  const float* stats;      // (B, 3) [max, lse, positive logit]
  const float* row_scale;  // (B,) or one float
  int scale_is_scalar;
  const float* q;    // (B, D) fp32
  const float* pos;  // (B, D) fp32
  float* out;        // dq (B, D) or dneg (N, D)
  float* dpos;       // dq kernel: dpos when it is its own buffer; dn kernel: non-null = dpos aliases dneg (add g0 q)
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ long long id_at(const void* p, long long i, int is64) {
  return is64 ? reinterpret_cast<const long long*>(p)[i] : (long long)reinterpret_cast<const int*>(p)[i];
}
__device__ __forceinline__ float logq_bias(const float* prob, long long n) {  // the forward's -log(p + 1e-16)
  return prob ? -logf(prob[n] + 1e-16f) : 0.0f;
}
__device__ __forceinline__ float scale_of(const Params& p, long long b) {  // c[b] / T
  return (p.scale_is_scalar ? p.row_scale[0] : p.row_scale[b]) * p.inv_temp;
}
// g[b, 0] = c[b] (p[b, 0] - 1) / T
__device__ __forceinline__ float pos_grad(const Params& p, long long b) {
  const float lse = p.stats[b * 3 + 1];
  return scale_of(p, b) * (ex2_approx((p.stats[b * 3 + 2] - lse) * LOG2E) - 1.0f);
}

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

// TRANS = false: the dQ kernel (resident rows are queries, streamed rows negatives); true: the dN kernel (resident rows
// are negatives, streamed rows queries).  KP = padded feature width (64 or 128): the n of the second product.
template <bool TRANS, int KP>
__device__ __forceinline__ void ce_bwd_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const Params& p) {
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
  // per streamed tile, double-buffered: dQ: logQ bias of the negative; dN: lse and c/T of the query (0 past the end)
  float* col_v = reinterpret_cast<float*>(bars + p.stages + 2);  // [2][128]
  float* col_s = col_v + 2 * BN;                                  // [2][128]
  int* ids_lo = reinterpret_cast<int*>(col_s + 2 * BN);           // [2][128]
  int* ids_hi = ids_lo + 2 * BN;                                  // [2][128]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long m0 = (long long)blockIdx.x * BM;
  // Thread 0 issues every TMA load.  The two warpgroups meet at a named barrier at the start of each tile; by then both
  // have waited for their MMAs of the previous tile, so its stage is free and is refilled right there.  No producer warp:
  // a ninth warp would share a register sub-partition with two consumer warps and cap every thread at 168 registers.
  auto load_tile = [&](int t) {
    const int stage = t % p.stages;
    const uint32_t fb = smem_u32(full_bar + stage);
    uint8_t* st = smem_b + (size_t)stage * STAGE_BYTES;
    mbar_expect_tx(fb, STAGE_BYTES);
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      tma_load_2d(smem_u32(st + kb * TILE_BYTES), &tmB, fb, kb * BLOCK_K, t * BN);
      tma_load_2d(smem_u32(st + (KB + kb) * TILE_BYTES), &tmB, fb, KP + kb * BLOCK_K, t * BN);
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
    for (int t = 0; t < p.stages && t < p.n_tiles; ++t) load_tile(t);
  }

  // ===================== consumers =====================
  const int wg = warp >> 2;
  const int part = lane & 3;
  const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // tile row of fragment row 0 (row 1 is 8 further)
  const bool do_mask = p.row_ids != nullptr;
  long long row[2], my_id[2] = {0, 0};
  bool rvalid[2];
  float r_bias[2] = {0.0f, 0.0f}, r_lse[2] = {0.0f, 0.0f}, r_scale[2] = {0.0f, 0.0f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row[h] = m0 + frow + 8 * h;
    rvalid[h] = row[h] < p.M;
    if (rvalid[h]) {
      if (TRANS) {
        r_bias[h] = logq_bias(p.neg_prob, row[h]);
      } else {
        r_lse[h] = p.stats[row[h] * 3 + 1];
        r_scale[h] = scale_of(p, row[h]);
      }
      if (do_mask) my_id[h] = id_at(p.row_ids, row[h], p.id_is64);
    }
  }
  float dacc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dacc[i] = 0.0f;
  int stage = 0, buf = 0;
  uint32_t phase = 0;
  mbar_wait(smem_u32(a_full), 0);
  const uint32_t a_base = smem_u32(smem_a) + (uint32_t)wg * (TILE_BYTES / 2);
  for (int t = 0; t < p.n_tiles; ++t) {
    const long long n0 = (long long)t * BN;
    float* cv = col_v + buf * BN;
    float* cs = col_s + buf * BN;
    int* cl = ids_lo + buf * BN;
    int* chh = ids_hi + buf * BN;
    buf ^= 1;
    // per-tile column data -> shared memory (the buffer of tile t-2 is free: its readers passed bar 1 of t-1)
    named_bar(1, kThreads);
    // every warp has finished tile t-1: refill its stage with tile t-1+stages
    if (threadIdx.x == 0 && t > 0 && t - 1 + p.stages < p.n_tiles) load_tile(t - 1 + p.stages);
    for (int i = threadIdx.x; i < BN; i += kThreads) {
      const long long c = n0 + i;
      const bool in = c < p.I;
      if (TRANS) {
        cv[i] = in ? p.stats[c * 3 + 1] : 0.0f;
        cs[i] = in ? scale_of(p, c) : 0.0f;
      } else {
        cv[i] = in ? logq_bias(p.neg_prob, c) : 0.0f;
      }
      if (do_mask) {
        const long long cid = in ? id_at(p.col_ids, c, p.id_is64) : 0;
        cl[i] = (int)cid;
        chh[i] = (int)(cid >> 32);
      }
    }
    named_bar(1, kThreads);

    // ---- S: 64 x 128 logits of this warpgroup (the forward's 3-pass split-bf16 product) ----
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

    // ---- G = c/T softmax, zero where masked or outside the matrix; acc[4 j + 2 h + e]: row h, column 8 j + 2 part + e ----
    const bool ragged = n0 + BN > p.I;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + 2 * part + e;
          const int i = 4 * j + 2 * h + e;
          bool ok = rvalid[h] && !(ragged && n0 + c >= p.I);
          if (do_mask && cl[c] == (int)my_id[h] && chh[c] == (int)(my_id[h] >> 32)) ok = false;
          const float s = (acc[i] + (TRANS ? r_bias[h] : cv[c])) * p.inv_temp;
          const float lse = TRANS ? cv[c] : r_lse[h];
          const float sc = TRANS ? cs[c] : r_scale[h];
          const float g = sc * ex2_approx((s - lse) * LOG2E);
          acc[i] = ok ? g : 0.0f;
        }
      }
    }
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
    if (++stage == p.stages) {
      stage = 0;
      phase ^= 1;
    }
  }

  // ---- epilogue: dacc[4 j + 2 h + e] is output row h, feature column 8 j + 2 part + e ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!rvalid[h]) continue;
    const long long r = row[h];
    // dQ: + g[b,0] pos[b] (and dpos = g[b,0] q[b] in its own buffer); dN with dpos aliasing dneg: + g[n,0] q[n]
    const bool add = TRANS ? p.dpos != nullptr : true;
    const float g0 = add ? pos_grad(p, r) : 0.0f;
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
          p.out[o] = v;
          if (!TRANS && p.dpos) p.dpos[o] = g0 * p.q[o];
        }
      }
    }
  }
}

template <int KP>
__global__ void __launch_bounds__(kThreads, 1)
inbatch_ce_dq_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Params p) {
  ce_bwd_body<false, KP>(tmA, tmB, p);
}
template <int KP>
__global__ void __launch_bounds__(kThreads, 1)
inbatch_ce_dn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Params p) {
  ce_bwd_body<true, KP>(tmA, tmB, p);
}

// loss[0] += sum_b c[b] (lse[b] - s[b,0]): one CTA, fixed summation order (double per thread, then a tree)
__global__ void inbatch_ce_loss_kernel(long long B, const float* __restrict__ stats, const float* __restrict__ row_scale,
                                       int scale_is_scalar, float* __restrict__ loss) {
  __shared__ double part[1024];
  double s = 0.0;
  for (long long b = threadIdx.x; b < B; b += blockDim.x) {
    const float c = scale_is_scalar ? row_scale[0] : row_scale[b];
    s += (double)c * ((double)stats[b * 3 + 1] - (double)stats[b * 3 + 2]);
  }
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] += (float)part[0];
}

typedef void (*BwdKernel)(const CUtensorMap, const CUtensorMap, const Params);

static int launch_bwd(const char* who, BwdKernel kern, int Kp, const CUtensorMap& tmA, const CUtensorMap& tmB, Params p, long long M,
                      cudaStream_t st) {
  const size_t tile_bytes = 2ull * (Kp / BLOCK_K) * TILE_BYTES;  // the resident tile and one stage are the same size
  const size_t extra = 4 * 2 * BN * sizeof(float);              // per-tile column data
  const size_t fixed = 1024 + tile_bytes + 8 * sizeof(uint64_t) + extra;
  int stages = (int)((227 * 1024 - fixed) / tile_bytes);
  if (stages > 4) stages = 4;
  MM_REQUIRE(stages >= 2, MM_ERR_UNSUPPORTED, "%s: tiles do not fit two pipeline stages", who);
  p.stages = stages;
  const size_t smem = 1024 + tile_bytes + stages * tile_bytes + (stages + 2) * sizeof(uint64_t) + extra;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    mm::set_error("%s: cudaFuncSetAttribute failed: %s", who, cudaGetErrorString(e));
    return (int)e;
  }
  kern<<<(unsigned)((M + BM - 1) / BM), kThreads, smem, st>>>(tmA, tmB, p);
  return mm::check_launch(who);
}

}  // namespace ibw
}  // namespace mm

extern "C" {

int mm_tc_padded_k(int K);

int mm_inbatch_softmax_ce_backward(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                                   const void* neg_ids, int id_dtype, int downscore, float false_neg_score, const float* neg_prob,
                                   float temperature, const float* stats, const float* q, const float* pos, const float* row_scale,
                                   int row_scale_is_scalar, float* dq, float* dpos, float* dneg, float* loss, void* stream) {
  const char* who = "mm_inbatch_softmax_ce_backward";
  MM_REQUIRE(q_split && neg_split && stats && q && pos && row_scale && dq && dpos && dneg, MM_ERR_ARG,
             "%s: null pointer (operands, stats, q, pos, row_scale and the three gradients are required)", who);
  MM_REQUIRE(B >= 0 && N > 0 && D > 0, MM_ERR_ARG, "%s: bad size (B >= 0, N > 0, D > 0)", who);
  MM_REQUIRE(temperature > 0.0f, MM_ERR_ARG, "%s: temperature must be positive", who);
  MM_REQUIRE(!downscore || (pos_ids && neg_ids), MM_ERR_ARG, "%s: down-scoring needs positive and negative ids", who);
  MM_REQUIRE(id_dtype == MM_I32 || id_dtype == MM_I64, MM_ERR_ARG, "%s: bad id dtype", who);
  MM_REQUIRE(dpos != dneg || N == B, MM_ERR_ARG, "%s: dpos may alias dneg only when the negatives are the positives (N == B)", who);
  MM_REQUIRE(dq != dpos && dq != dneg, MM_ERR_ARG, "%s: dq must not alias dpos / dneg", who);
  const int Kp = mm_tc_padded_k(D);
  MM_REQUIRE(Kp <= 128, MM_ERR_UNSUPPORTED, "%s: D up to 128 (the resident tile is kept in shared memory)", who);
  MM_REQUIRE(B < (1ll << 31) && N < (1ll << 31), MM_ERR_UNSUPPORTED, "%s: sizes exceed 32-bit TMA coordinates", who);
  MM_REQUIRE(((uintptr_t)q_split % 16) == 0 && ((uintptr_t)neg_split % 16) == 0, MM_ERR_ALIGN,
             "%s: split operands must be 16-B aligned", who);
  MM_REQUIRE(((uintptr_t)stats | (uintptr_t)q | (uintptr_t)pos | (uintptr_t)row_scale | (uintptr_t)dq | (uintptr_t)dpos |
              (uintptr_t)dneg | (uintptr_t)(loss ? loss : stats)) % 4 == 0,
             MM_ERR_ALIGN, "%s: fp32 buffers must be 4-B aligned", who);
  if (B == 0) return MM_OK;
  using namespace mm::ibw;
  CUtensorMap tmQ, tmN;
  int rc = mm::tc::make_map(&tmQ, q_split, (uint64_t)B, (uint64_t)2 * Kp, BM);
  if (rc) return rc;
  rc = mm::tc::make_map(&tmN, neg_split, (uint64_t)N, (uint64_t)2 * Kp, BN);
  if (rc) return rc;
  Params p;
  memset(&p, 0, sizeof(p));
  p.D = D;
  p.id_is64 = id_dtype == MM_I64;
  (void)false_neg_score;  // a masked logit is the constant false_neg_score / T: its gradient is zero whatever the score
  p.inv_temp = 1.0f / temperature;
  p.neg_prob = neg_prob;
  p.stats = stats;
  p.row_scale = row_scale;
  p.scale_is_scalar = row_scale_is_scalar != 0;
  p.q = q;
  p.pos = pos;
  cudaStream_t st = (cudaStream_t)stream;
  // dQ: resident queries, streamed negatives; dpos written here unless it is dneg's buffer
  Params pq = p;
  pq.M = B;
  pq.I = N;
  pq.n_tiles = (int)((N + BN - 1) / BN);
  pq.row_ids = downscore ? pos_ids : nullptr;
  pq.col_ids = downscore ? neg_ids : nullptr;
  pq.out = dq;
  pq.dpos = dpos == dneg ? nullptr : dpos;
  rc = launch_bwd("inbatch_ce_dq_kernel", Kp == 64 ? inbatch_ce_dq_kernel<64> : inbatch_ce_dq_kernel<128>, Kp, tmQ, tmN, pq, B, st);
  if (rc) return rc;
  // dN: resident negatives, streamed queries; adds g[n,0] q[n] when dpos aliases dneg
  Params pn = p;
  pn.M = N;
  pn.I = B;
  pn.n_tiles = (int)((B + BN - 1) / BN);
  pn.row_ids = downscore ? neg_ids : nullptr;
  pn.col_ids = downscore ? pos_ids : nullptr;
  pn.out = dneg;
  pn.dpos = dpos == dneg ? dpos : nullptr;
  rc = launch_bwd("inbatch_ce_dn_kernel", Kp == 64 ? inbatch_ce_dn_kernel<64> : inbatch_ce_dn_kernel<128>, Kp, tmN, tmQ, pn, N, st);
  if (rc) return rc;
  if (loss) {
    inbatch_ce_loss_kernel<<<1, 1024, 0, st>>>(B, stats, row_scale, row_scale_is_scalar != 0, loss);
    rc = mm::check_launch("inbatch_ce_loss_kernel");
  }
  return rc;
}

}  // extern "C"
