// In-batch pairwise ranking losses (BPR, BPR-max, TOP1, TOP1-v2, TOP1-max, logistic, hinge; the reference's
// losses/pairwise.py) forward and backward without materialising the (B, N) scores: every 128x128 score tile is
// recomputed from the split-bf16 operands on wgmma and reduced or turned into its gradient tile in registers.
//
//   inbatch_pw_fwd_kernel  one CTA per 128 queries (resident), streams the negatives: per-row statistics
//                          [row loss, dloss/dsp, lse, A]; the -max kinds stream the negatives twice (pass 1: the row's
//                          log-sum-exp, which the eps0 decision of pass 2 needs)
//   inbatch_pw_dq_kernel   one CTA per 128 queries, streams the negatives:  S = Q N^T, dQ += G N
//   inbatch_pw_dn_kernel   one CTA per 128 negatives, streams the queries:  S^T = N Q^T, dN += G^T Q
//   inbatch_pw_loss_kernel loss += c sum_b rowloss[b] in a fixed order (one CTA)
//
// G = c / T * dloss/ds with c = 1 / (B N) (Keras' SUM_OVER_BATCH_SIZE over the (B, N) per-element losses; top1_v2's
// per-row mean over N and batch mean over B give the same c).  The element functions live in pairwise.cuh.  The GEMM
// structure is inbatch_bwd.cu's: two warpgroups of 64 resident rows over a TMA ring, thread 0 issuing the loads, the
// second product taking G from registers and the streamed tile as an MN-major B operand.  Every output row is owned by
// one CTA: no atomics, bit-reproducible.
#include <cstring>

#include "pairwise.cuh"
#include "tc_common.cuh"
#include "tc_trans.cuh"

extern "C" int mm_tc_padded_k(int K);

namespace mm {
namespace ipw {

using namespace mm::tc;
using namespace mm::pw;

constexpr int BM = 128, BN = 128, BLOCK_K = 64, MMA_K = 16;
constexpr int kThreads = 256;
constexpr uint32_t TILE_BYTES = 128 * BLOCK_K * 2;
constexpr int FWD = 0, DQ = 1, DN = 2;

struct Params {
  long long M, I;  // resident rows, streamed rows
  int D, stages, n_tiles, passes;
  const void* row_ids;  // ids of the resident rows / streamed rows (null: no down-scoring)
  const void* col_ids;
  int id_is64;
  float inv_temp, masked_score, lambda, c;
  const float* pos_logit;  // (B,) the positive scores sp (already / T)
  float* stats;            // (B, 4) [row loss, dloss/dsp, lse, A]: written by the forward, read by the backward
  const float* q;          // (B, D) fp32
  const float* pos;        // (B, D) fp32
  float* out;              // dq (B, D) or dneg (N, D)
  float* dpos;             // dq kernel: dpos when it is its own buffer; dn kernel: non-null = dpos aliases dneg (add g0 q)
};

__device__ __forceinline__ long long id_at(const void* p, long long i, int is64) {
  return is64 ? reinterpret_cast<const long long*>(p)[i] : (long long)reinterpret_cast<const int*>(p)[i];
}

template <int MODE, int KP, int KIND>
__device__ __forceinline__ void pw_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const Params& p) {
  constexpr bool TRANS = MODE == DN;
  constexpr bool MAXK = is_max<KIND>::value;
  constexpr int KB = KP / BLOCK_K;
  constexpr uint32_t A_BYTES = 2u * KB * TILE_BYTES;
  constexpr uint32_t STAGE_BYTES = 2u * KB * TILE_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + (size_t)p.stages * STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* a_full = bars + p.stages;
  // per streamed tile, double-buffered: dN: the query's sp, lse and A; every kernel: the column ids
  float* col_sp = reinterpret_cast<float*>(bars + p.stages + 2);  // [2][128]
  float* col_l = col_sp + 2 * BN;                                 // [2][128]
  float* col_a = col_l + 2 * BN;                                  // [2][128]
  int* ids_lo = reinterpret_cast<int*>(col_a + 2 * BN);           // [2][128]
  int* ids_hi = ids_lo + 2 * BN;                                  // [2][128]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long m0 = (long long)blockIdx.x * BM;
  const int total = p.passes * p.n_tiles;
  auto load_tile = [&](int t) {
    const int stage = t % p.stages;
    const int tile = t % p.n_tiles;
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

  const int wg = warp >> 2;
  const int part = lane & 3;
  const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  const bool do_mask = p.row_ids != nullptr;
  long long row[2], my_id[2] = {0, 0};
  bool rvalid[2];
  float r_sp[2] = {0.0f, 0.0f}, r_lse[2] = {0.0f, 0.0f}, r_a[2] = {0.0f, 0.0f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row[h] = m0 + frow + 8 * h;
    rvalid[h] = row[h] < p.M;
    if (rvalid[h]) {
      if (!TRANS) r_sp[h] = p.pos_logit[row[h]];
      if (MODE == DQ) {
        r_lse[h] = p.stats[row[h] * 4 + 2];
        r_a[h] = p.stats[row[h] * 4 + 3];
      }
      if (do_mask) my_id[h] = id_at(p.row_ids, row[h], p.id_is64);
    }
  }
  // forward: per row, this thread's partials over the columns it sees (the four lanes of a quad share a row)
  RowAcc racc[2];
  float run_m[2] = {-INFINITY, -INFINITY}, run_s[2] = {0.0f, 0.0f};
  float dacc[64];
  if (MODE != FWD) {
#pragma unroll
    for (int i = 0; i < 64; ++i) dacc[i] = 0.0f;
  }
  int stage = 0, buf = 0;
  uint32_t phase = 0;
  mbar_wait(smem_u32(a_full), 0);
  const uint32_t a_base = smem_u32(smem_a) + (uint32_t)wg * (TILE_BYTES / 2);
  for (int t = 0; t < total; ++t) {
    const int pass = t / p.n_tiles;
    const long long n0 = (long long)(t - pass * p.n_tiles) * BN;
    float* csp = col_sp + buf * BN;
    float* cl_ = col_l + buf * BN;
    float* ca = col_a + buf * BN;
    int* cl = ids_lo + buf * BN;
    int* chh = ids_hi + buf * BN;
    buf ^= 1;
    named_bar(1, kThreads);
    if (threadIdx.x == 0 && t > 0 && t - 1 + p.stages < total) load_tile(t - 1 + p.stages);
    for (int i = threadIdx.x; i < BN; i += kThreads) {
      const long long c = n0 + i;
      const bool in = c < p.I;
      if (TRANS) {
        csp[i] = in ? p.pos_logit[c] : 0.0f;
        cl_[i] = in ? p.stats[c * 4 + 2] : 0.0f;
        ca[i] = in ? p.stats[c * 4 + 3] : 0.0f;
      }
      if (do_mask) {
        const long long cid = in ? id_at(p.col_ids, c, p.id_is64) : 0;
        cl[i] = (int)cid;
        chh[i] = (int)(cid >> 32);
      }
    }
    named_bar(1, kThreads);

    // ---- S: 64 x 128 scores of this warpgroup (3-pass split-bf16 product) ----
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

    // acc[4 j + 2 h + e]: row h, column 8 j + 2 part + e
    const bool ragged = n0 + BN > p.I;
    if (MODE == FWD && MAXK && pass == 0) {
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
            float s = acc[i] * p.inv_temp;
            if (do_mask && cl[c] == (int)my_id[h] && chh[c] == (int)(my_id[h] >> 32)) s = p.masked_score;
            if (ragged && n0 + c >= p.I) s = -INFINITY;
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
      if (t == p.n_tiles - 1) {
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
          r_lse[h] = run_m[h] + logf(run_s[h]);
        }
      }
    } else if (MODE == FWD) {
      // ---- the per-element losses of this tile into the row sums ----
#pragma unroll
      for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * j + 2 * part + e;
            const int i = 4 * j + 2 * h + e;
            const bool valid = rvalid[h] && !(ragged && n0 + c >= p.I);
            float s = acc[i] * p.inv_temp;
            if (do_mask && cl[c] == (int)my_id[h] && chh[c] == (int)(my_id[h] >> 32)) s = p.masked_score;
            fwd_elem<KIND>(valid, s, r_sp[h], r_lse[h], p.lambda, racc[h]);
          }
        }
      }
    } else {
      // ---- G = c / T dloss/ds, zero where masked (a constant score) or outside the matrix ----
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
            const float s = acc[i] * p.inv_temp;
            const float g = TRANS ? bwd_elem<KIND>(s, csp[c], cl_[c], ca[c], p.lambda)
                                  : bwd_elem<KIND>(s, r_sp[h], r_lse[h], r_a[h], p.lambda);
            acc[i] = ok ? p.c * p.inv_temp * g : 0.0f;
          }
        }
      }
      uint32_t ghi[32], glo[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) split_pair(acc[2 * i], acc[2 * i + 1], ghi[i], glo[i]);

      // ---- dX += G . X_tile: 3-pass split, X as the MN-major B operand ----
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
      RowAcc& a = racc[h];
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
        const float A = fwd_row<KIND>(r_sp[h], p.lambda, a);
        float4 v = make_float4(a.loss, a.gp, r_lse[h], A);
        *reinterpret_cast<float4*>(p.stats + row[h] * 4) = v;
      }
    }
  } else {
    // ---- epilogue: dacc[4 j + 2 h + e] is output row h, feature column 8 j + 2 part + e ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!rvalid[h]) continue;
      const long long r = row[h];
      const bool add = TRANS ? p.dpos != nullptr : true;
      const float g0 = add ? p.c * p.inv_temp * p.stats[r * 4 + 1] : 0.0f;
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
}

template <int MODE, int KP, int KIND>
__global__ void __launch_bounds__(kThreads, 1)
inbatch_pw_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Params p) {
  pw_body<MODE, KP, KIND>(tmA, tmB, p);
}

// loss[0] += c sum_b stats[b, 0]: one CTA, fixed summation order (double per thread, then a tree)
__global__ void inbatch_pw_loss_kernel(long long B, const float* __restrict__ stats, double c, float* __restrict__ loss) {
  __shared__ double part[1024];
  double s = 0.0;
  for (long long b = threadIdx.x; b < B; b += blockDim.x) s += (double)stats[b * 4];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] += (float)(c * part[0]);
}

typedef void (*Kernel)(const CUtensorMap, const CUtensorMap, const Params);

template <int MODE, int KP>
static Kernel pick(int kind) {
  switch (kind) {
    case BPR: return inbatch_pw_kernel<MODE, KP, BPR>;
    case BPR_MAX: return inbatch_pw_kernel<MODE, KP, BPR_MAX>;
    case TOP1: return inbatch_pw_kernel<MODE, KP, TOP1>;
    case TOP1_V2: return inbatch_pw_kernel<MODE, KP, TOP1_V2>;
    case TOP1_MAX: return inbatch_pw_kernel<MODE, KP, TOP1_MAX>;
    case LOGISTIC: return inbatch_pw_kernel<MODE, KP, LOGISTIC>;
    default: return inbatch_pw_kernel<MODE, KP, HINGE>;
  }
}
template <int MODE>
static Kernel pick(int Kp, int kind) {
  return Kp == 64 ? pick<MODE, 64>(kind) : pick<MODE, 128>(kind);
}

static int launch(const char* who, Kernel kern, int Kp, const CUtensorMap& tmA, const CUtensorMap& tmB, Params p, long long M,
                  cudaStream_t st) {
  const size_t tile_bytes = 2ull * (Kp / BLOCK_K) * TILE_BYTES;  // the resident tile and one stage are the same size
  const size_t extra = 5 * 2 * BN * sizeof(float);              // per-tile column data
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

// the argument rules both entry points share; fills the maps and the common parameters
static int prepare(const char* who, const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                   const void* neg_ids, int id_dtype, int downscore, float false_neg_score, float temperature, int kind,
                   float reg_lambda, const float* pos_logit, const float* stats, int* Kp, CUtensorMap* tmQ, CUtensorMap* tmN,
                   Params* p) {
  MM_REQUIRE(q_split && neg_split && pos_logit && stats, MM_ERR_ARG, "%s: null pointer (operands, pos_logit and stats are required)",
             who);
  MM_REQUIRE(B >= 0 && N > 0 && D > 0, MM_ERR_ARG, "%s: bad size (B >= 0, N > 0, D > 0)", who);
  MM_REQUIRE(temperature > 0.0f, MM_ERR_ARG, "%s: temperature must be positive", who);
  MM_REQUIRE(kind >= 0 && kind < N_KINDS, MM_ERR_ARG, "%s: unknown loss kind %d", who, kind);
  MM_REQUIRE(reg_lambda == reg_lambda && reg_lambda < INFINITY && reg_lambda > -INFINITY, MM_ERR_ARG, "%s: reg_lambda must be finite",
             who);
  MM_REQUIRE(!downscore || (pos_ids && neg_ids), MM_ERR_ARG, "%s: down-scoring needs positive and negative ids", who);
  MM_REQUIRE(id_dtype == MM_I32 || id_dtype == MM_I64, MM_ERR_ARG, "%s: bad id dtype", who);
  *Kp = mm_tc_padded_k(D);
  MM_REQUIRE(*Kp <= 128, MM_ERR_UNSUPPORTED, "%s: D up to 128 (the resident tile is kept in shared memory)", who);
  MM_REQUIRE(B < (1ll << 31) && N < (1ll << 31), MM_ERR_UNSUPPORTED, "%s: sizes exceed 32-bit TMA coordinates", who);
  MM_REQUIRE(((uintptr_t)q_split % 16) == 0 && ((uintptr_t)neg_split % 16) == 0 && ((uintptr_t)stats % 16) == 0, MM_ERR_ALIGN,
             "%s: split operands and stats must be 16-B aligned", who);
  MM_REQUIRE(((uintptr_t)pos_logit % 4) == 0, MM_ERR_ALIGN, "%s: fp32 buffers must be 4-B aligned", who);
  if (B == 0) return MM_OK;
  int rc = make_map(tmQ, q_split, (uint64_t)B, (uint64_t)2 * *Kp, BM);
  if (rc) return rc;
  rc = make_map(tmN, neg_split, (uint64_t)N, (uint64_t)2 * *Kp, BN);
  if (rc) return rc;
  memset(p, 0, sizeof(*p));
  p->D = D;
  p->id_is64 = id_dtype == MM_I64;
  p->inv_temp = 1.0f / temperature;
  p->masked_score = false_neg_score * p->inv_temp;  // the forward's order: rescore, then divide by T
  p->lambda = reg_lambda;
  p->c = (float)(1.0 / ((double)B * (double)N));
  p->pos_logit = pos_logit;
  p->stats = const_cast<float*>(stats);
  return MM_OK;
}

}  // namespace ipw
}  // namespace mm

extern "C" {

int mm_inbatch_pairwise_fwd(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                            const void* neg_ids, int id_dtype, int downscore, float false_neg_score, float temperature, int kind,
                            float reg_lambda, const float* pos_logit, float* stats, float* loss, void* stream) {
  const char* who = "mm_inbatch_pairwise_fwd";
  using namespace mm::ipw;
  MM_REQUIRE(((uintptr_t)loss % 4) == 0, MM_ERR_ALIGN, "%s: loss must be 4-B aligned", who);
  int Kp = 0;
  CUtensorMap tmQ, tmN;
  Params p;
  int rc = prepare(who, q_split, neg_split, B, N, D, pos_ids, neg_ids, id_dtype, downscore, false_neg_score, temperature, kind,
                   reg_lambda, pos_logit, stats, &Kp, &tmQ, &tmN, &p);
  if (rc || B == 0) return rc;
  p.M = B;
  p.I = N;
  p.n_tiles = (int)((N + BN - 1) / BN);
  p.passes = (kind == mm::pw::BPR_MAX || kind == mm::pw::TOP1_MAX) ? 2 : 1;
  p.row_ids = downscore ? pos_ids : nullptr;
  p.col_ids = downscore ? neg_ids : nullptr;
  cudaStream_t st = (cudaStream_t)stream;
  rc = launch("inbatch_pw_fwd_kernel", pick<FWD>(Kp, kind), Kp, tmQ, tmN, p, B, st);
  if (rc) return rc;
  if (loss) {
    inbatch_pw_loss_kernel<<<1, 1024, 0, st>>>(B, stats, 1.0 / ((double)B * (double)N), loss);
    rc = mm::check_launch("inbatch_pw_loss_kernel");
  }
  return rc;
}

int mm_inbatch_pairwise_bwd(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                            const void* neg_ids, int id_dtype, int downscore, float false_neg_score, float temperature, int kind,
                            float reg_lambda, const float* pos_logit, const float* stats, const float* q, const float* pos,
                            float* dq, float* dpos, float* dneg, void* stream) {
  const char* who = "mm_inbatch_pairwise_bwd";
  using namespace mm::ipw;
  MM_REQUIRE(q && pos && dq && dpos && dneg, MM_ERR_ARG, "%s: null pointer (q, pos and the three gradients are required)", who);
  MM_REQUIRE(dpos != dneg || N == B, MM_ERR_ARG, "%s: dpos may alias dneg only when the negatives are the positives (N == B)", who);
  MM_REQUIRE(dq != dpos && dq != dneg, MM_ERR_ARG, "%s: dq must not alias dpos / dneg", who);
  MM_REQUIRE(((uintptr_t)q | (uintptr_t)pos | (uintptr_t)dq | (uintptr_t)dpos | (uintptr_t)dneg) % 4 == 0, MM_ERR_ALIGN,
             "%s: fp32 buffers must be 4-B aligned", who);
  int Kp = 0;
  CUtensorMap tmQ, tmN;
  Params p;
  int rc = prepare(who, q_split, neg_split, B, N, D, pos_ids, neg_ids, id_dtype, downscore, false_neg_score, temperature, kind,
                   reg_lambda, pos_logit, stats, &Kp, &tmQ, &tmN, &p);
  if (rc || B == 0) return rc;
  p.q = q;
  p.pos = pos;
  p.passes = 1;
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
  rc = launch("inbatch_pw_dq_kernel", pick<DQ>(Kp, kind), Kp, tmQ, tmN, pq, B, st);
  if (rc) return rc;
  // dN: resident negatives, streamed queries; adds g0[n] q[n] when dpos aliases dneg
  Params pn = p;
  pn.M = N;
  pn.I = B;
  pn.n_tiles = (int)((B + BN - 1) / BN);
  pn.row_ids = downscore ? neg_ids : nullptr;
  pn.col_ids = downscore ? pos_ids : nullptr;
  pn.out = dneg;
  pn.dpos = dpos == dneg ? dpos : nullptr;
  return launch("inbatch_pw_dn_kernel", pick<DN>(Kp, kind), Kp, tmN, tmQ, pn, N, st);
}

}  // extern "C"
