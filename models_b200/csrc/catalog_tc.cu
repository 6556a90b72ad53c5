// Query x catalog scoring without materialising the (B, N_I) logits: wgmma GEMM whose epilogue
// streams every 128x128 logits tile straight into per-row running statistics —
//   * soft-max cross-entropy inputs: row max, log-sum-exp, logit of the target item
//     (CategoricalCrossEntropy(from_logits=True), merlin/models/tf/losses/listwise.py:38-50), and/or
//   * top-k scores + item ids (tf.math.top_k: outputs/topk.py:221-223, core/index.py:236-237).
// Logits: x @ E^T (+ bias) as in EmbeddingTablePrediction.call (outputs/classification.py:347-357)
// and ItemRetrievalScorer._get_logits_for_sampled_softmax (blocks/retrieval/base.py:431-438).
//
// Work item = (128-query block, split of the item range).  The query tile (A, split-bf16) is
// loaded once per work item and stays in shared memory; item tiles (B operand, 128 items x Kp,
// split-bf16, precomputed once per catalog with mm_split_rows) stream through a TMA pipeline that
// refills while the consumers reduce.  CTA = two consumer warpgroups (64 query rows each) + one TMA
// producer warp.  The reduction works on the wgmma accumulator fragment in registers: a thread holds
// two query rows and, of every tile, the 32 columns 8 j + 2 (lane % 4) + {0, 1}; it keeps (max,
// sum-exp, target logit, top-k list) per row for the columns it sees, so the four lanes of a quad are
// the kParts partial results of a row.  Partials go to a small workspace and a second kernel merges
// the kParts*S partials per row.  3-pass split-bf16 = fp32-grade logits.
#include <cstring>

#include "tc_common.cuh"

namespace mm {
namespace cat {

using namespace mm::tc;

constexpr int BM = 128, BN = 128, BLOCK_K = 64, MMA_K = 16;
constexpr int kConsumerWarps = 8;                // two warpgroups
constexpr int kParts = 4;                        // partial results per (row, item-range split): the lanes of a quad
constexpr int kThreads = 32 * (kConsumerWarps + 1);  // + warp 8: TMA producer
constexpr int MAX_K = 32;  // top-k list length held per thread and row
constexpr uint32_t TILE_BYTES = 128 * BLOCK_K * 2;  // one 128-row x 64-col bf16 tile = 16 KB

struct Params {
  long long M, I;
  int Kp, KB, stages, S, tiles_per_split, n_tiles;
  const float* bias;
  const void* targets;
  int id_is64;
  int do_lse, topk;
  float* ws_lse;         // (M, kParts*S, 3)
  float* ws_vals;        // (M, kParts*S, topk)
  long long* ws_ids;     // (M, kParts*S, topk)
  // in-batch contrastive extras (mm_inbatch_softmax_ce): logit = mask(dot + bias) * inv_temp with
  // mask: row_ids[r] == col_ids[c] -> false_neg_score (utils/tf_utils.py:126-154)
  int bias_is_prob;      // bias[c] holds a sampling probability: use -log(p + 1e-16) (outputs/contrastive.py:317-319)
  const void* row_ids;
  const void* col_ids;
  float false_neg_score, inv_temp;
};

// insert (x, id) into the descending list (tv, ti) of length k (x > tv[k-1] is known); returns the new k-th value
static __device__ __noinline__ float topk_insert(float* tv, long long* ti, int k, float x, long long id) {
  int pos = k - 1;
  while (pos > 0 && tv[pos - 1] < x) {
    tv[pos] = tv[pos - 1];
    ti[pos] = ti[pos - 1];
    --pos;
  }
  tv[pos] = x;
  ti[pos] = id;
  return tv[k - 1];
}

// LSE / TOPK / MASK select the epilogue at compile time: the log-sum-exp-only variants keep no top-k list (64 local
// words per thread and row otherwise) and the unmasked ones no id compares.
template <bool LSE, bool TOPK, bool MASK>
__global__ void __launch_bounds__(kThreads, 1)
catalog_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // pointer arithmetic keeps the shared state space (LDS/STS, not generic LD/ST)
  const uint32_t A_BYTES = 2u * p.KB * TILE_BYTES;      // [hi kb0..][lo kb0..]
  const uint32_t STAGE_BYTES = 2u * p.KB * TILE_BYTES;  // one item tile, all k-blocks, hi + lo
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + (size_t)p.stages * STAGE_BYTES);
  uint64_t* full_bar = bars;                        // [stages]
  uint64_t* empty_bar = bars + p.stages;            // [stages] one arrive per consumer warp
  uint64_t* a_full = bars + 2 * p.stages;           // [1]
  uint64_t* a_empty = bars + 2 * p.stages + 1;      // [1] one arrive per consumer warp
  float* bias_s = reinterpret_cast<float*>(bars + 2 * p.stages + 2);  // [2][128]
  int* ids_lo = reinterpret_cast<int*>(bias_s + 2 * BN);                // [2][128] low words of the column ids (MASK)
  int* ids_hi = ids_lo + 2 * BN;                                        // [2][128] high words

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long m_blocks = (p.M + BM - 1) / BM;
  const long long items = m_blocks * p.S;

  if (warp == kConsumerWarps && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(full_bar + s), 1);
      mbar_init(smem_u32(empty_bar + s), kConsumerWarps);
    }
    mbar_init(smem_u32(a_full), 1);
    mbar_init(smem_u32(a_empty), kConsumerWarps);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0, a_phase = 0;
      for (long long item = blockIdx.x; item < items; item += gridDim.x) {
        const int m0 = (int)(item / p.S) * BM;
        const int split = (int)(item % p.S);
        const int t0 = split * p.tiles_per_split, t1 = min(p.n_tiles, t0 + p.tiles_per_split);
        // query tile: reused by every item tile of this work item
        mbar_wait(smem_u32(a_empty), a_phase ^ 1);
        mbar_expect_tx(smem_u32(a_full), A_BYTES);
        for (int kb = 0; kb < p.KB; ++kb) {
          tma_load_2d(smem_u32(smem_a + kb * TILE_BYTES), &tmA, smem_u32(a_full), kb * BLOCK_K, m0);
          tma_load_2d(smem_u32(smem_a + (p.KB + kb) * TILE_BYTES), &tmA, smem_u32(a_full), p.Kp + kb * BLOCK_K, m0);
        }
        a_phase ^= 1;
        for (int t = t0; t < t1; ++t) {
          mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
          const uint32_t fb = smem_u32(full_bar + stage);
          uint8_t* st = smem_b + (size_t)stage * STAGE_BYTES;
          mbar_expect_tx(fb, STAGE_BYTES);
          for (int kb = 0; kb < p.KB; ++kb) {
            tma_load_2d(smem_u32(st + kb * TILE_BYTES), &tmB, fb, kb * BLOCK_K, t * BN);
            tma_load_2d(smem_u32(st + (p.KB + kb) * TILE_BYTES), &tmB, fb, p.Kp + kb * BLOCK_K, t * BN);
          }
          if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumers: MMA + streaming reduction =====================
    // Per logit: one FMNMX for the chunk maximum, then FFMA + MUFU.EX2 + FADD into one of four independent
    // partial sums.
    const int wg = warp >> 2;
    const int part = lane & 3;
    const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // tile row of fragment row 0 (row 1 is 8 further)
    int stage = 0, buf = 0;
    uint32_t phase = 0, a_phase = 0;
    const float LOG2E = 1.4426950408889634f;
    const bool has_bias = p.bias != nullptr;
    for (long long item = blockIdx.x; item < items; item += gridDim.x) {
      const long long m0 = (item / p.S) * BM;
      const int split = (int)(item % p.S);
      const int t0 = split * p.tiles_per_split, t1 = min(p.n_tiles, t0 + p.tiles_per_split);
      long long row[2], target[2] = {-1, -1}, my_id[2] = {0, 0};
      const bool do_mask = MASK && p.row_ids != nullptr;
      float run_m[2], run_s[2], tlogit[2], thr[2];
      float tv[2][TOPK ? MAX_K : 1];
      long long ti[2][TOPK ? MAX_K : 1];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        row[h] = m0 + frow + 8 * h;
        if (LSE && p.targets && row[h] < p.M)
          target[h] = p.id_is64 ? reinterpret_cast<const long long*>(p.targets)[row[h]]
                                : (long long)reinterpret_cast<const int*>(p.targets)[row[h]];
        if (do_mask && row[h] < p.M)
          my_id[h] = p.id_is64 ? reinterpret_cast<const long long*>(p.row_ids)[row[h]]
                               : (long long)reinterpret_cast<const int*>(p.row_ids)[row[h]];
        run_m[h] = -INFINITY;
        run_s[h] = 0.0f;
        tlogit[h] = __int_as_float(0x7fc00000);  // NaN = "not seen"
        thr[h] = -INFINITY;  // k-th best value of this row's list (register copy of tv[h][topk-1])
        if (TOPK) {
#pragma unroll
          for (int r = 0; r < MAX_K; ++r) {
            tv[h][r] = -INFINITY;
            ti[h][r] = -1;
          }
        }
      }
      mbar_wait(smem_u32(a_full), a_phase);
      a_phase ^= 1;
      const uint32_t a_base = smem_u32(smem_a) + (uint32_t)wg * (TILE_BYTES / 2);
      for (int t = t0; t < t1; ++t) {
        const long long n0 = (long long)t * BN;
        float* bs = bias_s + buf * BN;
        int* cl = ids_lo + buf * BN;
        int* chh = ids_hi + buf * BN;
        buf ^= 1;
        if (has_bias || do_mask) {  // per-tile column data -> shared memory (the buffer of tile t-2 is free: its readers passed bar 1 of t-1)
          named_bar(1, 32 * kConsumerWarps);
          for (int i = threadIdx.x; i < BN; i += 32 * kConsumerWarps) {
            const bool in = n0 + i < p.I;
            if (has_bias) {
              float bv = in ? p.bias[n0 + i] : 0.0f;
              if (p.bias_is_prob) bv = -logf(bv + 1e-16f);
              bs[i] = bv;
            }
            if (do_mask) {
              const long long cid = !in ? (long long)0x7fffffffffffffffll
                                        : (p.id_is64 ? reinterpret_cast<const long long*>(p.col_ids)[n0 + i]
                                                     : (long long)reinterpret_cast<const int*>(p.col_ids)[n0 + i]);
              cl[i] = (int)cid;
              chh[i] = (int)(cid >> 32);
            }
          }
          named_bar(1, 32 * kConsumerWarps);
        }
        // ---- 64 x 128 logits of this warpgroup ----
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
        mbar_wait(smem_u32(full_bar + stage), phase);
        const uint32_t b_base = smem_u32(smem_b + (size_t)stage * STAGE_BYTES);
        wgmma_fence_acc(acc);
        wgmma_fence();
        for (int kb = 0; kb < p.KB; ++kb) {
          const uint32_t a_hi = a_base + kb * TILE_BYTES, a_lo = a_base + (p.KB + kb) * TILE_BYTES;
          const uint32_t b_hi = b_base + kb * TILE_BYTES, b_lo = b_base + (p.KB + kb) * TILE_BYTES;
#pragma unroll
          for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss(BN, acc, make_desc_sw128(a_hi + k * 32), make_desc_sw128(b_lo + k * 32));
#pragma unroll
          for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss(BN, acc, make_desc_sw128(a_lo + k * 32), make_desc_sw128(b_hi + k * 32));
#pragma unroll
          for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss(BN, acc, make_desc_sw128(a_hi + k * 32), make_desc_sw128(b_hi + k * 32));
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_acc(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(empty_bar + stage));
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // fragment row h: v[j] is column 8 (j / 2) + 2 part + (j % 2) of the tile (ascending in j)
          float v[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = acc[4 * (j >> 1) + 2 * h + (j & 1)];
          if (has_bias) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] += bs[8 * (j >> 1) + 2 * part + (j & 1)];
          }
          if (MASK) {
            if (do_mask) {  // compare the low words; the high word only on a low-word match
              const int my_lo = (int)my_id[h], my_hi = (int)(my_id[h] >> 32);
#pragma unroll
              for (int j = 0; j < 32; j += 2) {
                const int c = 8 * (j >> 1) + 2 * part;
                const int2 c2 = *reinterpret_cast<const int2*>(cl + c);
                if (c2.x == my_lo && chh[c] == my_hi) v[j] = p.false_neg_score;
                if (c2.y == my_lo && chh[c + 1] == my_hi) v[j + 1] = p.false_neg_score;
              }
            }
            if (p.inv_temp != 1.0f) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] *= p.inv_temp;
            }
          }
          if (n0 + BN > p.I) {  // ragged last tile only
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (n0 + 8 * (j >> 1) + 2 * part + (j & 1) >= p.I) v[j] = -INFINITY;
          }
          float cmax = v[0];
#pragma unroll
          for (int j = 1; j < 32; ++j) cmax = fmaxf(cmax, v[j]);
          if (LSE && cmax > -INFINITY) {
            const float m_new = fmaxf(run_m[h], cmax);
            const float mb = m_new * LOG2E;
            float s0 = run_s[h] * ex2_approx(fmaf(run_m[h], LOG2E, -mb)), s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;  // run_m = -inf -> 0
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              s0 += ex2_approx(fmaf(v[j], LOG2E, -mb));
              s1 += ex2_approx(fmaf(v[j + 1], LOG2E, -mb));
              s2 += ex2_approx(fmaf(v[j + 2], LOG2E, -mb));
              s3 += ex2_approx(fmaf(v[j + 3], LOG2E, -mb));
            }
            run_m[h] = m_new;
            run_s[h] = (s0 + s1) + (s2 + s3);
            const long long dt = target[h] - n0 - 2 * part;
            if (dt >= 0 && dt < BN) {  // predicated selects (a dynamic v[dt] would put v[] in local memory)
              const int di = (int)dt;
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (di == 8 * (j >> 1) + (j & 1)) tlogit[h] = v[j];
            }
          }
          if (TOPK && cmax > thr[h]) {
            // ascending item order inside a thread; strict '>' keeps the lower id on ties.  The values stay in
            // registers (fully unrolled compares against the list's k-th value); only the rare insertion touches
            // the list, which lives in local memory.
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (v[j] > thr[h]) thr[h] = topk_insert(tv[h], ti[h], p.topk, v[j], n0 + 8 * (j >> 1) + 2 * part + (j & 1));
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(a_empty));  // every MMA of this warp that read the query tile has completed
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (row[h] < p.M) {
          const long long pidx = row[h] * ((long long)kParts * p.S) + split * kParts + part;
          if (LSE) {
            p.ws_lse[pidx * 3 + 0] = run_m[h];
            p.ws_lse[pidx * 3 + 1] = run_s[h];
            p.ws_lse[pidx * 3 + 2] = tlogit[h];
          }
          if (TOPK) {
            for (int r = 0; r < p.topk; ++r) {
              p.ws_vals[pidx * p.topk + r] = tv[h][r];
              p.ws_ids[pidx * p.topk + r] = ti[h][r];
            }
          }
        }
      }
    }
  }
}

// merge the kParts*S partials of every row: one warp per row.  `extra` (nullable): one more logit per row that is
// part of the soft-max AND is the target — the positive column of the in-batch contrastive logits.
__global__ void catalog_merge_kernel(long long M, int P, int do_lse, int topk, const float* __restrict__ ws_lse,
                                     const float* __restrict__ ws_vals, const long long* __restrict__ ws_ids,
                                     float* __restrict__ out_stats, float* __restrict__ out_scores,
                                     long long* __restrict__ out_ids, const float* __restrict__ extra) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long row = warp0; row < M; row += n_warps) {
    if (do_lse) {
      float m = -INFINITY, tl = __int_as_float(0x7fc00000);
      for (int i = lane; i < P; i += 32) {
        m = fmaxf(m, ws_lse[(row * P + i) * 3]);
        const float t = ws_lse[(row * P + i) * 3 + 2];
        if (t == t) tl = t;
      }
      m = warp_max(m);
      const float ex = extra ? extra[row] : -INFINITY;
      if (extra) {
        m = fmaxf(m, ex);
        tl = ex;
      }
      float s = (extra && lane == 0) ? expf(ex - m) : 0.0f;
      for (int i = lane; i < P; i += 32) {
        const float mi = ws_lse[(row * P + i) * 3];
        if (mi > -INFINITY) s += ws_lse[(row * P + i) * 3 + 1] * expf(mi - m);
      }
      s = warp_sum(s);
      // the target logit lives in exactly one partial (or is the extra logit)
      unsigned has = __ballot_sync(0xffffffffu, tl == tl);
      if (has && !extra) tl = __shfl_sync(0xffffffffu, tl, __ffs(has) - 1);
      if (lane == 0) {
        out_stats[row * 3 + 0] = m;
        out_stats[row * 3 + 1] = m + logf(s);
        out_stats[row * 3 + 2] = tl;
      }
    }
    if (topk > 0) {
      // k rounds of warp arg-max over the P*topk candidates, (value desc, id asc); picked ones are skipped
      const int C = P * topk;
      float last_v = INFINITY;
      long long last_i = -1;
      for (int r = 0; r < topk; ++r) {
        float bv = -INFINITY;
        long long bi = 0x7fffffffffffffffll;
        for (int c = lane; c < C; c += 32) {
          const float v = ws_vals[row * C + c];
          const long long id = ws_ids[row * C + c];
          if (id < 0) continue;
          // strictly after the previously emitted (value, id) in the output order
          const bool after = (v < last_v) || (v == last_v && id > last_i);
          if (!after) continue;
          if (v > bv || (v == bv && id < bi)) {
            bv = v;
            bi = id;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ov > bv || (ov == bv && oi < bi)) {
            bv = ov;
            bi = oi;
          }
        }
        if (lane == 0) {
          out_scores[row * topk + r] = bv;
          out_ids[row * topk + r] = (bi == 0x7fffffffffffffffll) ? -1 : bi;
        }
        last_v = bv;
        last_i = bi;
      }
    }
  }
}

static int splits_for(long long M, long long I) {
  const long long m_blocks = (M + BM - 1) / BM;
  const long long n_tiles = (I + BN - 1) / BN;
  long long S = (4ll * sm_count() + m_blocks - 1) / m_blocks;
  if (S > n_tiles) S = n_tiles;
  if (S > 64) S = 64;
  if (S < 1) S = 1;
  return (int)S;
}

}  // namespace cat
}  // namespace mm

extern "C" {

int mm_tc_padded_k(int K);

int64_t mm_catalog_workspace_bytes(int64_t B, int64_t I, int k) {
  if (B <= 0 || I <= 0 || k < 0) return 0;
  const int64_t P = (int64_t)mm::cat::kParts * mm::cat::splits_for(B, I);
  return B * P * (3 * (int64_t)sizeof(float) + (int64_t)k * (sizeof(float) + sizeof(long long))) + 256;
}

}  // extern "C"

namespace mm {
namespace cat {

struct Extras {  // in-batch contrastive additions; all null / neutral for plain catalog scoring
  int contrastive = 0;
  int bias_is_prob = 0;
  const void* row_ids = nullptr;
  const void* col_ids = nullptr;
  float false_neg_score = 0.0f, inv_temp = 1.0f;
  const float* extra_logit = nullptr;
};

static int launch(const char* who, const void* q_split, int64_t B, int D, const void* e_split, int64_t I, const float* bias,
                  const void* targets, int id_dtype, float* out_stats, int k, float* topk_scores, int64_t* topk_ids,
                  void* workspace, int64_t workspace_bytes, const Extras& ex, void* stream) {
  MM_REQUIRE(q_split && e_split && workspace && B >= 0 && I > 0 && D > 0, MM_ERR_ARG, "%s: null pointer or bad size", who);
  MM_REQUIRE(out_stats || k > 0, MM_ERR_ARG, "%s: nothing requested (out_stats null and k == 0)", who);
  MM_REQUIRE(k >= 0 && k <= MAX_K && (k == 0 || (topk_scores && topk_ids)), MM_ERR_ARG,
             "%s: k must be 0..%d with score/id outputs", who, MAX_K);
  MM_REQUIRE(k <= I, MM_ERR_ARG, "%s: k exceeds the catalog size", who);
  MM_REQUIRE(id_dtype == MM_I32 || id_dtype == MM_I64, MM_ERR_ARG, "%s: bad id dtype", who);
  const int Kp = mm_tc_padded_k(D);
  MM_REQUIRE(Kp <= 128, MM_ERR_UNSUPPORTED, "%s: D up to 128 (query tile is kept resident in shared memory)", who);
  MM_REQUIRE(B < (1ll << 31) && I < (1ll << 31), MM_ERR_UNSUPPORTED, "%s: sizes exceed 32-bit TMA coordinates", who);
  MM_REQUIRE(workspace_bytes >= mm_catalog_workspace_bytes(B, I, k), MM_ERR_ARG, "%s: workspace too small (%lld < %lld)", who,
             (long long)workspace_bytes, (long long)mm_catalog_workspace_bytes(B, I, k));
  MM_REQUIRE(((uintptr_t)q_split % 16) == 0 && ((uintptr_t)e_split % 16) == 0 && ((uintptr_t)workspace % 16) == 0, MM_ERR_ALIGN,
             "%s: operands / workspace must be 16-B aligned", who);
  if (B == 0) return MM_OK;
  Params p;
  memset(&p, 0, sizeof(p));
  p.M = B;
  p.I = I;
  p.Kp = Kp;
  p.KB = Kp / BLOCK_K;
  p.S = splits_for(B, I);
  p.n_tiles = (int)((I + BN - 1) / BN);
  p.tiles_per_split = (p.n_tiles + p.S - 1) / p.S;
  p.bias = bias;
  p.targets = targets;
  p.id_is64 = id_dtype == MM_I64;
  p.do_lse = out_stats != nullptr;
  p.topk = k;
  p.bias_is_prob = ex.bias_is_prob;
  p.row_ids = ex.row_ids;
  p.col_ids = ex.col_ids;
  p.false_neg_score = ex.false_neg_score;
  p.inv_temp = ex.inv_temp;
  const bool mask = ex.contrastive != 0;
  MM_REQUIRE(!mask || (k == 0 && out_stats && (!ex.row_ids == !ex.col_ids)), MM_ERR_ARG,
             "%s: the contrastive variant computes log-sum-exp statistics only", who);
  const int64_t P = (int64_t)kParts * p.S;
  uint8_t* ws = (uint8_t*)workspace;
  p.ws_lse = (float*)ws;
  p.ws_ids = (long long*)(ws + ((B * P * 3 * (int64_t)sizeof(float) + 15) / 16) * 16);
  p.ws_vals = (float*)((uint8_t*)p.ws_ids + B * P * (int64_t)k * sizeof(long long));
  const size_t a_bytes = 2ull * p.KB * TILE_BYTES, stage_bytes = 2ull * p.KB * TILE_BYTES;
  const size_t fixed = 1024 + a_bytes + 16 * sizeof(uint64_t) + 2 * BN * sizeof(float) + 2 * BN * sizeof(long long);
  int stages = (int)((227 * 1024 - fixed) / stage_bytes);
  if (stages > 4) stages = 4;
  MM_REQUIRE(stages >= 2, MM_ERR_UNSUPPORTED, "%s: tiles do not fit two pipeline stages", who);
  p.stages = stages;
  const size_t smem = 1024 + a_bytes + stages * stage_bytes + (2 * stages + 2) * sizeof(uint64_t) + 2 * BN * sizeof(float) +
                      2 * BN * sizeof(long long);
  CUtensorMap tmA, tmB;
  int rc = make_map(&tmA, q_split, (uint64_t)B, (uint64_t)2 * Kp, BM);
  if (rc) return rc;
  rc = make_map(&tmB, e_split, (uint64_t)I, (uint64_t)2 * Kp, BN);
  if (rc) return rc;
  auto kern = mask ? catalog_kernel<true, false, true>
                   : (k == 0 ? catalog_kernel<true, false, false>
                             : (out_stats ? catalog_kernel<true, true, false> : catalog_kernel<false, true, false>));
  {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      mm::set_error("%s: cudaFuncSetAttribute failed: %s", who, cudaGetErrorString(e));
      return (int)e;
    }
  }
  const long long items = ((B + BM - 1) / BM) * p.S;
  const int sms = mm::sm_count();
  const unsigned grid = (unsigned)(items < sms ? items : sms);
  cudaStream_t st = (cudaStream_t)stream;
  kern<<<grid, kThreads, smem, st>>>(tmA, tmB, p);
  rc = mm::check_launch(who);
  if (rc) return rc;
  long long blocks = (B * 32 + 255) / 256;
  const long long cap = (long long)sms * 16;
  if (blocks > cap) blocks = cap;
  catalog_merge_kernel<<<(unsigned)blocks, 256, 0, st>>>(B, (int)P, p.do_lse, k, p.ws_lse, p.ws_vals, p.ws_ids, out_stats,
                                                        topk_scores, (long long*)topk_ids, ex.extra_logit);
  return mm::check_launch(who);
}

}  // namespace cat
}  // namespace mm

extern "C" {

int mm_catalog_score(const void* q_split, int64_t B, int D, const void* e_split, int64_t I, const float* bias,
                     const void* targets, int id_dtype, float* out_stats, int k, float* topk_scores,
                     int64_t* topk_ids, void* workspace, int64_t workspace_bytes, void* stream) {
  return mm::cat::launch("mm_catalog_score", q_split, B, D, e_split, I, bias, targets, id_dtype, out_stats, k, topk_scores, topk_ids,
                         workspace, workspace_bytes, mm::cat::Extras(), stream);
}

int mm_inbatch_softmax_ce(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                          const void* neg_ids, int id_dtype, int downscore, float false_neg_score, const float* pos_logit,
                          const float* neg_prob, float temperature, float* out_stats, void* workspace,
                          int64_t workspace_bytes, void* stream) {
  MM_REQUIRE(pos_logit && out_stats, MM_ERR_ARG, "mm_inbatch_softmax_ce: pos_logit and out_stats are required");
  MM_REQUIRE(temperature > 0.0f, MM_ERR_ARG, "mm_inbatch_softmax_ce: temperature must be positive");
  MM_REQUIRE(!downscore || (pos_ids && neg_ids), MM_ERR_ARG, "mm_inbatch_softmax_ce: down-scoring needs positive and negative ids");
  mm::cat::Extras ex;
  ex.contrastive = 1;
  ex.bias_is_prob = neg_prob != nullptr;
  if (downscore) {
    ex.row_ids = pos_ids;
    ex.col_ids = neg_ids;
  }
  ex.false_neg_score = false_neg_score;
  ex.inv_temp = 1.0f / temperature;
  ex.extra_logit = pos_logit;
  return mm::cat::launch("mm_inbatch_softmax_ce", q_split, B, D, neg_split, N, neg_prob, nullptr, id_dtype, out_stats, 0, nullptr,
                         nullptr, workspace, workspace_bytes, ex, stream);
}

}  // extern "C"
