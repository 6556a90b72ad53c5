// Tensor-core dense layer for sm_90a: wgmma (bf16 operands, fp32 register accumulators) fed by
// TMA through an mbarrier ring, warp-specialised persistent CTAs.
//
//   out = act(x @ W + bias)            (Keras Dense, merlin/models/tf/blocks/mlp.py:275-280)
//   out = x0 * (x @ W + bias) + x      (DCN-v2 cross, blocks/cross.py:196-198)
//
// fp32 parity on bf16 tensor cores: every fp32 operand is carried as a split-bf16 pair
// x = hi + lo (hi = bf16(x), lo = bf16(x - hi)); passes = 3 accumulates hi*lo + lo*hi + hi*hi
// into ONE fp32 accumulator (relative error ~2^-16: fp32-grade, well inside the 1e-3 logit
// tolerance of the north star); passes = 1 is plain bf16.
//
// Layout in HBM:  a_split (M, 2*Kp) bf16 = [hi(0..Kp) | lo(0..Kp)]      K-major rows
//                 w_split (Np, 2*Kp) bf16 = transpose of the Keras kernel, same split
// Kp = K rounded up to 64 (one 128-byte swizzle row per k-block), Np = N rounded up to 16
// (<= 128) or to 128 (> 128).  Padding is zero, so it contributes nothing.
//
// CTA = 9 warps: warps 0-7 are two consumer warpgroups (wgmma over 64 rows of the 128-row tile
// each, then the epilogue of those rows), warp 8 is the TMA producer.  A pipeline stage holds the
// four 64-wide k-block tiles {A_hi, A_lo, B_hi, B_lo}; the producer refills the ring while the
// consumers run the epilogue.  The epilogue goes through a shared-memory image of the fp32
// accumulator (thread = one row, 32 columns per step), whose 32x32 chunks double as the per-warp
// transpose tiles of the coalesced stores.
#include <cuda.h>
#include <cuda_bf16.h>

#include "mm_common.cuh"
#include "tc_common.cuh"

namespace mm {
namespace tc {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // bf16 elements = 128 bytes = one SWIZZLE_128B row
constexpr int MMA_K = 16;
constexpr int kEpiWarps = 8;              // two consumer warpgroups
constexpr int kThreads = 32 * (kEpiWarps + 1);  // + warp 8: TMA producer
constexpr uint32_t A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB

// row pitch (floats) of the accumulator image: whole 32-column chunks + 4 floats (bank spread)
__host__ __device__ constexpr int image_pitch(int BN) { return ((BN + 31) / 32) * 32 + 4; }

struct Params {
  long long M;
  int N, Np, Kp, BN, n_tiles_n, passes, act, stages;
  // resident-A schedule (scorer with Kp <= 128): a CTA owns a CONTIGUOUS range of tiles (n fastest), keeps the A
  // (query) k-blocks of the current m-tile in shared memory and streams only B (item) tiles through the ring
  int resident_a;
  long long tiles_per_cta;
  const float* bias;
  const float* x0;
  const float* xres;
  long long x_stride;
  float* out_f32;
  long long out_stride;
  __nv_bfloat16* out_split;
  int out_Kp;
  // scorer epilogue (mm_inbatch_scores_tc): logits[m, n] = mask(pos_id[m] == neg_id[n]) ? fns : acc - log(p_n + 1e-16),
  // all divided by `temperature`; `bias` then holds the negative sampling probabilities p_n (or null)
  int score_mode;
  int id_is64;
  const void* pos_ids;
  const void* neg_ids;
  float fns;
  float temperature;
  // fused output head: after this layer's activation, out_head[m] = head_act(sum_n v[m,n] * head_w[n] + head_b)
  // — a following Dense(N -> 1) evaluated in the epilogue on CUDA cores (N <= 32: the row sits in one thread)
  const float* head_w;
  float head_b;
  int head_act;
  float* head_out;
};

// ---------------------------------------------------------------------------------------------
// the GEMM kernel
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1)
dense_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [resident A] [stages][A_hi | A_lo | B_hi | B_lo] (1024-B aligned tiles), accumulator image, barriers
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // pointer arithmetic keeps the shared state space (LDS/STS, not generic LD/ST)
  const uint32_t B_TILE_BYTES = (uint32_t)p.BN * BLOCK_K * 2;
  const int KB_ = p.Kp / BLOCK_K;
  const uint32_t A_RES_BYTES = p.resident_a ? (uint32_t)KB_ * 2 * A_TILE_BYTES : 0u;  // [kb][A_hi | A_lo]
  const uint32_t STAGE_BYTES = p.resident_a ? 2 * B_TILE_BYTES : 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
  const int IP = image_pitch(p.BN);
  uint8_t* a_res = smem;
  smem += A_RES_BYTES;  // the ring starts after the resident A region
  float* img = reinterpret_cast<float*>(smem + (size_t)p.stages * STAGE_BYTES);  // [BLOCK_M][IP] fp32 accumulator
  uint64_t* bars = reinterpret_cast<uint64_t*>(img + (size_t)BLOCK_M * IP);
  uint64_t* full_bar = bars;                       // [stages]
  uint64_t* empty_bar = bars + p.stages;           // [stages] one arrive per consumer warp
  uint64_t* a_full = bars + 2 * p.stages;          // resident A landed (TMA tx)
  uint64_t* a_empty = bars + 2 * p.stages + 1;     // MMAs of the m-row retired (one arrive per consumer warp)
  long long* ids_s = reinterpret_cast<long long*>(bars + 2 * p.stages + 2);               // [256] negative ids of the tile (scorer)
  float* bias_s = reinterpret_cast<float*>(ids_s + 256);                                   // [256] bias of the tile, zero padded

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const long long tiles = m_tiles * p.n_tiles_n;
  const int KB = p.Kp / BLOCK_K;
  // tile sequence of this CTA: interleaved (tile, tile + grid, ...) or, resident-A, a contiguous range
  const long long tile_first = p.resident_a ? (long long)blockIdx.x * p.tiles_per_cta : (long long)blockIdx.x;
  const long long tile_step = p.resident_a ? 1 : (long long)gridDim.x;
  const long long tile_end = p.resident_a ? (tile_first + p.tiles_per_cta < tiles ? tile_first + p.tiles_per_cta : tiles) : tiles;

  if (warp == kEpiWarps && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(full_bar + s), 1);
      mbar_init(smem_u32(empty_bar + s), kEpiWarps);
    }
    mbar_init(smem_u32(a_full), 1);
    mbar_init(smem_u32(a_empty), kEpiWarps);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kEpiWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const uint32_t tx = (p.passes == 3) ? STAGE_BYTES : (A_TILE_BYTES + B_TILE_BYTES);
      int cur_m = -1;
      uint32_t a_loads = 0;
      for (long long tile = tile_first; tile < tile_end; tile += tile_step) {
        const int m0 = (int)(tile / p.n_tiles_n) * BLOCK_M;
        const int n0 = (int)(tile % p.n_tiles_n) * p.BN;
        if (p.resident_a && m0 != cur_m) {  // new m-row: (re)load the query k-blocks once the previous row's MMAs retired
          if (a_loads > 0) mbar_wait(smem_u32(a_empty), (a_loads - 1) & 1);
          const uint32_t ab = smem_u32(a_full);
          mbar_expect_tx(ab, A_RES_BYTES);
          for (int kb = 0; kb < KB; ++kb) {
            tma_load_2d(smem_u32(a_res + (size_t)kb * 2 * A_TILE_BYTES), &tmA, ab, kb * BLOCK_K, m0);
            tma_load_2d(smem_u32(a_res + (size_t)kb * 2 * A_TILE_BYTES + A_TILE_BYTES), &tmA, ab, p.Kp + kb * BLOCK_K, m0);
          }
          cur_m = m0;
          ++a_loads;
        }
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
          const uint32_t fb = smem_u32(full_bar + stage);
          uint8_t* st = smem + (size_t)stage * STAGE_BYTES;
          if (p.resident_a) {  // only the item tiles stream
            mbar_expect_tx(fb, STAGE_BYTES);
            tma_load_2d(smem_u32(st), &tmB, fb, kb * BLOCK_K, n0);
            tma_load_2d(smem_u32(st + B_TILE_BYTES), &tmB, fb, p.Kp + kb * BLOCK_K, n0);
          } else {
            mbar_expect_tx(fb, tx);
            tma_load_2d(smem_u32(st), &tmA, fb, kb * BLOCK_K, m0);
            tma_load_2d(smem_u32(st + 2 * A_TILE_BYTES), &tmB, fb, kb * BLOCK_K, n0);
            if (p.passes == 3) {
              tma_load_2d(smem_u32(st + A_TILE_BYTES), &tmA, fb, p.Kp + kb * BLOCK_K, m0);
              tma_load_2d(smem_u32(st + 2 * A_TILE_BYTES + B_TILE_BYTES), &tmB, fb, p.Kp + kb * BLOCK_K, n0);
            }
          }
          if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups (warps 0..7): MMA, then epilogue =====================
    // warpgroup wg computes accumulator rows 64 wg ..; its warps then finish the 32-row quarters 2 wg, 2 wg + 1
    // from the image: thread = one accumulator row, 32 columns per step, two warps per quarter interleaved over
    // 32-column chunks.  Epilogue: image -> registers -> bias/act/cross -> per-warp shared-memory transpose
    // tile (the chunk's own image region) -> coalesced 16-byte global stores.
    const int wg = warp >> 2;
    const int q = 2 * wg + (warp & 1);  // 32-row quarter of the tile this warp finishes
    const int half = (warp >> 1) & 1;   // which interleaved set of 32-column chunks
    int stage = 0;
    uint32_t phase = 0;
    long long cur_mrow = -1;
    uint32_t a_seen = 0;
    const bool vec_f32 = p.out_f32 && ((p.out_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out_f32) & 15) == 0);
    const bool vec_x = p.x0 && ((p.x_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.x0) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(p.xres) & 15) == 0);
    float col_b = 0.0f, col_h = 0.0f;
    long long col_id = 0;
    uint32_t tile_wide = 0u;  // 1 when a negative id of the current tile needs 64 bits (OR-reduced by the staging barrier)
    auto load_columns = [&](int n0_, float& b, float& h, long long& id) {  // thread i < BN owns column n0_ + i (BN <= 256 threads)
      const int i = (int)threadIdx.x;
      b = 0.0f;
      h = 0.0f;
      id = -0x7fffffffffffffffll;
      if (i < p.BN) {
        const int n = n0_ + i;
        if (p.bias && n < p.N) b = p.score_mode ? -logf(p.bias[n] + 1e-16f) : p.bias[n];
        if (p.head_w && n < p.N) h = p.head_w[n];
        if (p.score_mode && p.neg_ids && n < p.N)
          id = p.id_is64 ? reinterpret_cast<const long long*>(p.neg_ids)[n] : (long long)reinterpret_cast<const int*>(p.neg_ids)[n];
      }
    };
    for (long long tile = tile_first; tile < tile_end; tile += tile_step) {
      const long long m0 = (tile / p.n_tiles_n) * BLOCK_M;
      const int n0 = (int)(tile % p.n_tiles_n) * p.BN;
      const long long row0 = m0 + q * 32;  // first row of this warp
      // per-tile column data: bias (or -log sampling prob), head weights and, for the scorer, the negative ids.
      // The global loads for tile t+1 are issued while tile t is processed (registers), so only shared-memory
      // stores sit between the two barriers — not a global-memory round trip per tile.
      if (tile == tile_first) load_columns(n0, col_b, col_h, col_id);
      named_bar(1, 32 * kEpiWarps);  // previous tile's readers are done
      {
        const int i = (int)threadIdx.x;
        const bool col_hi_flag = p.score_mode && p.neg_ids && i < p.BN && col_id != -0x7fffffffffffffffll &&
                                 ((unsigned long long)col_id >> 32) != 0ull;
        if (i < p.BN) {
          bias_s[i] = col_b;
          if (p.head_w) {
            bias_s[128 + i] = col_h;
            if (i + p.BN < 32) bias_s[128 + i + p.BN] = 0.0f;
          }
          if (p.score_mode && p.neg_ids) {
            uint32_t* lo_s = reinterpret_cast<uint32_t*>(ids_s);
            lo_s[i] = (uint32_t)(unsigned long long)col_id;
            lo_s[256 + i] = (uint32_t)((unsigned long long)col_id >> 32);
          }
        }
        // the barrier that publishes the column data also ORs "some negative id of this tile needs 64 bits"
        asm volatile("{\n .reg .pred p, q;\n setp.ne.u32 q, %1, 0;\n bar.red.or.pred p, 1, %2, q;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(tile_wide)
                     : "r"((uint32_t)col_hi_flag), "n"(32 * kEpiWarps)
                     : "memory");
      }
      if (tile + tile_step < tile_end) load_columns((int)((tile + tile_step) % p.n_tiles_n) * p.BN, col_b, col_h, col_id);
      long long my_pid = 0;
      if (p.score_mode && p.pos_ids && row0 + lane < p.M)
        my_pid = p.id_is64 ? reinterpret_cast<const long long*>(p.pos_ids)[row0 + lane]
                           : (long long)reinterpret_cast<const int*>(p.pos_ids)[row0 + lane];

      // ---- main loop: this warpgroup's 64 x BN accumulator over all k-blocks ----
      if (p.resident_a && tile / p.n_tiles_n != cur_mrow) {
        mbar_wait(smem_u32(a_full), a_seen & 1);
        ++a_seen;
        cur_mrow = tile / p.n_tiles_n;
      }
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
      for (int kb = 0; kb < KB; ++kb) {
        mbar_wait(smem_u32(full_bar + stage), phase);
        const uint32_t st = smem_u32(smem + (size_t)stage * STAGE_BYTES);
        const uint32_t a_hi = (p.resident_a ? smem_u32(a_res + (size_t)kb * 2 * A_TILE_BYTES) : st) + (uint32_t)wg * (A_TILE_BYTES / 2),
                       a_lo = a_hi + A_TILE_BYTES;
        const uint32_t b_hi = p.resident_a ? st : st + 2 * A_TILE_BYTES, b_lo = b_hi + B_TILE_BYTES;
        wgmma_fence_acc(acc);
        wgmma_fence();
        if (p.passes == 3) {
          // small cross terms first, the dominant hi*hi product last
#pragma unroll
          for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss(p.BN, acc, make_desc_sw128(a_hi + k * 32), make_desc_sw128(b_lo + k * 32));
#pragma unroll
          for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss(p.BN, acc, make_desc_sw128(a_lo + k * 32), make_desc_sw128(b_hi + k * 32));
        }
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k) wgmma_ss(p.BN, acc, make_desc_sw128(a_hi + k * 32), make_desc_sw128(b_hi + k * 32));
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_acc(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(empty_bar + stage));  // this warp is done with the stage
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
      if (p.resident_a && (tile + 1 >= tile_end || (tile + 1) / p.n_tiles_n != cur_mrow)) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(a_empty));  // last tile of this m-row: the resident A may be replaced
      }
      // ---- accumulator fragment -> image rows 64 wg .. (the warpgroup's previous epilogue is done with them) ----
      named_bar(2 + wg, 128);
      {
        const int r = 64 * wg + 16 * (warp & 3) + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          if (8 * j < p.BN) {
            *reinterpret_cast<float2*>(img + (size_t)r * IP + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(img + (size_t)(r + 8) * IP + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
        }
      }
      named_bar(2 + wg, 128);

      const int n_chunks = (p.BN + 31) >> 5;
      for (int ch = half; ch < n_chunks; ch += 2) {
        const int c0 = ch << 5;
        const int ncols = min(32, p.BN - c0);  // BN is a multiple of 16
        // this warp's 32 x 32 chunk of the image: read row `lane`, then reuse the chunk as its transpose tile
        float* stg_f = img + (size_t)(q * 32) * IP + c0;
        float v[32];
        {
          const float4* a4 = reinterpret_cast<const float4*>(stg_f + (size_t)lane * IP);
          if (p.bias != nullptr) {  // warp-uniform; bias_s is zero padded, read 4 columns per shared-memory load
            const float4* b4 = reinterpret_cast<const float4*>(bias_s + c0);
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 a = a4[j >> 2], b = b4[j >> 2];
              v[j] = a.x + b.x;
              v[j + 1] = a.y + b.y;
              v[j + 2] = a.z + b.z;
              v[j + 3] = a.w + b.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 a = a4[j >> 2];
              v[j] = a.x;
              v[j + 1] = a.y;
              v[j + 2] = a.z;
              v[j + 3] = a.w;
            }
          }
        }
        if (p.x0) {
          // cross epilogue: x0 * (xW + b) + x ; x0 / x tiles come in through the transpose tile (coalesced)
#pragma unroll 1
          for (int which = 0; which < 2; ++which) {
            const float* src = which == 0 ? p.x0 : p.xres;
            __syncwarp();
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int rr = it * 4 + (lane >> 3), cv = (lane & 7) * 4;
              const long long grow = row0 + rr;
              const int n = n0 + c0 + cv;
              float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
              if (grow < p.M && cv < ncols) {
                const float* g = src + grow * p.x_stride + n;
                if (vec_x && n + 3 < p.N) t = *reinterpret_cast<const float4*>(g);
                else {
                  if (n < p.N) t.x = g[0];
                  if (n + 1 < p.N) t.y = g[1];
                  if (n + 2 < p.N) t.z = g[2];
                  if (n + 3 < p.N) t.w = g[3];
                }
              }
              *reinterpret_cast<float4*>(stg_f + rr * IP + cv) = t;
            }
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 t = *reinterpret_cast<const float4*>(stg_f + lane * IP + j);
              if (which == 0) {
                v[j] = __fmul_rn(t.x, v[j]); v[j + 1] = __fmul_rn(t.y, v[j + 1]);
                v[j + 2] = __fmul_rn(t.z, v[j + 2]); v[j + 3] = __fmul_rn(t.w, v[j + 3]);
              } else {
                v[j] = __fadd_rn(v[j], t.x); v[j + 1] = __fadd_rn(v[j + 1], t.y);
                v[j + 2] = __fadd_rn(v[j + 2], t.z); v[j + 3] = __fadd_rn(v[j + 3], t.w);
              }
            }
          }
        } else if (p.score_mode) {
          // false-negative mask (utils/tf_utils.py:140-150) then LogitsTemperatureScaler (x / T)
          if (p.pos_ids != nullptr) {
            // ids are stored as (low word, high word) arrays; when every high word of the tile's columns and
            // of this warp's rows is zero (ids < 2^32, the common case) the compare is one 32-bit ISETP per
            // logit on 128-bit shared-memory loads, else the exact 64-bit compare
            const uint32_t* lo_s = reinterpret_cast<const uint32_t*>(ids_s);
            const uint32_t* hi_s = lo_s + 256;
            const uint32_t pid_lo = (uint32_t)(unsigned long long)my_pid, pid_hi = (uint32_t)((unsigned long long)my_pid >> 32);
            const bool narrow = (tile_wide == 0u) && !__any_sync(0xffffffffu, pid_hi != 0u);
            if (narrow) {
              const uint4* l4 = reinterpret_cast<const uint4*>(lo_s + c0);
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const uint4 L = l4[j >> 2];
                v[j] = L.x == pid_lo ? p.fns : v[j];
                v[j + 1] = L.y == pid_lo ? p.fns : v[j + 1];
                v[j + 2] = L.z == pid_lo ? p.fns : v[j + 2];
                v[j + 3] = L.w == pid_lo ? p.fns : v[j + 3];
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (lo_s[c0 + j] == pid_lo && hi_s[c0 + j] == pid_hi) v[j] = p.fns;
            }
          }
          if (p.temperature != 1.0f) {  // x / 1 == x exactly: skip the IEEE division in the common case
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = __fdiv_rn(v[j], p.temperature);
          }
        } else if (p.act == MM_ACT_RELU) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.0f);
        } else if (p.act != MM_ACT_LINEAR) {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (n0 + c0 + j < p.N) v[j] = apply_act_slow(v[j], p.act);  // warp-uniform: skip padding columns
        }
        // padding columns (n >= N) must be exact zeros for the next layer's operand
        if (n0 + c0 + 32 > p.N) {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (n0 + c0 + j >= p.N) v[j] = 0.0f;
        }
        if (p.head_w) {  // fused Dense(N -> 1): BN <= 32, so this chunk is the whole row
          float h = p.head_b;
#pragma unroll
          for (int j = 0; j < 32; ++j) h = fmaf(v[j], bias_s[128 + j], h);
          if (row0 + lane < p.M) p.head_out[row0 + lane] = apply_act(h, p.head_act);
        }
        if (p.out_f32) {
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 32; j += 4)
            *reinterpret_cast<float4*>(stg_f + lane * IP + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
          __syncwarp();
          if (vec_f32 && row0 + 32 <= p.M && n0 + c0 + 32 <= p.N) {
            // interior chunk (the common case): no per-element predicates
            const int rsub = lane >> 3, cv = (lane & 7) * 4;
            float* g = p.out_f32 + (row0 + rsub) * p.out_stride + (n0 + c0 + cv);
            const float* src = stg_f + rsub * IP + cv;
#pragma unroll
            for (int it = 0; it < 8; ++it)
              *reinterpret_cast<float4*>(g + (long long)it * 4 * p.out_stride) = *reinterpret_cast<const float4*>(src + it * 4 * IP);
          } else if (vec_f32) {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int rr = it * 4 + (lane >> 3), cv = (lane & 7) * 4;
              const long long grow = row0 + rr;
              const int n = n0 + c0 + cv;
              if (grow < p.M && cv < ncols && n < p.N) {
                const float4 t = *reinterpret_cast<const float4*>(stg_f + rr * IP + cv);
                float* g = p.out_f32 + grow * p.out_stride + n;
                if (n + 3 < p.N) *reinterpret_cast<float4*>(g) = t;
                else {
                  g[0] = t.x;
                  if (n + 1 < p.N) g[1] = t.y;
                  if (n + 2 < p.N) g[2] = t.z;
                }
              }
            }
          } else {
            // rows only 4-byte aligned (e.g. the (B, 1+N) logits at column 1): a warp store covers 32
            // consecutive floats of one row
            const int n = n0 + c0 + lane;
            if (lane < ncols && n < p.N) {
              const int rmax = (int)min((long long)32, p.M - row0);
              for (int rr = 0; rr < rmax; ++rr) p.out_f32[(row0 + rr) * p.out_stride + n] = stg_f[rr * IP + lane];
            }
          }
        }
        if (p.out_split && n0 + c0 < p.out_Kp) {
          // [hi | lo] bf16 rows of the next layer's A operand: hi in the first 64 B of each tile row, lo in the next
          __syncwarp();
          uint8_t* th = reinterpret_cast<uint8_t*>(stg_f);
          uint8_t* tl = th + 64;
          const int pitch = IP * 4;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            __align__(16) __nv_bfloat16 h[8], l[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) split_bf16(v[j + e], h[e], l[e]);
            *reinterpret_cast<uint4*>(th + lane * pitch + j * 2) = *reinterpret_cast<const uint4*>(h);
            *reinterpret_cast<uint4*>(tl + lane * pitch + j * 2) = *reinterpret_cast<const uint4*>(l);
          }
          __syncwarp();
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int rr = it * 8 + (lane >> 2), cv = (lane & 3) * 8;  // 8 bf16 = 16 B per lane
            const long long grow = row0 + rr;
            if (grow < p.M && cv < ncols && n0 + c0 + cv < p.out_Kp) {
              __nv_bfloat16* oh = p.out_split + grow * (2ll * p.out_Kp) + n0 + c0 + cv;
              *reinterpret_cast<uint4*>(oh) = *reinterpret_cast<const uint4*>(th + rr * pitch + cv * 2);
              *reinterpret_cast<uint4*>(oh + p.out_Kp) = *reinterpret_cast<const uint4*>(tl + rr * pitch + cv * 2);
            }
          }
        }
      }
    }
  }
}

// fp32 rows -> split-bf16 rows [hi | lo], zero padded to Kp
__global__ void split_rows_kernel(const float* __restrict__ x, long long M, int K, long long x_stride,
                                  __nv_bfloat16* __restrict__ out, int Kp) {
  const long long total = M * (Kp / 8);
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long m = e / (Kp / 8);
    const int k0 = (int)(e % (Kp / 8)) * 8;
    __align__(16) __nv_bfloat16 h[8], l[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = (k0 + j < K) ? x[m * x_stride + k0 + j] : 0.0f;
      split_bf16(v, h[j], l[j]);
    }
    __nv_bfloat16* o = out + m * (2ll * Kp) + k0;
    *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(h);
    *reinterpret_cast<uint4*>(o + Kp) = *reinterpret_cast<const uint4*>(l);
  }
}

// Keras kernel (K, N) fp32 -> (Np, 2*Kp) bf16, transposed (K-major), split, zero padded
__global__ void split_weights_kernel(const float* __restrict__ W, int K, int N, __nv_bfloat16* __restrict__ out,
                                     int Kp, int Np) {
  const long long total = (long long)Np * Kp;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(e / Kp), k = (int)(e % Kp);
    const float v = (n < N && k < K) ? W[(long long)k * N + n] : 0.0f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    out[(long long)n * 2 * Kp + k] = h;
    out[(long long)n * 2 * Kp + Kp + k] = l;
  }
}

}  // namespace tc
}  // namespace mm

extern "C" {

int mm_tc_padded_k(int K) { return ((K + 63) / 64) * 64; }
int mm_tc_padded_n(int N) { return N <= 128 ? ((N + 15) / 16) * 16 : ((N + 127) / 128) * 128; }

int mm_split_rows(const float* x, int64_t M, int K, int64_t x_stride, void* out_split, int Kp, void* stream) {
  MM_REQUIRE(x && out_split && M >= 0 && K > 0 && x_stride >= K, MM_ERR_ARG, "mm_split_rows: null pointer or bad K/stride");
  MM_REQUIRE(Kp >= K && Kp % 64 == 0, MM_ERR_ARG, "mm_split_rows: Kp must be a multiple of 64 and >= K");
  MM_REQUIRE(((uintptr_t)out_split % 16) == 0, MM_ERR_ALIGN, "mm_split_rows: out_split must be 16-B aligned");
  if (M == 0) return MM_OK;
  const long long total = M * (Kp / 8);
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)mm::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  mm::tc::split_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, M, K, x_stride,
                                                                               (__nv_bfloat16*)out_split, Kp);
  return mm::check_launch("mm_split_rows");
}

int mm_split_weights(const float* W, int K, int N, void* w_split, int Kp, int Np, void* stream) {
  MM_REQUIRE(W && w_split && K > 0 && N > 0, MM_ERR_ARG, "mm_split_weights: null pointer or non-positive K/N");
  MM_REQUIRE(Kp == mm_tc_padded_k(K) && Np == mm_tc_padded_n(N), MM_ERR_ARG,
             "mm_split_weights: Kp/Np must be mm_tc_padded_k(K)=%d / mm_tc_padded_n(N)=%d", mm_tc_padded_k(K),
             mm_tc_padded_n(N));
  const long long total = (long long)Np * Kp;
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)mm::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  mm::tc::split_weights_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(W, K, N, (__nv_bfloat16*)w_split, Kp, Np);
  return mm::check_launch("mm_split_weights");
}

static int dense_tc_launch(const void* a_split, int64_t M, int K, int Kp, const void* w_split, int N, int Np,
                           const float* bias, int act, int passes, const float* x0, const float* xres,
                           int64_t x_stride, float* out_f32, int64_t out_stride, void* out_split, int out_Kp,
                           int score_mode, const void* pos_ids, const void* neg_ids, int id_is64, float fns,
                           float temperature, int64_t b_rows, const float* head_w, float head_b, int head_act,
                           float* head_out, void* stream) {
  using namespace mm::tc;
  MM_REQUIRE(a_split && w_split && M >= 0 && K > 0 && N > 0, MM_ERR_ARG, "mm_dense_tc: null operand or non-positive K/N");
  MM_REQUIRE(Kp == mm_tc_padded_k(K) && Np == mm_tc_padded_n(N), MM_ERR_ARG,
             "mm_dense_tc: Kp/Np must be the padded sizes (%d / %d)", mm_tc_padded_k(K), mm_tc_padded_n(N));
  MM_REQUIRE(passes == 1 || passes == 3, MM_ERR_ARG, "mm_dense_tc: passes must be 1 (bf16) or 3 (split-bf16)");
  MM_REQUIRE(act >= MM_ACT_LINEAR && act <= MM_ACT_GELU, MM_ERR_ARG, "mm_dense_tc: unknown activation %d", act);
  MM_REQUIRE((x0 == nullptr) == (xres == nullptr), MM_ERR_ARG, "mm_dense_tc: x0 and xres go together");
  MM_REQUIRE(!score_mode || (!x0 && !out_split), MM_ERR_ARG, "mm_dense_tc: scorer epilogue excludes cross / split outputs");
  MM_REQUIRE(!x0 || x_stride >= N, MM_ERR_ARG, "mm_dense_tc: x_stride < N for the cross epilogue");
  MM_REQUIRE(out_f32 || out_split || head_out, MM_ERR_ARG, "mm_dense_tc: no output requested");
  MM_REQUIRE((head_w == nullptr) == (head_out == nullptr), MM_ERR_ARG, "mm_dense_tc: head weights and head output go together");
  MM_REQUIRE(!head_w || (Np <= 32 && !score_mode && !x0), MM_ERR_UNSUPPORTED,
             "mm_dense_tc: the fused Dense(N->1) head needs N <= 32 and a plain dense epilogue");
  MM_REQUIRE(!head_w || (head_act >= MM_ACT_LINEAR && head_act <= MM_ACT_GELU), MM_ERR_ARG, "mm_dense_tc: unknown head activation");
  MM_REQUIRE(!out_f32 || out_stride >= N, MM_ERR_ARG, "mm_dense_tc: out_stride < N");
  MM_REQUIRE(!out_split || (out_Kp == mm_tc_padded_k(N) && ((uintptr_t)out_split % 16) == 0), MM_ERR_ARG,
             "mm_dense_tc: out_Kp must be mm_tc_padded_k(N)=%d and out_split 16-B aligned", mm_tc_padded_k(N));
  MM_REQUIRE(((uintptr_t)a_split % 16) == 0 && ((uintptr_t)w_split % 16) == 0, MM_ERR_ALIGN,
             "mm_dense_tc: operands must be 16-B aligned");
  MM_REQUIRE(M < (1ll << 31), MM_ERR_UNSUPPORTED, "mm_dense_tc: M too large for 32-bit TMA coordinates");
  if (M == 0) return MM_OK;

  Params p;
  p.M = M;
  p.N = N;
  p.Np = Np;
  p.Kp = Kp;
  p.BN = Np <= 128 ? Np : 128;
  p.n_tiles_n = Np / p.BN;
  p.passes = passes;
  p.act = act;
  p.bias = bias;
  p.x0 = x0;
  p.xres = xres;
  p.x_stride = x_stride;
  p.out_f32 = out_f32;
  p.out_stride = out_stride;
  p.out_split = (__nv_bfloat16*)out_split;
  p.out_Kp = out_Kp;
  p.score_mode = score_mode;
  p.id_is64 = id_is64;
  p.pos_ids = pos_ids;
  p.neg_ids = neg_ids;
  p.fns = fns;
  p.temperature = temperature;
  p.head_w = head_w;
  p.head_b = head_b;
  p.head_act = head_act;
  p.head_out = head_out;
  // resident-A schedule: many n-tiles per m-tile and a short K (the in-batch scorer): operand traffic halves
  p.resident_a = (score_mode && passes == 3 && Kp <= 2 * BLOCK_K && p.n_tiles_n >= 8) ? 1 : 0;
  const size_t a_res_bytes = p.resident_a ? (size_t)(Kp / BLOCK_K) * 2 * A_TILE_BYTES : 0;
  const size_t stage_bytes = (p.resident_a ? 0 : 2 * (size_t)A_TILE_BYTES) + 2 * (size_t)p.BN * BLOCK_K * 2;
  const size_t epi_bytes = 256 * sizeof(long long) + 256 * sizeof(float);
  const size_t image_bytes = (size_t)BLOCK_M * image_pitch(p.BN) * sizeof(float);
  const size_t fixed = 1024 + a_res_bytes + image_bytes + 16 * sizeof(uint64_t) + epi_bytes;
  int stages = (int)((227 * 1024 - fixed) / stage_bytes);
  if (stages > 6) stages = 6;
  if (!p.resident_a && stages > Kp / BLOCK_K * 2) stages = Kp / BLOCK_K * 2 > 2 ? Kp / BLOCK_K * 2 : 2;
  MM_REQUIRE(stages >= 2, MM_ERR_UNSUPPORTED, "mm_dense_tc: tile does not fit two pipeline stages");
  p.stages = stages;
  const size_t smem = 1024 + a_res_bytes + stages * stage_bytes + image_bytes + (2 * stages + 2) * sizeof(uint64_t) + epi_bytes;

  CUtensorMap tmA, tmB;
  int rc = make_map(&tmA, a_split, (uint64_t)M, (uint64_t)2 * Kp, BLOCK_M);
  if (rc) return rc;
  rc = make_map(&tmB, w_split, (uint64_t)b_rows, (uint64_t)2 * Kp, (uint32_t)p.BN);  // rows past b_rows read as zeros
  if (rc) return rc;

  static size_t smem_set = 0;  // raise the dynamic-smem limit once (monotone), not per launch
  if (smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(dense_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      mm::set_error("mm_dense_tc: cudaFuncSetAttribute(227 KB smem) failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
    smem_set = 227 * 1024;
  }
  const long long tiles = ((M + BLOCK_M - 1) / BLOCK_M) * p.n_tiles_n;
  const int sms = mm::sm_count();
  unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
  p.tiles_per_cta = (tiles + grid - 1) / grid;
  if (p.resident_a) grid = (unsigned)((tiles + p.tiles_per_cta - 1) / p.tiles_per_cta);  // no empty CTAs
  dense_tc_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(tmA, tmB, p);
  return mm::check_launch("mm_dense_tc");
}

int mm_dense_tc(const void* a_split, int64_t M, int K, int Kp, const void* w_split, int N, int Np,
                const float* bias, int act, int passes, const float* x0, const float* xres,
                int64_t x_stride, float* out_f32, int64_t out_stride, void* out_split, int out_Kp,
                void* stream) {
  return dense_tc_launch(a_split, M, K, Kp, w_split, N, Np, bias, act, passes, x0, xres, x_stride, out_f32, out_stride,
                         out_split, out_Kp, 0, nullptr, nullptr, 0, 0.0f, 1.0f, Np, nullptr, 0.0f, 0, nullptr, stream);
}

int mm_dense_tc_head(const void* a_split, int64_t M, int K, int Kp, const void* w_split, int N, int Np,
                     const float* bias, int act, int passes, const float* head_w, float head_b, int head_act,
                     float* head_out, void* stream) {
  return dense_tc_launch(a_split, M, K, Kp, w_split, N, Np, bias, act, passes, nullptr, nullptr, 0, nullptr, 0, nullptr, 0, 0,
                         nullptr, nullptr, 0, 0.0f, 1.0f, Np, head_w, head_b, head_act, head_out, stream);
}

int mm_inbatch_scores_tc(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D,
                         const void* pos_ids, const void* neg_ids, int id_dtype, int downscore,
                         float false_neg_score, const float* neg_prob, float temperature, float* out,
                         int64_t out_stride, void* stream) {
  MM_REQUIRE(q_split && neg_split && out && B >= 0 && N > 0 && D > 0, MM_ERR_ARG, "mm_inbatch_scores_tc: null pointer or bad size");
  MM_REQUIRE(N < (1ll << 31) && out_stride >= N + 1, MM_ERR_ARG, "mm_inbatch_scores_tc: N too large or out_stride < 1+N");
  MM_REQUIRE(!downscore || (pos_ids && neg_ids), MM_ERR_ARG, "mm_inbatch_scores_tc: downscore needs positive and negative ids");
  MM_REQUIRE(id_dtype == MM_I32 || id_dtype == MM_I64, MM_ERR_ARG, "mm_inbatch_scores_tc: bad id dtype");
  MM_REQUIRE(temperature != 0.0f, MM_ERR_ARG, "mm_inbatch_scores_tc: temperature must be non-zero");
  // negatives play the role of the weight matrix: (N, D) K-major rows; columns 1.. of `out`
  return dense_tc_launch(q_split, B, D, mm_tc_padded_k(D), neg_split, (int)N, mm_tc_padded_n((int)N), neg_prob,
                         MM_ACT_LINEAR, 3, nullptr, nullptr, 0, out + 1, out_stride, nullptr, 0, 1,
                         downscore ? pos_ids : nullptr, downscore ? neg_ids : nullptr, id_dtype == MM_I64,
                         false_neg_score, temperature, N, nullptr, 0.0f, 0, nullptr, stream);
}


}  // extern "C"
