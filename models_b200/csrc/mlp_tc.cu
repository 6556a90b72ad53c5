// Whole-tower MLP for sm_90a: the first Dense layer is a TMA-fed wgmma GEMM (as dense_tc.cu); every
// following layer whose width is <= 128 runs ON CHIP — its activations never leave the registers:
//
//   D1 (registers, fp32)  --bias + act, split-bf16-->  A2 (registers: the wgmma A fragment, packed bf16 hi | lo)
//   A2 x W2 (weights resident in shared memory, SWIZZLE_128B K-major)  --wgmma, A from registers-->  D2
//   D2 --bias + act, split--> A3 --x W3--> D3 ... --> last layer: fp32 rows to HBM and/or the fused
//   Dense(N -> 1) output head (BinaryOutput: sigmoid(x.w + b)).
//
// Replaces the layer-by-layer MLPBlock of the reference (merlin/models/tf/blocks/mlp.py:97-139: a
// SequentialBlock of Keras Dense layers, `_Dense.call` :275-280) + BinaryOutput's Dense(1)
// (outputs/classification.py:114) for the README towers (bottom 13 -> 128 -> 64, top 415 -> 128 -> 64 -> 32 -> 1):
// one launch instead of one per layer, and the (B, 128) / (B, 64) intermediate activations (33 + 17 MB of
// split-bf16 rows written and re-read per step at B = 65 536) never reach HBM.
//
// fp32 parity: all operands are split-bf16 pairs (x = hi + lo), every layer accumulates
// hi*lo + lo*hi + hi*hi into one fp32 accumulator (same arithmetic as mm_dense_tc, passes = 3).
//
// CTA = 9 warps, persistent over 128-row tiles: warps 0-7 are two consumer warpgroups (64 rows of the
// tile each: layer-1 MMAs, every epilogue and every chain MMA of those rows), warp 8 is the TMA producer
// (layer-1 operands; the chain weights once).  The accumulator fragment of a layer maps register for
// register onto the A fragment of the next layer's MMA (columns 16 s .. 16 s + 15 of D are k-step s of A).
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstring>

#include "mm_common.cuh"
#include "tc_common.cuh"

namespace mm {
namespace mlp {

using namespace mm::tc;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int MMA_K = 16;
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * (kConsumerWarps + 1);
constexpr int kMaxChain = 3;
constexpr uint32_t A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB

struct ChainLayer {
  int N, Np;        // true / padded (multiple of 16) width of this layer
  int Kp;           // K padded to 64 (row pitch of the split weights = 2 * Kp elements)
  int ksteps;       // MMA k-steps actually issued = padded width of the previous layer / 16
  int act;
  uint32_t w_off;   // byte offset of this layer's resident weight tiles inside the weight arena
};

struct Params {
  long long M;
  int K1p, N1, N1p, act1, stages, n_chain;
  ChainLayer c[kMaxChain];
  const float* bias[kMaxChain + 1];  // layer 1, chain layers
  uint32_t w_bytes;                  // total resident weight bytes
  float* out_f32;                    // (M, N_last) fp32 rows, or null
  uint8_t* out_operand;              // (M, 2*N_last) bf16 split rows [hi | lo], or null
  long long out_stride;
  const float* head_w;               // fused Dense(N_last -> 1) head, or null
  float head_b;
  int head_act;
  float* head_out;
};

__device__ __forceinline__ void split_pair(float x, float y, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(x, y);  // .x (low half) = x: K element 2c in the low 16 bits
  hi = *reinterpret_cast<uint32_t*>(&h);
  const float xh = __uint_as_float(hi << 16), yh = __uint_as_float(hi & 0xffff0000u);
  __nv_bfloat162 l = __floats2bfloat162_rn(x - xh, y - yh);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

__global__ void __launch_bounds__(kThreads, 1)
mlp_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW1,
              const __grid_constant__ CUtensorMap tmC0, const __grid_constant__ CUtensorMap tmC1,
              const __grid_constant__ CUtensorMap tmC2, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // keeps the shared state space
  // layer-1 ring: each slot holds ONE half of a k-block, {A_hi, W1_hi} or {A_lo, W1_lo} (32 KB at N1 = 128):
  // finer slots keep more bytes in flight than whole {hi, lo} stages in the same shared memory
  const uint32_t B_TILE_BYTES = (uint32_t)p.N1p * BLOCK_K * 2;
  const uint32_t STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
  uint8_t* wres = smem + (size_t)p.stages * STAGE_BYTES;  // resident chain weights (1024-B aligned tiles)
  uint64_t* bars = reinterpret_cast<uint64_t*>(wres + p.w_bytes);
  uint64_t* full_bar = bars;                        // [stages]
  uint64_t* empty_bar = bars + p.stages;            // [stages] one arrive per consumer warp
  uint64_t* w_full = bars + 2 * p.stages;           // resident weights landed
  float* bias_s = reinterpret_cast<float*>(bars + 2 * p.stages + 2);  // [kMaxChain + 1][128], zero padded
  float* head_s = bias_s + (kMaxChain + 1) * 128;                     // [128], zero padded

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int KB = p.K1p / BLOCK_K;

  if (warp == kConsumerWarps && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW1) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(full_bar + s), 1);
      mbar_init(smem_u32(empty_bar + s), kConsumerWarps);
    }
    mbar_init(smem_u32(w_full), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // biases / head weights are the same for every tile (each layer is a single n-tile): stage them once
  for (int i = threadIdx.x; i < (kMaxChain + 1) * 128; i += kThreads) {
    const int l = i >> 7, n = i & 127;
    const int N = l == 0 ? p.N1 : (l <= p.n_chain ? p.c[l - 1].N : 0);
    bias_s[i] = (p.bias[l] != nullptr && n < N) ? p.bias[l][n] : 0.0f;
  }
  if (threadIdx.x < 128) {
    const int Nl = p.n_chain ? p.c[p.n_chain - 1].N : p.N1;
    head_s[threadIdx.x] = (p.head_w != nullptr && (int)threadIdx.x < Nl) ? p.head_w[threadIdx.x] : 0.0f;
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      if (p.n_chain > 0) {  // chain weights: loaded once, resident for the whole kernel
        const uint32_t wb = smem_u32(w_full);
        mbar_expect_tx(wb, p.w_bytes);
        for (int c = 0; c < p.n_chain; ++c) {
          const CUtensorMap* tm = c == 0 ? &tmC0 : (c == 1 ? &tmC1 : &tmC2);
          const uint32_t tile_b = (uint32_t)p.c[c].Np * BLOCK_K * 2;
          const int kbs = p.c[c].Kp / BLOCK_K;
          for (int kb = 0; kb < kbs; ++kb) {
            tma_load_2d(smem_u32(wres + p.c[c].w_off + (size_t)kb * tile_b), tm, wb, kb * BLOCK_K, 0);                     // hi
            tma_load_2d(smem_u32(wres + p.c[c].w_off + (size_t)(kbs + kb) * tile_b), tm, wb, p.c[c].Kp + kb * BLOCK_K, 0);  // lo
          }
        }
      }
      int stage = 0;
      uint32_t phase = 0;
      for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m0 = (int)tile * BLOCK_M;
        for (int kb2 = 0; kb2 < 2 * KB; ++kb2) {  // slot order: hi(0), lo(0), hi(1), lo(1), ...
          const int kb = kb2 >> 1, col = (kb2 & 1) * p.K1p + kb * BLOCK_K;
          mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
          const uint32_t fb = smem_u32(full_bar + stage);
          uint8_t* st = smem + (size_t)stage * STAGE_BYTES;
          mbar_expect_tx(fb, STAGE_BYTES);
          tma_load_2d(smem_u32(st), &tmA, fb, col, m0);
          tma_load_2d(smem_u32(st + A_TILE_BYTES), &tmW1, fb, col, 0);
          if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups: 64 rows each, every layer =====================
    const int wg = warp >> 2;
    const int c2 = 2 * (lane & 3);  // fragment column offset inside an 8-column block
    const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // tile row of fragment row 0 (row 1 is 8 further)
    const uint32_t a_off = (uint32_t)wg * (A_TILE_BYTES / 2);
    int stage = 0;
    uint32_t phase = 0;
    bool weights_ready = p.n_chain == 0;
    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
      for (int kb = 0; kb < KB; ++kb) {
        // hi slot: the dominant hi*hi product starts as soon as it lands
        const int s_hi = stage;
        mbar_wait(smem_u32(full_bar + s_hi), phase);
        const uint32_t a_hi = smem_u32(smem + (size_t)s_hi * STAGE_BYTES), b_hi = a_hi + A_TILE_BYTES;
        wgmma_fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k)
          wgmma_ss(p.N1p, acc, make_desc_sw128(a_hi + a_off + k * 32), make_desc_sw128(b_hi + k * 32));
        wgmma_commit();
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
        // lo slot: the two cross terms
        const int s_lo = stage;
        mbar_wait(smem_u32(full_bar + s_lo), phase);
        const uint32_t a_lo = smem_u32(smem + (size_t)s_lo * STAGE_BYTES), b_lo = a_lo + A_TILE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k)
          wgmma_ss(p.N1p, acc, make_desc_sw128(a_hi + a_off + k * 32), make_desc_sw128(b_lo + k * 32));
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k)
          wgmma_ss(p.N1p, acc, make_desc_sw128(a_lo + a_off + k * 32), make_desc_sw128(b_hi + k * 32));
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_acc(acc);
        __syncwarp();
        if (lane == 0) {  // both slots are free once this warp's MMAs have completed
          mbar_arrive(smem_u32(empty_bar + s_hi));
          mbar_arrive(smem_u32(empty_bar + s_lo));
        }
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }

      for (int layer = 0; layer <= p.n_chain; ++layer) {
        const bool last = layer == p.n_chain;
        const int N = layer == 0 ? p.N1 : p.c[layer - 1].N;
        const int Np = layer == 0 ? p.N1p : p.c[layer - 1].Np;
        const int act = layer == 0 ? p.act1 : p.c[layer - 1].act;
        const float* bs = bias_s + layer * 128;
        // bias + activation on the fragment; padding columns (>= N) become exact zeros
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          if (8 * j < Np) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int col = 8 * j + c2 + (e & 1);
              float v = acc[4 * j + e] + bs[col];
              if (act == MM_ACT_RELU) v = fmaxf(v, 0.0f);
              else if (act != MM_ACT_LINEAR && col < N) v = apply_act_slow(v, act);
              acc[4 * j + e] = col < N ? v : 0.0f;
            }
          }
        }
        if (!last) {
          // next layer's A fragment: k-step s = columns 16 s .. 16 s + 15 = n8 blocks 2 s, 2 s + 1
          uint32_t ahi[32], alo[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) split_pair(acc[2 * i], acc[2 * i + 1], ahi[i], alo[i]);
          const ChainLayer& L = p.c[layer];
          if (!weights_ready) {
            mbar_wait(smem_u32(w_full), 0);
            weights_ready = true;
          }
          const uint32_t tile_b = (uint32_t)L.Np * BLOCK_K * 2;
          const uint32_t w_hi = smem_u32(wres + L.w_off), w_lo = w_hi + (uint32_t)(L.Kp / BLOCK_K) * tile_b;
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
          wgmma_fence_acc(acc);
          wgmma_fence();
          // a k-step covers 16 K elements = 32 bytes of a weight row
#pragma unroll
          for (int ks = 0; ks < 8; ++ks) {
            if (ks < L.ksteps) {
              const uint32_t f[4] = {ahi[4 * ks], ahi[4 * ks + 1], ahi[4 * ks + 2], ahi[4 * ks + 3]};
              wgmma_rs(L.Np, acc, f, make_desc_sw128(w_lo + (ks >> 2) * tile_b + (ks & 3) * 32));
            }
          }
#pragma unroll
          for (int ks = 0; ks < 8; ++ks) {
            if (ks < L.ksteps) {
              const uint32_t f[4] = {alo[4 * ks], alo[4 * ks + 1], alo[4 * ks + 2], alo[4 * ks + 3]};
              wgmma_rs(L.Np, acc, f, make_desc_sw128(w_hi + (ks >> 2) * tile_b + (ks & 3) * 32));
            }
          }
#pragma unroll
          for (int ks = 0; ks < 8; ++ks) {
            if (ks < L.ksteps) {
              const uint32_t f[4] = {ahi[4 * ks], ahi[4 * ks + 1], ahi[4 * ks + 2], ahi[4 * ks + 3]};
              wgmma_rs(L.Np, acc, f, make_desc_sw128(w_hi + (ks >> 2) * tile_b + (ks & 3) * 32));
            }
          }
          wgmma_commit();
          wgmma_wait_all();
          wgmma_fence_acc(acc);
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const long long row = tile * BLOCK_M + frow + 8 * h;
            if (p.head_w) {  // fused Dense(N -> 1): Np <= 32; the four lanes of a quad hold a row's columns
              float hsum = 0.0f;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                hsum = fmaf(acc[4 * j + 2 * h], head_s[8 * j + c2], hsum);
                hsum = fmaf(acc[4 * j + 2 * h + 1], head_s[8 * j + c2 + 1], hsum);
              }
              hsum += __shfl_xor_sync(0xffffffffu, hsum, 1);
              hsum += __shfl_xor_sync(0xffffffffu, hsum, 2);
              if ((lane & 3) == 0 && row < p.M) p.head_out[row] = apply_act(hsum + p.head_b, p.head_act);
            }
            if (row < p.M && (p.out_f32 || p.out_operand)) {
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const int n = 8 * j + c2;
                if (8 * j < Np && n < N) {
                  const float x = acc[4 * j + 2 * h], y = acc[4 * j + 2 * h + 1];
                  if (p.out_operand) {  // N % 4 == 0: the pair (n, n + 1) is whole
                    uint32_t hi, lo;
                    split_pair(x, y, hi, lo);
                    uint8_t* rowp = p.out_operand + row * ((long long)N * 4);
                    *reinterpret_cast<uint32_t*>(rowp + n * 2) = hi;
                    *reinterpret_cast<uint32_t*>(rowp + N * 2 + n * 2) = lo;
                  }
                  if (p.out_f32) {
                    float* g = p.out_f32 + row * p.out_stride + n;
                    g[0] = x;
                    if (n + 1 < N) g[1] = y;
                  }
                }
              }
            }
          }
        }
      }
    }
  }
}

}  // namespace mlp
}  // namespace mm

// Fills the shape-dependent part of Params and the shared-memory size; false when the tower does not fit.
static bool plan_tower(int K, int n_layers, const int* widths, mm::mlp::Params& p, size_t& smem) {
  using namespace mm::mlp;
  memset(&p, 0, sizeof(p));
  p.K1p = mm_tc_padded_k(K);
  p.N1 = widths[0];
  p.N1p = mm_tc_padded_n(widths[0]);
  p.n_chain = n_layers - 1;
  uint32_t w_off = 0;
  int prev_np = p.N1p, prev_n = p.N1;
  for (int c = 0; c < p.n_chain; ++c) {
    ChainLayer& L = p.c[c];
    L.N = widths[c + 1];
    L.Np = mm_tc_padded_n(L.N);
    L.Kp = mm_tc_padded_k(prev_n);
    L.ksteps = prev_np / MMA_K;
    L.w_off = w_off;
    w_off += (uint32_t)(2 * (L.Kp / BLOCK_K)) * (uint32_t)L.Np * BLOCK_K * 2;
    prev_np = L.Np;
    prev_n = L.N;
  }
  p.w_bytes = w_off;
  // ring slot = one half ({A_hi, W_hi} or {A_lo, W_lo}) of a k-block
  const size_t stage_bytes = (size_t)A_TILE_BYTES + (size_t)p.N1p * BLOCK_K * 2;
  const size_t fixed = 1024 + (size_t)p.w_bytes + 40 * sizeof(uint64_t) + ((kMaxChain + 1) * 128 + 128) * sizeof(float);
  if (fixed + 4 * stage_bytes > 227 * 1024) return false;
  int stages = (int)((227 * 1024 - fixed) / stage_bytes);
  if (stages > 12) stages = 12;
  const int kb1 = p.K1p / BLOCK_K;
  if (stages > 4 * kb1) stages = 4 * kb1 > 4 ? 4 * kb1 : 4;
  p.stages = stages;
  smem = 1024 + stages * stage_bytes + p.w_bytes + (2 * stages + 2) * sizeof(uint64_t) +
         ((kMaxChain + 1) * 128 + 128) * sizeof(float);
  return true;
}

extern "C" {

int mm_mlp_tc_supported(int K, int n_layers, const int* widths, int with_head) {
  if (K <= 0 || !widths || n_layers < 2 || n_layers > mm::mlp::kMaxChain + 1) return 0;
  for (int l = 0; l < n_layers; ++l)
    if (widths[l] < 1 || widths[l] > 128) return 0;
  if (with_head && widths[n_layers - 1] > 32) return 0;
  mm::mlp::Params p;
  size_t smem = 0;
  return plan_tower(K, n_layers, widths, p, smem) ? 1 : 0;
}

}  // extern "C"

static int mlp_tc_impl(const void* a_split, int64_t M, int K, int n_layers, const void* const* w_split, const int* widths,
                       const float* const* bias, const int* acts, float* out, int64_t out_stride, const float* head_w,
                       float head_b, int head_act, float* head_out, void* out_operand, void* stream) {
  using namespace mm::mlp;
  MM_REQUIRE(a_split && w_split && widths && bias && acts && M >= 0 && K > 0, MM_ERR_ARG, "mm_mlp_tc: null pointer or bad M/K");
  MM_REQUIRE(n_layers >= 1 && n_layers <= kMaxChain + 1, MM_ERR_UNSUPPORTED, "mm_mlp_tc: 1..%d layers (got %d)", kMaxChain + 1,
             n_layers);
  MM_REQUIRE(out || head_out || out_operand, MM_ERR_ARG, "mm_mlp_tc: no output requested");
  MM_REQUIRE(!out_operand || (widths[n_layers - 1] % 4 == 0 && ((uintptr_t)out_operand % 16) == 0 &&
                              (!out || ((out_stride & 3) == 0 && ((uintptr_t)out % 16) == 0))),
             MM_ERR_ALIGN, "mm_mlp_tc: operand-format output needs a last width that is a multiple of 4 and 16-B aligned outputs");
  MM_REQUIRE((head_w == nullptr) == (head_out == nullptr), MM_ERR_ARG, "mm_mlp_tc: head weights and head output go together");
  MM_REQUIRE(((uintptr_t)a_split % 16) == 0, MM_ERR_ALIGN, "mm_mlp_tc: a_split must be 16-B aligned");
  MM_REQUIRE(M < (1ll << 31), MM_ERR_UNSUPPORTED, "mm_mlp_tc: M too large for 32-bit TMA coordinates");
  for (int l = 0; l < n_layers; ++l) {
    MM_REQUIRE(w_split[l] && ((uintptr_t)w_split[l] % 16) == 0, MM_ERR_ARG, "mm_mlp_tc: layer %d weights null or misaligned", l);
    MM_REQUIRE(widths[l] >= 1 && widths[l] <= 128, MM_ERR_UNSUPPORTED, "mm_mlp_tc: layer %d width %d is not in 1..128", l,
               widths[l]);
    MM_REQUIRE(acts[l] >= MM_ACT_LINEAR && acts[l] <= MM_ACT_GELU, MM_ERR_ARG, "mm_mlp_tc: unknown activation %d", acts[l]);
  }
  const int n_last = widths[n_layers - 1];
  MM_REQUIRE(!head_w || n_last <= 32, MM_ERR_UNSUPPORTED, "mm_mlp_tc: the fused Dense(N->1) head needs a last width <= 32");
  MM_REQUIRE(!head_w || (head_act >= MM_ACT_LINEAR && head_act <= MM_ACT_GELU), MM_ERR_ARG, "mm_mlp_tc: unknown head activation");
  MM_REQUIRE(!out || out_stride >= n_last, MM_ERR_ARG, "mm_mlp_tc: out_stride < last width");
  if (M == 0) return MM_OK;

  Params p;
  size_t smem = 0;
  MM_REQUIRE(plan_tower(K, n_layers, widths, p, smem), MM_ERR_UNSUPPORTED,
             "mm_mlp_tc: the tower does not fit in shared memory with two pipeline stages (mm_mlp_tc_supported)");
  p.M = M;
  p.act1 = acts[0];
  for (int l = 0; l < n_layers; ++l) p.bias[l] = bias[l];
  for (int c = 0; c < p.n_chain; ++c) p.c[c].act = acts[c + 1];
  p.out_f32 = out;
  p.out_stride = out_stride;
  p.out_operand = (uint8_t*)out_operand;
  p.head_w = head_w;
  p.head_b = head_b;
  p.head_act = head_act;
  p.head_out = head_out;

  CUtensorMap tmA, tmW1, tmC[kMaxChain];
  int rc = mm::tc::make_map(&tmA, a_split, (uint64_t)M, (uint64_t)2 * p.K1p, BLOCK_M);
  if (rc) return rc;
  rc = mm::tc::make_map(&tmW1, w_split[0], (uint64_t)p.N1p, (uint64_t)2 * p.K1p, (uint32_t)p.N1p);
  if (rc) return rc;
  for (int c = 0; c < kMaxChain; ++c) {
    if (c < p.n_chain) {
      rc = mm::tc::make_map(&tmC[c], w_split[c + 1], (uint64_t)p.c[c].Np, (uint64_t)2 * p.c[c].Kp, (uint32_t)p.c[c].Np);
      if (rc) return rc;
    } else {
      tmC[c] = tmW1;
    }
  }

  static size_t smem_set = 0;
  if (smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(mlp_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      mm::set_error("mm_mlp_tc: cudaFuncSetAttribute(227 KB smem) failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
    smem_set = 227 * 1024;
  }
  const long long tiles = (M + BLOCK_M - 1) / BLOCK_M;
  const int sms = mm::sm_count();
  const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
  mlp_tc_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(tmA, tmW1, tmC[0], tmC[1], tmC[2], p);
  return mm::check_launch("mm_mlp_tc");
}

extern "C" {

int mm_mlp_tc(const void* a_split, int64_t M, int K, int n_layers, const void* const* w_split, const int* widths,
              const float* const* bias, const int* acts, float* out, int64_t out_stride, const float* head_w,
              float head_b, int head_act, float* head_out, void* stream) {
  return mlp_tc_impl(a_split, M, K, n_layers, w_split, widths, bias, acts, out, out_stride, head_w, head_b, head_act, head_out,
                     nullptr, stream);
}

int mm_mlp_tc_operand_out(const void* a_split, int64_t M, int K, int n_layers, const void* const* w_split, const int* widths,
                          const float* const* bias, const int* acts, float* out, int64_t out_stride, void* out_operand,
                          void* stream) {
  MM_REQUIRE(out_operand != nullptr, MM_ERR_ARG, "mm_mlp_tc_operand_out: out_operand is null");
  return mlp_tc_impl(a_split, M, K, n_layers, w_split, widths, bias, acts, out, out_stride, nullptr, 0.0f, 0, nullptr, out_operand,
                     stream);
}

}  // extern "C"
