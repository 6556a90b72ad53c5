// Narrow-input two-layer tower in one launch:  h = act2(act1(concat(columns) W1 + b1) W2 + b2)
//
// The DLRM bottom tower (13 continuous columns -> 128 -> 64) is 1.3 GFLOP and 20 MB of traffic per 65 536-sample
// batch — far too small for the TMA/wgmma tower kernel, whose per-tile latency chain (plus the separate
// concat+split launch in front of it) cost 34 us of a 147 us step.  Here one warp owns 16 samples:
//   * the <= 16 input columns are read straight from their column arrays (ContinuousFeatures + ConcatFeatures:
//     sorted-name order, cast to fp32; merlin/models/tf/inputs/continuous.py:117-138, core/aggregation.py:54-66)
//     into the m16k16 A fragment — no concatenated matrix, no bf16 operand in HBM;
//   * layer 1 and layer 2 run on mma.sync.m16n8k16 with the same 3-pass bf16 split as every other dense layer
//     (hi*lo + lo*hi + hi*hi, fp32 accumulate); the layer-1 accumulator fragment IS the layer-2 A fragment
//     (row/column ownership coincides), so the hidden activations never leave registers;
//   * both weight matrices sit in shared memory (pre-split K-major rows, padded against bank conflicts) and are
//     fetched as B fragments by ldmatrix.x4 (hi and lo of one n-tile per instruction);
//   * the last epilogue writes fp32 rows and/or split-bf16 rows [hi | lo] (the interaction kernel's operand format).
// Replaces MLPBlock([N1, N2]) over a dict of <= 16 scalar features (blocks/mlp.py:97-139, :275-280).
#include <cuda_bf16.h>

#include <cstring>

#include "mm_common.cuh"
#include "warp_mma.cuh"

namespace mm {
namespace tsm {

constexpr int MAX_COLS = 16;
constexpr int WARPS = 16;  // 512 threads x <= 128 registers: the hidden layer is processed in halves to fit

struct Cols {  // one entry per input COLUMN (a width-w piece contributes w entries)
  const void* src[MAX_COLS];
  long long stride[MAX_COLS];  // elements between consecutive rows
  int off[MAX_COLS];           // element offset of this column inside a row of its piece
  int dtype[MAX_COLS];
  int K;
};

struct Params {
  long long B;
  const __nv_bfloat16* w1;  // mm_split_weights layout (N1p, 2*K1p)
  const __nv_bfloat16* w2;  // (N2p, 2*K2p), K2 = N1
  int K1p, K2p;
  const float* b1;
  const float* b2;
  int act1, act2;
  float* out_f32;
  long long out_stride;
  __nv_bfloat16* out_split;  // (B, 2*N2) [hi | lo]
};

constexpr int W1_STRIDE = 80;  // bytes per n-row of W1 in shared memory: [hi k0..15 | lo k0..15] = 64 B + 16 B pad

// N1T / N2T: number of 8-column n-tiles of layer 1 / layer 2 (N1 = 8*N1T is also the K of layer 2, a multiple of 16)
template <bool RELU>
__device__ __forceinline__ float act_fn(float v, int act) {
  return RELU ? fmaxf(v, 0.0f) : apply_act(v, act);
}

// RELU: both activations are relu (compile-time fast path: no per-element dispatch)
template <int N1T, int N2T, bool RELU>
__global__ void __launch_bounds__(32 * WARPS)
tower_small_kernel(const __grid_constant__ Cols cols, const Params p) {
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int N1 = 8 * N1T, N2 = 8 * N2T;
  constexpr int W2_STRIDE = N1 * 4 + 16;  // [hi k0..N1 | lo k0..N1] + pad
  uint8_t* w1s = smem;
  uint8_t* w2s = w1s + N1 * W1_STRIDE;
  float* b1s = reinterpret_cast<float*>(w2s + N2 * W2_STRIDE);
  float* b2s = b1s + N1;
  // ---- weights -> shared memory (once per CTA), 16 bytes per load
  for (int e = threadIdx.x; e < N1 * 4; e += blockDim.x) {  // W1 row n: hi k0..15 (2 x 16 B) | lo k0..15 (2 x 16 B)
    const int n = e >> 2, c = e & 3;
    const uint4 v = *reinterpret_cast<const uint4*>(p.w1 + (long long)n * 2 * p.K1p + (c < 2 ? c * 8 : p.K1p + (c - 2) * 8));
    *reinterpret_cast<uint4*>(w1s + n * W1_STRIDE + c * 16) = v;
  }
  constexpr int C2 = N1 / 8;  // 16-byte chunks per half row of W2
  for (int e = threadIdx.x; e < N2 * 2 * C2; e += blockDim.x) {
    const int n = e / (2 * C2), c = e % (2 * C2);
    const uint4 v = *reinterpret_cast<const uint4*>(p.w2 + (long long)n * 2 * p.K2p + (c < C2 ? c * 8 : p.K2p + (c - C2) * 8));
    *reinterpret_cast<uint4*>(w2s + n * W2_STRIDE + c * 16) = v;
  }
  for (int e = threadIdx.x; e < N1; e += blockDim.x) b1s[e] = p.b1 ? p.b1[e] : 0.0f;
  for (int e = threadIdx.x; e < N2; e += blockDim.x) b2s[e] = p.b2 ? p.b2[e] : 0.0f;
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const uint32_t w1_lane = (uint32_t)__cvta_generic_to_shared(w1s) + (uint32_t)(lane & 7) * W1_STRIDE + (uint32_t)(lane >> 3) * 16u;
  // W2: matrices (hi, chunk 2ks) (hi, 2ks+1) (lo, 2ks) (lo, 2ks+1) of rows 8nt + (lane & 7)
  const uint32_t w2_lane = (uint32_t)__cvta_generic_to_shared(w2s) + (uint32_t)(lane & 7) * W2_STRIDE +
                           (uint32_t)((lane >> 3) & 1) * 16u + (uint32_t)(lane >> 4) * (N1 * 2);
  // this lane's four input columns k = 2t, 2t+1, 2t+8, 2t+9 as running byte pointers (row g of the warp's first tile)
  const long long tiles = (p.B + 15) >> 4;
  const long long tile0 = (long long)blockIdx.x * WARPS + warp, tstep = (long long)gridDim.x * WARPS;
  const uint8_t* cptr[4];
  int cstep[4];  // bytes between consecutive rows of the column
  uint32_t cdts = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = 2 * t + (j & 1) + ((j >> 1) << 3);
    const bool on = k < cols.K;
    const int kk = on ? k : 0;
    const int dt = cols.dtype[kk];
    const int esz = (dt == MM_I64 || dt == MM_F64) ? 8 : 4;
    cstep[j] = (int)(cols.stride[kk] * esz);
    cptr[j] = on ? reinterpret_cast<const uint8_t*>(cols.src[kk]) + (long long)cols.off[kk] * esz + (tile0 * 16 + g) * (long long)cstep[j]
                 : nullptr;
    cdts |= (uint32_t)dt << (8 * j);
  }
  for (long long tile = tile0; tile < tiles; tile += tstep) {
    const long long r0 = tile * 16 + g, r1 = r0 + 8;
    const bool v0 = r0 < p.B, v1 = r1 < p.B;
    // ---- A fragment of layer 1 from the column arrays: rows {g, g+8} x k {2t, 2t+1, 2t+8, 2t+9}
    float x[2][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int dt = (int)((cdts >> (8 * j)) & 0xff);
      x[0][j] = (cptr[j] && v0) ? load_as_f32<true>(cptr[j], 0, dt) : 0.0f;
      x[1][j] = (cptr[j] && v1) ? load_as_f32<true>(cptr[j] + 8 * (long long)cstep[j], 0, dt) : 0.0f;
      if (cptr[j]) cptr[j] += tstep * 16 * (long long)cstep[j];
    }
    uint32_t ah[4], al[4];
    split_pair(x[0][0], x[0][1], ah[0], al[0]);
    split_pair(x[1][0], x[1][1], ah[1], al[1]);
    split_pair(x[0][2], x[0][3], ah[2], al[2]);
    split_pair(x[1][2], x[1][3], ah[3], al[3]);
    // ---- the hidden layer in halves of HT n-tiles: layer 1 computes HT*8 hidden units, which are at once consumed as
    // HT/2 k-steps of layer 2 (the accumulator fragment of n-tiles (2k, 2k+1) IS the A fragment of k-step k), so only half
    // of the hidden activations is live at a time.  Groups of 4 n-tiles, pass-major: four independent accumulators
    // between dependent MMAs.
    constexpr int HT = N1T >= 8 ? N1T / 2 : N1T;
    float acc2[N2T][4];
#pragma unroll
    for (int nt = 0; nt < N2T; ++nt) acc2[nt][0] = acc2[nt][1] = acc2[nt][2] = acc2[nt][3] = 0.0f;
#pragma unroll
    for (int half = 0; half < N1T / HT; ++half) {
      float acc1[HT][4];
#pragma unroll
      for (int n0 = 0; n0 < HT; n0 += 4) {
        uint32_t bh[4][2], bl[4][2];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          ldsm_x4(w1_lane + (uint32_t)(half * HT + n0 + u) * (8 * W1_STRIDE), bh[u][0], bh[u][1], bl[u][0], bl[u][1]);
          acc1[n0 + u][0] = acc1[n0 + u][1] = acc1[n0 + u][2] = acc1[n0 + u][3] = 0.0f;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) mma16816(acc1[n0 + u], ah, bl[u][0], bl[u][1]);
#pragma unroll
        for (int u = 0; u < 4; ++u) mma16816(acc1[n0 + u], al, bh[u][0], bh[u][1]);
#pragma unroll
        for (int u = 0; u < 4; ++u) mma16816(acc1[n0 + u], ah, bh[u][0], bh[u][1]);
      }
#pragma unroll
      for (int nt = 0; nt < HT; ++nt) {
        const float2 b = *reinterpret_cast<const float2*>(b1s + 8 * (half * HT + nt) + 2 * t);
        acc1[nt][0] = act_fn<RELU>(acc1[nt][0] + b.x, p.act1);
        acc1[nt][1] = act_fn<RELU>(acc1[nt][1] + b.y, p.act1);
        acc1[nt][2] = act_fn<RELU>(acc1[nt][2] + b.x, p.act1);
        acc1[nt][3] = act_fn<RELU>(acc1[nt][3] + b.y, p.act1);
      }
#pragma unroll
      for (int kq = 0; kq < HT / 2; ++kq) {
        const int ks = half * (HT / 2) + kq;
        uint32_t a2h[4], a2l[4];
        split_pair(acc1[2 * kq][0], acc1[2 * kq][1], a2h[0], a2l[0]);
        split_pair(acc1[2 * kq][2], acc1[2 * kq][3], a2h[1], a2l[1]);
        split_pair(acc1[2 * kq + 1][0], acc1[2 * kq + 1][1], a2h[2], a2l[2]);
        split_pair(acc1[2 * kq + 1][2], acc1[2 * kq + 1][3], a2h[3], a2l[3]);
        constexpr int G = N2T < 4 ? N2T : 4;
#pragma unroll
        for (int n0 = 0; n0 < N2T; n0 += G) {
          uint32_t bh[G][2], bl[G][2];
#pragma unroll
          for (int u = 0; u < G; ++u)
            ldsm_x4(w2_lane + (uint32_t)(n0 + u) * (8 * W2_STRIDE) + (uint32_t)ks * 32u, bh[u][0], bh[u][1], bl[u][0], bl[u][1]);
#pragma unroll
          for (int u = 0; u < G; ++u) mma16816(acc2[n0 + u], a2h, bl[u][0], bl[u][1]);
#pragma unroll
          for (int u = 0; u < G; ++u) mma16816(acc2[n0 + u], a2l, bh[u][0], bh[u][1]);
#pragma unroll
          for (int u = 0; u < G; ++u) mma16816(acc2[n0 + u], a2h, bh[u][0], bh[u][1]);
        }
      }
    }
    // ---- epilogue: bias + activation, fp32 rows and / or split-bf16 rows
#pragma unroll
    for (int nt = 0; nt < N2T; ++nt) {
      const int n = 8 * nt + 2 * t;
      const float2 b = *reinterpret_cast<const float2*>(b2s + n);
      const float y00 = act_fn<RELU>(acc2[nt][0] + b.x, p.act2), y01 = act_fn<RELU>(acc2[nt][1] + b.y, p.act2);
      const float y10 = act_fn<RELU>(acc2[nt][2] + b.x, p.act2), y11 = act_fn<RELU>(acc2[nt][3] + b.y, p.act2);
      if (p.out_f32) {
        if (v0) *reinterpret_cast<float2*>(p.out_f32 + r0 * p.out_stride + n) = make_float2(y00, y01);
        if (v1) *reinterpret_cast<float2*>(p.out_f32 + r1 * p.out_stride + n) = make_float2(y10, y11);
      }
      if (p.out_split) {
        uint32_t h0, l0, h1, l1;
        split_pair(y00, y01, h0, l0);
        split_pair(y10, y11, h1, l1);
        if (v0) {
          *reinterpret_cast<uint32_t*>(p.out_split + r0 * (2 * N2) + n) = h0;
          *reinterpret_cast<uint32_t*>(p.out_split + r0 * (2 * N2) + N2 + n) = l0;
        }
        if (v1) {
          *reinterpret_cast<uint32_t*>(p.out_split + r1 * (2 * N2) + n) = h1;
          *reinterpret_cast<uint32_t*>(p.out_split + r1 * (2 * N2) + N2 + n) = l1;
        }
      }
    }
  }
}

template <int N1T, int N2T, bool RELU>
static int launch(const Cols& c, const Params& p, cudaStream_t st) {
  constexpr int N1 = 8 * N1T, N2 = 8 * N2T;
  const size_t smem = (size_t)N1 * W1_STRIDE + (size_t)N2 * (N1 * 4 + 16) + (size_t)(N1 + N2) * sizeof(float);
  auto kern = tower_small_kernel<N1T, N2T, RELU>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("mm_tower2_small: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
  }
  const long long tiles = (p.B + 15) / 16;
  long long blocks = (tiles + WARPS - 1) / WARPS;
  const long long cap = (long long)sm_count();  // one 16-warp CTA per SM: the weight fill is paid once per SM
  if (blocks > cap) blocks = cap;
  kern<<<(unsigned)blocks, 32 * WARPS, smem, st>>>(c, p);
  return check_launch("mm_tower2_small");
}

}  // namespace tsm
}  // namespace mm

extern "C" {

int mm_tower2_small_supported(int K, int N1, int N2) {
  return (K >= 1 && K <= mm::tsm::MAX_COLS && (N1 == 128 || N1 == 64 || N1 == 32) && (N2 == 64 || N2 == 32 || N2 == 16)) ? 1 : 0;
}

int mm_tower2_small(const mm_concat_piece* pieces_host, int n_pieces, int64_t B, const void* w1_split, int N1,
                    const float* bias1, int act1, const void* w2_split, int N2, const float* bias2, int act2, float* out,
                    int64_t out_stride, void* out_split, void* stream) {
  using namespace mm::tsm;
  MM_REQUIRE(pieces_host && n_pieces > 0 && w1_split && w2_split && B >= 0 && (out || out_split), MM_ERR_ARG,
             "mm_tower2_small: null pointer, no pieces or no output");
  Cols c;
  memset(&c, 0, sizeof(c));
  int K = 0;
  for (int i = 0; i < n_pieces; ++i) {
    const mm_concat_piece& pc = pieces_host[i];
    MM_REQUIRE(pc.src && pc.width >= 1 && pc.src_stride >= pc.width && pc.dtype >= MM_I32 && pc.dtype <= MM_F64, MM_ERR_ARG,
               "mm_tower2_small: piece %d: null source, bad width / stride / dtype", i);
    MM_REQUIRE(pc.out_col == K, MM_ERR_ARG, "mm_tower2_small: pieces must be listed in column order without gaps (piece %d)", i);
    for (int w = 0; w < pc.width; ++w) {
      MM_REQUIRE(K < MAX_COLS, MM_ERR_UNSUPPORTED, "mm_tower2_small: more than %d input columns", MAX_COLS);
      c.src[K] = pc.src;
      c.stride[K] = pc.src_stride;
      c.off[K] = w;
      c.dtype[K] = pc.dtype;
      ++K;
    }
  }
  c.K = K;
  MM_REQUIRE(mm_tower2_small_supported(K, N1, N2), MM_ERR_UNSUPPORTED, "mm_tower2_small: K=%d N1=%d N2=%d is outside the kernel (K <= 16, "
             "N1 in {32,64,128}, N2 in {16,32,64})", K, N1, N2);
  MM_REQUIRE(act1 >= MM_ACT_LINEAR && act1 <= MM_ACT_GELU && act2 >= MM_ACT_LINEAR && act2 <= MM_ACT_GELU, MM_ERR_ARG,
             "mm_tower2_small: unknown activation");
  MM_REQUIRE(!out || (out_stride >= N2 && (out_stride & 1) == 0 && ((uintptr_t)out % 8) == 0), MM_ERR_ALIGN,
             "mm_tower2_small: out needs an even stride >= N2 and 8-byte alignment");
  MM_REQUIRE(!out_split || ((uintptr_t)out_split % 4) == 0, MM_ERR_ALIGN, "mm_tower2_small: out_split misaligned");
  if (B == 0) return MM_OK;
  Params p;
  memset(&p, 0, sizeof(p));
  p.B = B;
  p.w1 = (const __nv_bfloat16*)w1_split;
  p.w2 = (const __nv_bfloat16*)w2_split;
  p.K1p = mm_tc_padded_k(K);
  p.K2p = mm_tc_padded_k(N1);
  p.b1 = bias1;
  p.b2 = bias2;
  p.act1 = act1;
  p.act2 = act2;
  p.out_f32 = out;
  p.out_stride = out_stride;
  p.out_split = (__nv_bfloat16*)out_split;
  cudaStream_t st = (cudaStream_t)stream;
  const bool relu = act1 == MM_ACT_RELU && act2 == MM_ACT_RELU;
#define MM_TSM(a, b) \
  if (N1 == 8 * a && N2 == 8 * b) return relu ? launch<a, b, true>(c, p, st) : launch<a, b, false>(c, p, st);
  MM_TSM(16, 8) MM_TSM(16, 4) MM_TSM(16, 2) MM_TSM(8, 8) MM_TSM(8, 4) MM_TSM(8, 2) MM_TSM(4, 8) MM_TSM(4, 4) MM_TSM(4, 2)
#undef MM_TSM
  return MM_ERR_UNSUPPORTED;
}

}  // extern "C"
