// Narrow-input two-layer tower in one launch:  h = act2(act1(concat(columns) W1 + b1) W2 + b2)
//
// The DLRM bottom tower (13 continuous columns -> 128 -> 64) is 1.3 GFLOP and 20 MB of traffic per 65 536-sample
// batch — far too small for the TMA/wgmma tower kernel, whose per-tile latency chain (plus a separate concat+split
// launch in front of it) would dominate at these widths.  Here one warp owns 16 samples:
//   * the <= 16 input columns are read straight from their column arrays (ContinuousFeatures + ConcatFeatures:
//     sorted-name order, cast to fp32; merlin/models/tf/inputs/continuous.py:117-138, core/aggregation.py:54-66)
//     into the m16k16 A fragment — no concatenated matrix, no bf16 operand in HBM.  Each lane cp.asyncs its 8 values
//     of the warp's NEXT tile into a per-warp stage before the MMAs of the current one (the first tile's values are
//     in flight during the weight fill); all-fp32 inputs take an instantiation without any dtype handling;
//   * layer 1 and layer 2 run on mma.sync.m16n8k16 with the same 3-pass bf16 split as every other dense layer
//     (hi*lo + lo*hi + hi*hi, fp32 accumulate); the layer-1 accumulator fragment IS the layer-2 A fragment
//     (row/column ownership coincides), so the hidden activations never leave registers;
//   * both weight matrices sit in shared memory (pre-split K-major rows, padded against bank conflicts) and are
//     fetched as B fragments by ldmatrix.x4 (hi and lo of one n-tile per instruction);
//   * the last epilogue stages the tile's fp32 rows and/or split-bf16 rows [hi | lo] (the interaction kernel's
//     operand format) in a per-warp shared-memory area and writes them out with 16-byte stores, so every store
//     instruction covers whole 32-byte sectors.
// Replaces MLPBlock([N1, N2]) over a dict of <= 16 scalar features (blocks/mlp.py:97-139, :275-280).
#include <cuda_bf16.h>

#include <cstring>

#include "mm_common.cuh"
#include "warp_mma.cuh"

namespace mm {
namespace tsm {

constexpr int MAX_COLS = 16;
constexpr int WARPS = 16;  // 512 threads x <= 128 registers: the hidden layer is processed in chunks to fit

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
  int out_f32_v16;           // out_f32 rows can be written with 16-byte stores (else 8-byte)
  int out_split_v16;         // out_split is 16-byte aligned (else 4-byte stores)
};

struct ColS {  // one input column as the kernel reads it, in shared memory
  const uint8_t* base;  // row 0
  long long pitch;      // bytes between consecutive rows
  int dtype;
  int pad;
};

constexpr int W1_STRIDE = 80;  // bytes per n-row of W1 in shared memory: [hi k0..15 | lo k0..15] = 64 B + 16 B pad

// Shared memory of one CTA (byte offsets)
template <int N1T, int N2T, bool F32>
struct Layout {
  static constexpr int N1 = 8 * N1T, N2 = 8 * N2T;
  static constexpr int W2_STRIDE = N1 * 4 + 16;  // [hi k0..N1 | lo k0..N1] + pad
  static constexpr int SLOT = F32 ? 4 : 8;        // bytes per staged input value (8: raw int64 / fp64 bits)
  static constexpr int SPLIT_PITCH = 4 * N2 + 16;  // staged split row [hi | lo] + pad: rows g land 16 B apart in the banks
  static constexpr int F32_PITCH = 4 * N2 + 32;    // staged fp32 row + pad: the float2 writes of 4 rows are conflict-free
  static constexpr int W1 = 0;
  static constexpr int W2 = W1 + N1 * W1_STRIDE;
  static constexpr int B1 = W2 + N2 * W2_STRIDE;
  static constexpr int B2 = B1 + 4 * N1;
  static constexpr int COLS = B2 + 4 * N2;
  static constexpr int XIN = COLS + MAX_COLS * (int)sizeof(ColS);
  static constexpr int XIN_WARP = 2 * 8 * 32 * SLOT;  // two tiles x [value v][lane] slots
  static constexpr int OUT = XIN + WARPS * XIN_WARP;
  static constexpr int OUT_WARP = 16 * F32_PITCH;  // also holds 16 split rows (SPLIT_PITCH < F32_PITCH)
  static constexpr int BYTES = OUT + WARPS * OUT_WARP;
};

// N1T / N2T: number of 8-column n-tiles of layer 1 / layer 2 (N1 = 8*N1T is also the K of layer 2, a multiple of 16)
template <bool RELU>
__device__ __forceinline__ float act_fn(float v, int act) {
  return RELU ? fmaxf(v, 0.0f) : apply_act(v, act);
}

// A staged input value (raw bits as copied; the high word only for 8-byte dtypes) -> fp32, as load_as_f32 converts it
__device__ __forceinline__ float raw_to_f32(uint2 raw, int dt) {
  const long long i64 = (long long)(((unsigned long long)raw.y << 32) | raw.x);
  float f = __uint_as_float(raw.x);  // MM_F32
  f = dt == MM_I32 ? (float)(int)raw.x : f;
  f = dt == MM_I64 ? (float)i64 : f;
  f = dt == MM_F64 ? (float)__longlong_as_double(i64) : f;
  return f;
}

// 16 staged rows of ROW_BYTES -> global rows dst + r * dst_pitch (r < rows), sizeof(V) bytes per lane and store:
// consecutive lanes write consecutive pieces of a row
template <int ROW_BYTES, typename V>
__device__ __forceinline__ void store_rows(const uint8_t* st, int pitch, uint8_t* dst, long long dst_pitch, int rows, int lane) {
  constexpr int PER_ROW = ROW_BYTES / (int)sizeof(V), N = 16 * PER_ROW;
#pragma unroll
  for (int i = 0; i < (N + 31) / 32; ++i) {
    const int c = i * 32 + lane;
    const int r = c / PER_ROW, q = c % PER_ROW;
    if ((N % 32 == 0 || c < N) && r < rows)
      *reinterpret_cast<V*>(dst + r * dst_pitch + q * (int)sizeof(V)) = *reinterpret_cast<const V*>(st + r * pitch + q * (int)sizeof(V));
  }
}

// RELU: both activations are relu (compile-time fast path: no per-element dispatch).  F32: every column is fp32.
template <int N1T, int N2T, bool RELU, bool F32>
__global__ void __launch_bounds__(32 * WARPS)
tower_small_kernel(const __grid_constant__ Cols cols, const Params p) {
  extern __shared__ __align__(16) uint8_t smem[];
  using L = Layout<N1T, N2T, F32>;
  constexpr int N1 = L::N1, N2 = L::N2, W2_STRIDE = L::W2_STRIDE, SLOT = L::SLOT;
  uint8_t* w1s = smem + L::W1;
  uint8_t* w2s = smem + L::W2;
  float* b1s = reinterpret_cast<float*>(smem + L::B1);
  float* b2s = reinterpret_cast<float*>(smem + L::B2);
  ColS* cs = reinterpret_cast<ColS*>(smem + L::COLS);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  uint8_t* xin = smem + L::XIN + warp * L::XIN_WARP;
  uint8_t* ost = smem + L::OUT + warp * L::OUT_WARP;

  if (threadIdx.x < MAX_COLS) {  // columns past K read column 0's address with zero fill
    const int k = threadIdx.x < cols.K ? threadIdx.x : 0;
    const int dt = cols.dtype[k];
    const int esz = (dt == MM_I64 || dt == MM_F64) ? 8 : 4;
    cs[threadIdx.x] = ColS{reinterpret_cast<const uint8_t*>(cols.src[k]) + (long long)cols.off[k] * esz, cols.stride[k] * esz, dt, 0};
  }
  __syncthreads();

  // this lane's values of tile `tile` -> stage `buf`: columns k = 2t, 2t+1, 2t+8, 2t+9 (j = 0..3) of rows g and g+8
  // (h = 0, 1) as value v = 2j + h; rows at or past B and columns at or past K are zero-filled
  const long long tiles = (p.B + 15) >> 4;
  const long long tstep = (long long)gridDim.x * WARPS;
  auto issue = [&](long long tile, int buf) {
    const uint32_t dst0 = (uint32_t)__cvta_generic_to_shared(xin) + (uint32_t)(buf * 8 * 32 * SLOT + lane * SLOT);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = 2 * t + (j & 1) + ((j >> 1) << 3);
      const ColS c = cs[k];
      const bool on = k < cols.K;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = tile * 16 + g + 8 * h;
        const bool valid = on && r < p.B;
        const uint8_t* src = c.base + (valid ? r * c.pitch : 0);
        const uint32_t dst = dst0 + (uint32_t)((2 * j + h) * 32 * SLOT);
        if (F32 || !(c.dtype == MM_I64 || c.dtype == MM_F64))
          cp_async4_zfill(dst, src, valid);
        else
          cp_async8_zfill(dst, src, valid);
      }
    }
    cp_async_commit();
  };
  long long tile = (long long)blockIdx.x * WARPS + warp;
  issue(tile, 0);  // in flight during the weight fill

  // ---- weights -> shared memory (once per CTA), 16-byte cp.async: every chunk of a thread in flight at once
  for (int e = threadIdx.x; e < N1 * 4; e += blockDim.x) {  // W1 row n: hi k0..15 (2 x 16 B) | lo k0..15 (2 x 16 B)
    const int n = e >> 2, c = e & 3;
    cp_async16_if(true, (uint32_t)__cvta_generic_to_shared(w1s + n * W1_STRIDE + c * 16),
                  p.w1 + (long long)n * 2 * p.K1p + (c < 2 ? c * 8 : p.K1p + (c - 2) * 8));
  }
  constexpr int C2 = N1 / 8;  // 16-byte chunks per half row of W2
  for (int e = threadIdx.x; e < N2 * 2 * C2; e += blockDim.x) {
    const int n = e / (2 * C2), c = e % (2 * C2);
    cp_async16_if(true, (uint32_t)__cvta_generic_to_shared(w2s + n * W2_STRIDE + c * 16),
                  p.w2 + (long long)n * 2 * p.K2p + (c < C2 ? c * 8 : p.K2p + (c - C2) * 8));
  }
  cp_async_commit();
  for (int e = threadIdx.x; e < N1; e += blockDim.x) b1s[e] = p.b1 ? p.b1[e] : 0.0f;
  for (int e = threadIdx.x; e < N2; e += blockDim.x) b2s[e] = p.b2 ? p.b2[e] : 0.0f;
  cp_async_wait<0>();  // (also the first tile's values, issued before the weights)
  __syncthreads();

  const uint32_t w1_lane = (uint32_t)__cvta_generic_to_shared(w1s) + (uint32_t)(lane & 7) * W1_STRIDE + (uint32_t)(lane >> 3) * 16u;
  // W2: matrices (hi, chunk 2ks) (hi, 2ks+1) (lo, 2ks) (lo, 2ks+1) of rows 8nt + (lane & 7)
  const uint32_t w2_lane = (uint32_t)__cvta_generic_to_shared(w2s) + (uint32_t)(lane & 7) * W2_STRIDE +
                           (uint32_t)((lane >> 3) & 1) * 16u + (uint32_t)(lane >> 4) * (N1 * 2);
  for (int buf = 0; tile < tiles; tile += tstep, buf ^= 1) {
    issue(tile + tstep, buf ^ 1);  // zero-filled past the last tile
    cp_async_wait<1>();            // this tile's values (each lane reads only the slots it copied itself)
    // ---- A fragment of layer 1: rows {g, g+8} x k {2t, 2t+1, 2t+8, 2t+9}
    float x[2][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint8_t* s = xin + buf * 8 * 32 * SLOT + (2 * j + h) * 32 * SLOT + lane * SLOT;
        if (F32) {
          x[h][j] = *reinterpret_cast<const float*>(s);
        } else {
          const int k = 2 * t + (j & 1) + ((j >> 1) << 3);
          x[h][j] = raw_to_f32(*reinterpret_cast<const uint2*>(s), k < cols.K ? cols.dtype[k] : cs[0].dtype);
        }
      }
    }
    uint32_t ah[4], al[4];
    split_pair(x[0][0], x[0][1], ah[0], al[0]);
    split_pair(x[1][0], x[1][1], ah[1], al[1]);
    split_pair(x[0][2], x[0][3], ah[2], al[2]);
    split_pair(x[1][2], x[1][3], ah[3], al[3]);
    // ---- the hidden layer in chunks of HT = 4 n-tiles: layer 1 computes 32 hidden units, which are at once consumed as
    // 2 k-steps of layer 2 (the accumulator fragment of n-tiles (2k, 2k+1) IS the A fragment of k-step k), so only 32
    // hidden activations per row are live at a time.  Groups of 4 n-tiles, pass-major: four independent accumulators
    // between dependent MMAs.  The chunk loop stays rolled for the wide relu shapes: unrolled, ptxas hoists the next
    // chunk's fragment loads and spills.
    constexpr int HT = 4;
    float acc2[N2T][4];
#pragma unroll
    for (int nt = 0; nt < N2T; ++nt) acc2[nt][0] = acc2[nt][1] = acc2[nt][2] = acc2[nt][3] = 0.0f;
#pragma unroll (RELU && N1T * N2T >= 64 ? 1 : N1T / HT)
    for (int ch = 0; ch < N1T / HT; ++ch) {
      float acc1[HT][4];
#pragma unroll
      for (int n0 = 0; n0 < HT; n0 += 4) {
        uint32_t bh[4][2], bl[4][2];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          ldsm_x4(w1_lane + (uint32_t)(ch * HT + n0 + u) * (8 * W1_STRIDE), bh[u][0], bh[u][1], bl[u][0], bl[u][1]);
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
        const float2 b = *reinterpret_cast<const float2*>(b1s + 8 * (ch * HT + nt) + 2 * t);
        acc1[nt][0] = act_fn<RELU>(acc1[nt][0] + b.x, p.act1);
        acc1[nt][1] = act_fn<RELU>(acc1[nt][1] + b.y, p.act1);
        acc1[nt][2] = act_fn<RELU>(acc1[nt][2] + b.x, p.act1);
        acc1[nt][3] = act_fn<RELU>(acc1[nt][3] + b.y, p.act1);
      }
#pragma unroll
      for (int kq = 0; kq < HT / 2; ++kq) {
        const int ks = ch * (HT / 2) + kq;
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
    // ---- epilogue: bias + activation; fp32 rows and / or split-bf16 rows, each staged and then stored row-contiguous
#pragma unroll
    for (int nt = 0; nt < N2T; ++nt) {
      const float2 b = *reinterpret_cast<const float2*>(b2s + 8 * nt + 2 * t);
      acc2[nt][0] = act_fn<RELU>(acc2[nt][0] + b.x, p.act2);
      acc2[nt][1] = act_fn<RELU>(acc2[nt][1] + b.y, p.act2);
      acc2[nt][2] = act_fn<RELU>(acc2[nt][2] + b.x, p.act2);
      acc2[nt][3] = act_fn<RELU>(acc2[nt][3] + b.y, p.act2);
    }
    const int rows = (int)min(16LL, p.B - tile * 16);
    if (p.out_split) {
#pragma unroll
      for (int nt = 0; nt < N2T; ++nt) {
        const int n = 8 * nt + 2 * t;
        uint32_t h0, l0, h1, l1;
        split_pair(acc2[nt][0], acc2[nt][1], h0, l0);
        split_pair(acc2[nt][2], acc2[nt][3], h1, l1);
        *reinterpret_cast<uint32_t*>(ost + g * L::SPLIT_PITCH + 2 * n) = h0;
        *reinterpret_cast<uint32_t*>(ost + g * L::SPLIT_PITCH + 2 * (N2 + n)) = l0;
        *reinterpret_cast<uint32_t*>(ost + (g + 8) * L::SPLIT_PITCH + 2 * n) = h1;
        *reinterpret_cast<uint32_t*>(ost + (g + 8) * L::SPLIT_PITCH + 2 * (N2 + n)) = l1;
      }
      __syncwarp();
      uint8_t* dst = reinterpret_cast<uint8_t*>(p.out_split) + tile * 16 * (4 * N2);
      if (p.out_split_v16)
        store_rows<4 * N2, uint4>(ost, L::SPLIT_PITCH, dst, 4 * N2, rows, lane);
      else
        store_rows<4 * N2, uint32_t>(ost, L::SPLIT_PITCH, dst, 4 * N2, rows, lane);
      __syncwarp();
    }
    if (p.out_f32) {
#pragma unroll
      for (int nt = 0; nt < N2T; ++nt) {
        const int n = 8 * nt + 2 * t;
        *reinterpret_cast<float2*>(ost + g * L::F32_PITCH + 4 * n) = make_float2(acc2[nt][0], acc2[nt][1]);
        *reinterpret_cast<float2*>(ost + (g + 8) * L::F32_PITCH + 4 * n) = make_float2(acc2[nt][2], acc2[nt][3]);
      }
      __syncwarp();
      const long long pitch = p.out_stride * 4;
      uint8_t* dst = reinterpret_cast<uint8_t*>(p.out_f32) + tile * 16 * pitch;
      if (p.out_f32_v16)
        store_rows<4 * N2, uint4>(ost, L::F32_PITCH, dst, pitch, rows, lane);
      else
        store_rows<4 * N2, uint2>(ost, L::F32_PITCH, dst, pitch, rows, lane);
      __syncwarp();
    }
  }
  cp_async_wait<0>();
}

template <int N1T, int N2T, bool RELU, bool F32>
static int launch(const Cols& c, const Params& p, cudaStream_t st) {
  const size_t smem = (size_t)Layout<N1T, N2T, F32>::BYTES;
  auto kern = tower_small_kernel<N1T, N2T, RELU, F32>;
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

template <int N1T, int N2T>
static int launch(const Cols& c, const Params& p, bool relu, bool f32, cudaStream_t st) {
  if (f32) return relu ? launch<N1T, N2T, true, true>(c, p, st) : launch<N1T, N2T, false, true>(c, p, st);
  return relu ? launch<N1T, N2T, true, false>(c, p, st) : launch<N1T, N2T, false, false>(c, p, st);
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
  bool f32 = true;
  for (int i = 0; i < n_pieces; ++i) {
    const mm_concat_piece& pc = pieces_host[i];
    MM_REQUIRE(pc.src && pc.width >= 1 && pc.src_stride >= pc.width && pc.dtype >= MM_I32 && pc.dtype <= MM_F64, MM_ERR_ARG,
               "mm_tower2_small: piece %d: null source, bad width / stride / dtype", i);
    MM_REQUIRE(pc.out_col == K, MM_ERR_ARG, "mm_tower2_small: pieces must be listed in column order without gaps (piece %d)", i);
    f32 = f32 && pc.dtype == MM_F32;
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
  p.out_f32_v16 = ((uintptr_t)out % 16) == 0 && (out_stride % 4) == 0;
  p.out_split_v16 = ((uintptr_t)out_split % 16) == 0;
  cudaStream_t st = (cudaStream_t)stream;
  const bool relu = act1 == MM_ACT_RELU && act2 == MM_ACT_RELU;
#define MM_TSM(a, b) \
  if (N1 == 8 * a && N2 == 8 * b) return launch<a, b>(c, p, relu, f32, st);
  MM_TSM(16, 8) MM_TSM(16, 4) MM_TSM(16, 2) MM_TSM(8, 8) MM_TSM(8, 4) MM_TSM(8, 2) MM_TSM(4, 8) MM_TSM(4, 4) MM_TSM(4, 2)
#undef MM_TSM
  return MM_ERR_UNSUPPORTED;
}

}  // extern "C"
