// Backward of the DLRM lookup + interaction stage and the optimizer kernels of the training step (SURVEY §8(f)-4).
//
//   mm_dlrm_interact_backward   per sample: X = the F staged rows (table rows looked up again + bottom vector),
//       G = symmetric (F x F) matrix of the pair gradients dA[P + pair(i, j)], zero diagonal; dX = G X.
//       Row `bottom_slot` of dX (+ the shortcut gradient dA[:D], masked by bottom > 0 when the bottom tower ends in
//       relu) is the bottom tower's gradient; every other row is the gradient of ONE embedding row and leaves as the
//       reference's IndexedSlices: values (B, D) per table, indices = the batch's ids (tf.GradientTape over
//       tf.gather, inputs/embedding.py:401-471; DotProductInteraction blocks/interaction.py:86-116).
//       One warp per sample on mma.sync (3-pass split-bf16 like the forward kernel): G is the A operand (built from the
//       staged dA row through a per-lane offset table), X the B operand.
//   mm_sparse_rows_*            the optimizer step on IndexedSlices with duplicate ids, as Keras applies it
//       (`_resource_apply_sparse_duplicate_indices`: sum the duplicates, then ONE update per unique row;
//       LazyAdam blocks/optimizer.py:342 touches only the looked-up rows).  Dedup without a sort: a per-row int32 map
//       (rows x 4 B, HBM is plentiful) elects the smallest sample index of every id as its representative
//       (atomicMin), the other duplicates add their slice into the representative's slice (vector reds), and
//       the representatives apply the update and reset the map.
//   mm_bag_grad_rows            backward of a pooled multi-hot feature: the pooled-row gradient expanded to one scaled
//       row per id, the IndexedSlices that mm_sparse_rows_apply consumes.
//   mm_dense_apply              SGD / Adagrad / Adam over a flat parameter arena (+ clears the gradients).
//   mm_opt_tick[_schedule]      the per-step tick of one optimizer's device hyper-parameters (step counter, Adam's lr_t),
//       with a learning-rate schedule evaluated at the step counter first (K25).
#include <cuda_bf16.h>

#include <climits>
#include <cstring>

#include "mm_common.cuh"
#include "warp_mma.cuh"

namespace mm {
namespace trs {

__device__ __align__(16) float g_zero_row[128];

struct IbwdParams {
  long long B;
  int F, P, bottom_slot;
  const float* bottom;  // (B, D) fp32 rows, the forward's bottom vector (null: no bottom row)
  long long bottom_stride;
  const float* dA;  // (B, P + F(F-1)/2): gradient of [bottom | pairs]
  long long dA_stride;
  int dA_vec;  // 16-byte copies of a dA row are legal
  float* d_bottom;
  long long d_bottom_stride;
  int mask_bottom;
  float* grad[MM_LOOKUP_MAX_ROWS];  // per staged row: (B, D) slice values of that table (null: none)
  long long grad_stride;
  int n_warps;
  unsigned buf_bytes, stage_off, stage_floats;
};

template <int KD>
__global__ void __launch_bounds__(256, 1) interact_bwd_kernel(const __grid_constant__ LookupParams lk, const __grid_constant__ IbwdParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int D = KD;
  constexpr int XS = D + 4;        // floats per staged row (+16 B: conflict-free column reads)
  constexpr int L = D / 4;         // lanes per row in the copy loop
  constexpr int R = 32 / L;        // rows per copy instruction
  constexpr int NTL = D / 8;       // n-tiles
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int F = p.F;
  const int OW = p.P + F * (F - 1) / 2;
  const uint32_t wbase = (uint32_t)__cvta_generic_to_shared(smem) + (uint32_t)warp * (2u * p.buf_bytes);

  // ---- rows >= F of both buffers and the zero slot of the dA stage stay zero for the whole kernel
  {
    float* mine = reinterpret_cast<float*>(smem + (size_t)warp * 2 * p.buf_bytes);
    for (int e = lane; e < (int)(2 * p.buf_bytes / 4); e += 32) mine[e] = 0.0f;
    __syncwarp();
  }

  // ---- G offsets (bytes into the dA stage) of this lane's A fragment elements: tile (mt, kt), register, element
  uint32_t goff[2][2][4][2];
  const uint32_t zero_slot = (p.stage_floats - 1) * 4u;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int kt = 0; kt < 2; ++kt)
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 16 * mt + g + 8 * (r & 1);
          const int j = 16 * kt + 2 * t + e + 8 * (r >> 1);
          uint32_t off = zero_slot;
          if (i != j && i < F && j < F) {
            const int a = min(i, j), b = max(i, j);
            off = (uint32_t)(p.P + a * (2 * F - a - 1) / 2 + (b - a - 1)) * 4u;
          }
          goff[mt][kt][r][e] = off;
        }

  // ---- owner role: lane r resolves the source of staged row r
  const bool is_table = lane < F && lane != p.bottom_slot && lk.weights[lane] != nullptr;
  const float* my_base = is_table ? lk.weights[lane] : nullptr;
  const unsigned long long my_rows = is_table ? (unsigned long long)lk.rows[lane] : 0ull;
  const int my_w = is_table ? lk.idx_bytes[lane] : 4;
  const void* my_ids = is_table ? lk.indices[lane] : nullptr;

  const int cl = lane % L, rl = lane / L;
  float* gptr[4];
#pragma unroll
  for (int qd = 0; qd < 4; ++qd) {
    const int i = 8 * qd + g;
    gptr[qd] = (i < F && i != p.bottom_slot) ? p.grad[i] : nullptr;
  }

  const long long stride_s = (long long)gridDim.x * p.n_warps;
  const long long s_first = (long long)blockIdx.x * p.n_warps + warp;

  auto issue = [&](long long s, uint32_t buf) {
    const bool live = s < p.B;
    const float* my_src = g_zero_row;
    if (live) {
      if (is_table) {
        const unsigned long long idx = (unsigned long long)load_id(my_ids, my_w, s);
        if (idx < my_rows) my_src = my_base + idx * D;
      } else if (lane == p.bottom_slot && p.bottom) {
        my_src = p.bottom + s * p.bottom_stride;
      }
    }
    const uint32_t lo = (uint32_t)(uintptr_t)my_src, hi = (uint32_t)((uintptr_t)my_src >> 32);
    const uint32_t xs = wbase + buf;
    for (int r0 = 0; r0 < F; r0 += R) {
      const int row = r0 + rl;
      const uint32_t slo = __shfl_sync(0xffffffffu, lo, row & 31);
      const uint32_t shi = __shfl_sync(0xffffffffu, hi, row & 31);
      const uint8_t* src = reinterpret_cast<const uint8_t*>(((uintptr_t)shi << 32) | slo) + cl * 16;
      cp_async16_if(live && row < F, xs + (uint32_t)(row * XS * 4 + cl * 16), src);
    }
    // the sample's dA row
    const float* da = p.dA + s * p.dA_stride;
    const uint32_t st = xs + p.stage_off;
    if (p.dA_vec) {
      for (int c = lane; c * 4 < OW; c += 32) cp_async16_if(live, st + (uint32_t)c * 16u, da + c * 4);
    } else {
      for (int c = lane; c < OW; c += 32) cp_async4_if(live, st + (uint32_t)c * 4u, da + c);
    }
    cp_async_commit();
  };

  issue(s_first, 0);
  uint32_t buf = 0;
  for (long long s = s_first; s < p.B; s += stride_s) {
    issue(s + stride_s, buf ^ p.buf_bytes);
    cp_async_wait<1>();
    __syncwarp();
    const uint32_t xs = wbase + buf, st = xs + p.stage_off;
    // a vector copy of the dA row may have written up to 3 floats past OW: the zero slot is the LAST stage float and
    // the launcher keeps stage_floats >= roundup4(OW) + 4, so it is never touched.
    // ---- A fragments of G
    uint32_t ah[2][2][4], al[2][2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int kt = 0; kt < 2; ++kt)
#pragma unroll
        for (int r = 0; r < 4; ++r)
          split_pair(lds32(st + goff[mt][kt][r][0]), lds32(st + goff[mt][kt][r][1]), ah[mt][kt][r], al[mt][kt][r]);
    float acc[2][NTL][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.0f;
#pragma unroll
    for (int kt = 0; kt < 2; ++kt) {
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) {
        // B fragment: X[j][d], j = 16kt + {2t, 2t+1, 2t+8, 2t+9}, d = 8nt + g
        const uint32_t a0 = xs + (uint32_t)(((16 * kt + 2 * t) * XS + 8 * nt + g) * 4);
        uint32_t bh0, bl0, bh1, bl1;
        split_pair(lds32(a0), lds32(a0 + XS * 4), bh0, bl0);
        split_pair(lds32(a0 + 8 * XS * 4), lds32(a0 + 9 * XS * 4), bh1, bl1);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma16816(acc[mt][nt], ah[mt][kt], bl0, bl1);
          mma16816(acc[mt][nt], al[mt][kt], bh0, bh1);
          mma16816(acc[mt][nt], ah[mt][kt], bh0, bh1);
        }
      }
    }
    // ---- dX rows: acc[mt][nt][c] = dX[16mt + g + 8(c>>1)][8nt + 2t + (c&1)]
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int qd = 2 * mt + h, i = 8 * qd + g;
        if (i >= F) continue;
        if (i == p.bottom_slot) {
          if (p.d_bottom) {
            float* drow = p.d_bottom + s * p.d_bottom_stride;
#pragma unroll
            for (int nt = 0; nt < NTL; ++nt) {
              const int d = 8 * nt + 2 * t;
              float a = acc[mt][nt][2 * h], b = acc[mt][nt][2 * h + 1];
              if (p.P > 0) {
                a += lds32(st + (uint32_t)d * 4u);
                b += lds32(st + (uint32_t)d * 4u + 4u);
              }
              if (p.mask_bottom) {
                const uint32_t xa = xs + (uint32_t)((i * XS + d) * 4);
                a = lds32(xa) > 0.0f ? a : 0.0f;
                b = lds32(xa + 4u) > 0.0f ? b : 0.0f;
              }
              *reinterpret_cast<float2*>(drow + d) = make_float2(a, b);
            }
          }
        } else if (gptr[qd]) {
          float* drow = gptr[qd] + s * p.grad_stride;
#pragma unroll
          for (int nt = 0; nt < NTL; ++nt)
            *reinterpret_cast<float2*>(drow + 8 * nt + 2 * t) = make_float2(acc[mt][nt][2 * h], acc[mt][nt][2 * h + 1]);
        }
      }
    __syncwarp();  // the buffer is refilled by the next iteration's copies
    buf ^= p.buf_bytes;
  }
  cp_async_wait<0>();
}

template <int KD>
static int launch_ibwd(const LookupParams& lk, IbwdParams p, cudaStream_t st) {
  const int OW = p.P + p.F * (p.F - 1) / 2;
  p.stage_off = 32u * (KD + 4) * 4u;
  p.stage_floats = (unsigned)(((OW + 3) & ~3) + 4);
  p.buf_bytes = (p.stage_off + p.stage_floats * 4u + 15u) & ~15u;
  int warps = (int)((227u * 1024u) / (2u * p.buf_bytes));
  if (warps > 8) warps = 8;
  if (warps < 1) return MM_ERR_UNSUPPORTED;
  p.n_warps = warps;
  const size_t smem = (size_t)warps * 2 * p.buf_bytes;
  auto kern = interact_bwd_kernel<KD>;
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("mm_dlrm_interact_backward: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  long long want = (p.B + warps - 1) / warps;
  const long long sms = sm_count();
  const unsigned grid = (unsigned)(want < sms ? want : sms);
  kern<<<grid, 32 * warps, smem, st>>>(lk, p);
  return check_launch("mm_dlrm_interact_backward");
}

// ---------------------------------------------------------------------------------------------------------------
// Operand-format variant (D = 64): the tables' mirrors and the bottom vector are split-bf16 rows [hi(0..63) | lo(0..63)]
// (mm_split_rows, the format the forward kernel reads with MM_ROWS_OPERAND and the optimizer kernels keep in step).
// First version above: 1 124 warp instructions per sample at 8 warps per SM (254 registers) — 64 + 192 of them only to
// load and split the X fragments, 128 to assemble the G fragments through a 32-register offset table.  Here
//   * the rows land in shared memory with the forward kernel's 128-byte XOR swizzle and the B fragments (X, k = feature
//     row, n = embedding column) come from ldmatrix.trans: 16 instructions, no conversion;
//   * G is built once per sample as two (32 x 32) bf16 matrices (hi, lo) in shared memory — lane e handles pairs
//     e, e+32, ...: one load of dA, one split, four 2-byte stores (both triangles) — and the A fragments come from ldmatrix;
//   * a sample buffer holds only the F live rows (ldmatrix rows >= F point at a zero row of the CTA); ONE buffer per warp,
//     16 warps per SM: the other warps hide a warp's copy latency.  (Tried and slower: double-buffered rows with the G
//     fragments assembled in registers through a packed offset table, 12 warps at 168 registers: 241 us against 217 us —
//     it is the dependent instruction chains of the compute phase, not the copy latency, that occupancy has to hide.)
// ---------------------------------------------------------------------------------------------------------------
constexpr int PS_WARPS = 16;
constexpr unsigned PS_G_STRIDE = 80;  // bytes per row of a G matrix (64 + 16: conflict-free ldmatrix)
constexpr unsigned PS_G_BYTES = 2 * 32 * PS_G_STRIDE;

__global__ void __launch_bounds__(32 * PS_WARPS, 1)
interact_bwd_ps_kernel(const __grid_constant__ LookupParams lk, const __grid_constant__ IbwdParams p) {
  extern __shared__ __align__(256) uint8_t smem[];
  constexpr int D = 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int F = p.F;
  const int npairs = F * (F - 1) / 2;
  const int OW = p.P + npairs;
  // CTA: [zero row 256 B | pair table] then per warp [F rows of 256 B | dA stage | G hi | G lo]
  const uint32_t zrow = (uint32_t)__cvta_generic_to_shared(smem);
  uint16_t* pair_ij = reinterpret_cast<uint16_t*>(smem + 256);
  uint8_t* mine = smem + p.stage_off + (size_t)warp * p.buf_bytes;  // stage_off: bytes of the CTA-wide header
  const uint32_t xs = (uint32_t)__cvta_generic_to_shared(mine);
  const uint32_t st = xs + (uint32_t)F * 256u;
  const uint32_t gs = st + p.stage_floats * 4u;
  for (int e = threadIdx.x; e < 64; e += blockDim.x) reinterpret_cast<uint32_t*>(smem)[e] = 0u;
  for (int e = lane; e < (int)(p.buf_bytes / 4); e += 32) reinterpret_cast<uint32_t*>(mine)[e] = 0u;  // G diagonal, padding
  for (int e = threadIdx.x; e < npairs; e += blockDim.x) {  // pair e -> (i, j)
    int i = 0, rem = e;
    while (rem >= F - 1 - i) {
      rem -= F - 1 - i;
      ++i;
    }
    pair_ij[e] = (uint16_t)((i << 8) | (i + 1 + rem));
  }
  __syncthreads();

  const bool is_table = lane < F && lane != p.bottom_slot && lk.weights[lane] != nullptr;
  const float* my_base = is_table ? lk.weights[lane] : nullptr;  // mirror rows: 64 "floats" = 256 bytes each
  const unsigned long long my_rows = is_table ? (unsigned long long)lk.rows[lane] : 0ull;
  const int my_w = is_table ? lk.idx_bytes[lane] : 4;
  const void* my_ids = is_table ? lk.indices[lane] : nullptr;
  const int cl = lane & 15, rl = lane >> 4;
  float* gptr[4];
#pragma unroll
  for (int qd = 0; qd < 4; ++qd) {
    const int i = 8 * qd + g;
    gptr[qd] = (i < F && i != p.bottom_slot) ? p.grad[i] : nullptr;
  }
  // ldmatrix lane addresses
  const int q = lane >> 3, r8 = lane & 7;
  // A (G): matrices (i 0-7, j 0-7) (i 8-15, j 0-7) (i 0-7, j 8-15) (i 8-15, j 8-15) of m-tile mt, k-tile kt
  const uint32_t a_lane = (uint32_t)(((q & 1) * 8 + r8) * PS_G_STRIDE + (q >> 1) * 16);
  // B (X): matrices (j 0-7, nt 2u) (j 8-15, nt 2u) (j 0-7, nt 2u+1) (j 8-15, nt 2u+1); chunk nt of row j sits at
  // nt ^ (j & 7); rows >= F read the CTA's zero row
  const int b_nt = q >> 1;
  uint32_t brow[2];
#pragma unroll
  for (int kt = 0; kt < 2; ++kt) {
    const int j = 16 * kt + (q & 1) * 8 + r8;
    brow[kt] = j < F ? xs + (uint32_t)j * 256u : zrow;
  }
  // accumulator row (0..3) of this lane that is the bottom row, or -1
  const int bq = (p.bottom_slot >= 0 && (p.bottom_slot & 7) == g) ? (p.bottom_slot >> 3) : -1;

  const long long stride_s = (long long)gridDim.x * p.n_warps;
  const long long s_first = (long long)blockIdx.x * p.n_warps + warp;
  // Branch-free id fetch (lanes carry ids of different widths: a switch would serialise one global load per width): the
  // aligned 32-bit word(s) holding the id, one sample ahead; decoded with a funnel shift like the forward kernel.
  const uint32_t my_mask = my_w >= 4 ? 0xffffffffu : (0xffffffffu >> (32 - 8 * my_w));
  const bool my_64 = my_w == 8;
  const uint8_t* id_ptr = is_table ? reinterpret_cast<const uint8_t*>(my_ids) + (size_t)s_first * my_w : nullptr;
  const long long id_step = stride_s * my_w;
  uint32_t raw_a = 0, raw_b = 0, raw_sh = 0;
  auto fetch_id = [&](long long s) {
    raw_a = raw_b = raw_sh = 0;
    if (is_table && s < p.B) {
      const uintptr_t ad = reinterpret_cast<uintptr_t>(id_ptr);
      const uint32_t* wp = reinterpret_cast<const uint32_t*>(ad & ~(uintptr_t)3);
      raw_sh = 8u * (uint32_t)(ad & 3);
      raw_a = __ldg(wp);
      if (my_64 || (int)(ad & 3) + my_w > 4) raw_b = __ldg(wp + 1);
    }
    id_ptr += id_step;
  };
  fetch_id(s_first);
  const bool bottom_lane = lane == p.bottom_slot && p.bottom != nullptr;
  for (long long s = s_first; s < p.B; s += stride_s) {
    // ---- rows + dA row -> shared memory
    {
      const uint32_t v = __funnelshift_r(raw_a, raw_b, raw_sh) & my_mask;
      const uint32_t vhi = my_64 ? raw_b : (uint32_t)((int)v >> 31);
      const unsigned long long idx = ((unsigned long long)vhi << 32) | v;
      fetch_id(s + stride_s);  // the next sample's id is in flight while this one is computed
      const float* my_src = (is_table && idx < my_rows) ? my_base + idx * D : bottom_lane ? p.bottom + s * p.bottom_stride : g_zero_row;
      const uint32_t lo = (uint32_t)(uintptr_t)my_src, hi = (uint32_t)((uintptr_t)my_src >> 32);
#pragma unroll
      for (int r0 = 0; r0 < 32; r0 += 2) {  // no branch: rows >= F are shuffled for nothing and their copy is predicated off
        const int row = r0 + rl;
        const uint32_t slo = __shfl_sync(0xffffffffu, lo, row);
        const uint32_t shi = __shfl_sync(0xffffffffu, hi, row);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(((uintptr_t)shi << 32) | slo) + cl * 16;
        cp_async16_if(row < F, xs + (uint32_t)(row * 256 + ((cl ^ (row & 7)) << 4)), src);
      }
      const float* da = p.dA + s * p.dA_stride;
      if (p.dA_vec) {
        for (int c = lane; c * 4 < OW; c += 32) cp_async16_if(true, st + (uint32_t)c * 16u, da + c * 4);
      } else {
        for (int c = lane; c < OW; c += 32) cp_async4_if(true, st + (uint32_t)c * 4u, da + c);
      }
      cp_async_commit();
      cp_async_wait<0>();
      __syncwarp();
    }
    // ---- G (hi, lo) from the pair gradients
#pragma unroll 4
    for (int e = lane; e < npairs; e += 32) {
      const float v = lds32(st + (uint32_t)(p.P + e) * 4u);
      const uint32_t ij = pair_ij[e];
      const uint32_t i = ij >> 8, j = ij & 255u;
      __nv_bfloat16 h, l;
      split_bf16(v, h, l);
      const uint32_t a1 = gs + i * PS_G_STRIDE + j * 2, a2 = gs + j * PS_G_STRIDE + i * 2;
      const unsigned short hb = __bfloat16_as_ushort(h), lb = __bfloat16_as_ushort(l);
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(a1), "h"(hb) : "memory");
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(a2), "h"(hb) : "memory");
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(a1 + 32 * PS_G_STRIDE), "h"(lb) : "memory");
      asm volatile("st.shared.u16 [%0], %1;" ::"r"(a2 + 32 * PS_G_STRIDE), "h"(lb) : "memory");
    }
    __syncwarp();
    float acc[2][8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.0f;
#pragma unroll
    for (int kt = 0; kt < 2; ++kt) {
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const uint32_t a = gs + a_lane + (uint32_t)(mt * 16 * PS_G_STRIDE + kt * 32);
        ldsm_x4(a, ah[mt][0], ah[mt][1], ah[mt][2], ah[mt][3]);
        ldsm_x4(a + 32 * PS_G_STRIDE, al[mt][0], al[mt][1], al[mt][2], al[mt][3]);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        uint32_t bh[4], bl[4];
        const uint32_t b = brow[kt] + (uint32_t)((((2 * u + b_nt) ^ r8) & 7) << 4);
        ldsm_x4_t(b, bh[0], bh[1], bh[2], bh[3]);
        ldsm_x4_t(b + 128u, bl[0], bl[1], bl[2], bl[3]);
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const int nt = 2 * u + v;
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) mma16816(acc[mt][nt], ah[mt], bl[2 * v], bl[2 * v + 1]);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) mma16816(acc[mt][nt], al[mt], bh[2 * v], bh[2 * v + 1]);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) mma16816(acc[mt][nt], ah[mt], bh[2 * v], bh[2 * v + 1]);
        }
      }
    }
    // ---- dX rows.  Table rows: predicated vector stores, no branches (gptr is null for the bottom row and rows >= F)
    const long long goffs = s * p.grad_stride + 2 * t;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* drow = gptr[2 * mt + h] + goffs;
        const uint32_t on = gptr[2 * mt + h] != nullptr;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
          asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %3, 0;\n\t@p st.global.v2.f32 [%0], {%1, %2};\n\t}" ::"l"(drow + 8 * nt),
                       "f"(acc[mt][nt][2 * h]), "f"(acc[mt][nt][2 * h + 1]), "r"(on)
                       : "memory");
      }
    // the bottom row (one accumulator row of the lanes with g == bottom_slot % 8): + shortcut gradient, relu mask
    if (bq >= 0 && p.d_bottom) {
      float* drow = p.d_bottom + s * p.d_bottom_stride + 2 * t;
      const int i = p.bottom_slot;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        float a = bq == 0 ? acc[0][nt][0] : bq == 1 ? acc[0][nt][2] : bq == 2 ? acc[1][nt][0] : acc[1][nt][2];
        float b = bq == 0 ? acc[0][nt][1] : bq == 1 ? acc[0][nt][3] : bq == 2 ? acc[1][nt][1] : acc[1][nt][3];
        if (p.P > 0) {
          a += lds32(st + (uint32_t)(8 * nt + 2 * t) * 4u);
          b += lds32(st + (uint32_t)(8 * nt + 2 * t) * 4u + 4u);
        }
        if (p.mask_bottom) {
          // bottom[d] > 0  <=>  its bf16 hi part > 0 (relu outputs are >= 0; hi = 0 only for denormal-sized values)
          const uint32_t xa = xs + (uint32_t)(i * 256 + (((nt ^ (i & 7)) & 7) << 4) + 4 * t);
          uint32_t hv;
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(hv) : "r"(xa));
          a = __uint_as_float(hv << 16) > 0.0f ? a : 0.0f;
          b = __uint_as_float(hv & 0xffff0000u) > 0.0f ? b : 0.0f;
        }
        *reinterpret_cast<float2*>(drow + 8 * nt) = make_float2(a, b);
      }
    }
    __syncwarp();  // the buffer is refilled by the next iteration's copies
  }
}

static int launch_ibwd_ps(const LookupParams& lk, IbwdParams p, cudaStream_t st) {
  const int npairs = p.F * (p.F - 1) / 2;
  const int OW = p.P + npairs;
  p.stage_floats = (unsigned)(((OW + 3) & ~3) + 4);
  p.stage_off = (256u + (unsigned)npairs * 2u + 255u) & ~255u;  // CTA-wide header: zero row + pair table
  p.buf_bytes = ((unsigned)p.F * 256u + p.stage_floats * 4u + PS_G_BYTES + 15u) & ~15u;
  int warps = (int)((227u * 1024u - p.stage_off) / p.buf_bytes);
  if (warps > PS_WARPS) warps = PS_WARPS;
  if (warps < 1) return MM_ERR_UNSUPPORTED;
  p.n_warps = warps;
  const size_t smem = (size_t)p.stage_off + (size_t)warps * p.buf_bytes;
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(interact_bwd_ps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("mm_dlrm_interact_backward: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
      return (int)e;
    }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  long long want = (p.B + warps - 1) / warps;
  const long long sms = sm_count();
  const unsigned grid = (unsigned)(want < sms ? want : sms);
  interact_bwd_ps_kernel<<<grid, 32 * warps, smem, st>>>(lk, p);
  return check_launch("mm_dlrm_interact_backward");
}

// ---------------------------------------------------------------------------------------------------------------
// Sparse rows: dedup + optimizer
// ---------------------------------------------------------------------------------------------------------------
struct SparseTable {
  float* w;
  long long rows;
  const void* ids;
  int idx_bytes;
  float* grad;  // (B, D) slice values (duplicates are folded into the representative's slice)
  int* rep;     // (rows,) int32, INT_MAX when idle
  float* s1;    // Adagrad accumulator / Adam m
  float* s2;    // Adam v
  __nv_bfloat16* mirror;  // operand-format copy of the table (rows, 2D) [hi | lo] or null
  float* dense;           // (rows, D) gradient accumulator, all zero between calls, or null (election path)
};
struct SparseParams {
  SparseTable t[MM_LOOKUP_MAX_ROWS];
  long long B;
  int D;
  int lgL;  // ceil(log2(D / 4)): lanes per row, those past D/4 idle (a 64-bit division by a runtime value costs ~100 instructions and the XU pipe)
  int opt;
  const float* hyper;  // device: see mm_b200.h MM_HYPER_*
  int n;                                       // tables in t[]
  long long row_start[MM_LOOKUP_MAX_ROWS + 1];  // dense path: prefix sums of the tables' row counts
};

__global__ void sparse_elect_kernel(const __grid_constant__ SparseParams p) {
  const SparseTable& tb = p.t[blockIdx.y];
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  const unsigned long long id = (unsigned long long)load_id(tb.ids, tb.idx_bytes, b);
  if (id < (unsigned long long)tb.rows) atomicMin(tb.rep + id, (int)b);
}

__device__ __forceinline__ void red_add_v4(float* addr, const float4& v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Tables on the election path have rows >> batch: a sample is rarely a duplicate (2-13 % for the Criteo tables of 0.2-10 M
// rows).  One THREAD per (sample, table) tests the map; the warp then folds its duplicates one after the other, all 32
// lanes moving one slice (first version: D/4 lanes per sample all loading id and map entry — 16x the threads, 42 us).
__global__ void sparse_fold_kernel(const __grid_constant__ SparseParams p) {
  const SparseTable& tb = p.t[blockIdx.y];
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  int r = -1;
  if (b < p.B) {
    const unsigned long long id = (unsigned long long)load_id(tb.ids, tb.idx_bytes, b);
    if (id < (unsigned long long)tb.rows) {
      const int rep = tb.rep[id];
      if (rep != (int)b) r = rep;
    }
  }
  unsigned todo = __ballot_sync(0xffffffffu, r >= 0);
  const int n4 = p.D >> 2;  // float4 per slice
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const long long bs = __shfl_sync(0xffffffffu, b, src);
    const int rs = __shfl_sync(0xffffffffu, r, src);
    for (int c = lane; c < n4; c += 32) {
      const float4 v = *reinterpret_cast<const float4*>(tb.grad + bs * p.D + 4 * c);
      red_add_v4(tb.grad + (long long)rs * p.D + 4 * c, v);
    }
  }
}

struct Hyper {
  float lr, b1, b2, eps, lr_t;
};
__device__ __forceinline__ Hyper load_hyper(const float* hy) {
  Hyper h;
  h.lr = __ldg(hy + MM_HYPER_LR);
  h.b1 = __ldg(hy + MM_HYPER_BETA1);
  h.b2 = __ldg(hy + MM_HYPER_BETA2);
  h.eps = __ldg(hy + MM_HYPER_EPS);
  h.lr_t = __ldg(hy + MM_HYPER_LR_T);
  return h;
}
__device__ __forceinline__ float upd(int opt, float w, float g, float& s1, float& s2, const Hyper& h) {
  if (opt == MM_OPT_SGD) return w - h.lr * g;
  if (opt == MM_OPT_ADAGRAD) {
    s1 += g * g;
    return w - h.lr * g / (sqrtf(s1) + h.eps);
  }
  // Adam (Keras: lr_t = lr sqrt(1 - b2^t) / (1 - b1^t), computed by mm_opt_tick)
  s1 = h.b1 * s1 + (1.0f - h.b1) * g;
  s2 = h.b2 * s2 + (1.0f - h.b2) * g * g;
  return w - h.lr_t * s1 / (sqrtf(s2) + h.eps);
}

__global__ void sparse_apply_kernel(const __grid_constant__ SparseParams p) {
  const SparseTable& tb = p.t[blockIdx.y];
  const long long b = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> p.lgL;
  const int c = threadIdx.x & ((1 << p.lgL) - 1);
  if (b >= p.B || c >= (p.D >> 2)) return;
  const unsigned long long id = (unsigned long long)load_id(tb.ids, tb.idx_bytes, b);
  if (id >= (unsigned long long)tb.rows) return;
  // The row and its slots are requested TOGETHER with the map entry (one dependent round trip less: id -> {map, row});
  // for tables on this path nearly every sample is its id's representative, so almost nothing is fetched in vain.
  // Every lane of the group reads the map BEFORE lane 0 resets it (the group sits inside one warp: D/4 <= 32).
  const long long off = (long long)id * p.D + 4 * c;
  const int r = tb.rep[id];
  const float4 g = *reinterpret_cast<const float4*>(tb.grad + b * p.D + 4 * c);
  float4 w = *reinterpret_cast<float4*>(tb.w + off);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), v = a;
  if (p.opt != MM_OPT_SGD) a = *reinterpret_cast<float4*>(tb.s1 + off);
  if (p.opt == MM_OPT_ADAM) v = *reinterpret_cast<float4*>(tb.s2 + off);
  __syncwarp();
  if (r != (int)b) return;
  const Hyper hy = load_hyper(p.hyper);
  w.x = upd(p.opt, w.x, g.x, a.x, v.x, hy);
  w.y = upd(p.opt, w.y, g.y, a.y, v.y, hy);
  w.z = upd(p.opt, w.z, g.z, a.z, v.z, hy);
  w.w = upd(p.opt, w.w, g.w, a.w, v.w, hy);
  *reinterpret_cast<float4*>(tb.w + off) = w;
  if (p.opt != MM_OPT_SGD) *reinterpret_cast<float4*>(tb.s1 + off) = a;
  if (p.opt == MM_OPT_ADAM) *reinterpret_cast<float4*>(tb.s2 + off) = v;
  if (tb.mirror) {
    uint32_t h0, l0, h1, l1;
    split_pair(w.x, w.y, h0, l0);
    split_pair(w.z, w.w, h1, l1);
    __nv_bfloat16* m = tb.mirror + (long long)id * 2 * p.D + 4 * c;
    *reinterpret_cast<uint2*>(m) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(m + p.D) = make_uint2(l0, l1);
  }
  if (c == 0) tb.rep[id] = INT_MAX;
}

// ---- tables with few rows: the duplicates of an id are the norm, not the exception (a 4-row table sees every id 16 000 times
// per batch) and folding them through global atomics serialises on a handful of cache lines (first version: 0.87 ms of a
// 1.9 ms step).  Such tables accumulate into a dense (rows, D) gradient instead: `rep` is only a touched flag.
//   small (rows <= 1024): a CTA sorts its 2 048 samples by row and sums runs of equal rows in registers (below);
//   mid:   vector reds straight into the dense accumulator (tens of duplicates per row at most).
// Shared-memory fp32 atomics are compare-and-swap loops: summing 1 024 slices per CTA that way cost 160 us for the 8 tiny
// Criteo tables.  Instead the CTA counting-sorts its chunk of samples by row with INTEGER shared atomics (native), then
// every group of D/4 lanes walks a contiguous piece of the sorted order, sums runs of equal rows in registers and
// emits ONE vector red per run: rows + groups reds per CTA instead of one shared atomic per element.
constexpr int SMALL_CHUNK = 1024;     // samples per CTA
constexpr int SMALL_MAX_ROWS = 1024;  // rows of a "small" table (counter array in shared memory)
__global__ void __launch_bounds__(256) sparse_scatter_small_kernel(const __grid_constant__ SparseParams p) {
  __shared__ int cnt[SMALL_MAX_ROWS + 1];
  __shared__ unsigned short order[SMALL_CHUNK], orow[SMALL_CHUNK];
  __shared__ int scan_tmp[256];
  const SparseTable& tb = p.t[blockIdx.y];
  const int rows = (int)tb.rows;
  const long long b0 = (long long)blockIdx.x * SMALL_CHUNK;
  const int n = (int)min((long long)SMALL_CHUNK, p.B - b0);
  if (n <= 0) return;
  for (int r = threadIdx.x; r <= rows; r += blockDim.x) cnt[r] = 0;
  __syncthreads();
  constexpr int PER = SMALL_CHUNK / 256;
  int my_row[PER], my_pos[PER];
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int i = threadIdx.x + k * 256;
    my_row[k] = -1;
    if (i < n) {
      const unsigned long long id = (unsigned long long)load_id(tb.ids, tb.idx_bytes, b0 + i);
      if (id < (unsigned long long)rows) {
        my_row[k] = (int)id;
        my_pos[k] = atomicAdd(&cnt[id], 1);
      }
    }
  }
  __syncthreads();
  // exclusive scan of cnt[0..rows): each thread owns a contiguous span of rows
  {
    const int span = (rows + 255) / 256;
    const int r0 = threadIdx.x * span;
    int s = 0;
    for (int r = r0; r < min(rows, r0 + span); ++r) s += cnt[r];
    scan_tmp[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      int run = 0;
      for (int t = 0; t < 256; ++t) {
        const int v = scan_tmp[t];
        scan_tmp[t] = run;
        run += v;
      }
      cnt[rows] = run;  // number of valid samples
    }
    __syncthreads();
    int run = scan_tmp[threadIdx.x];
    for (int r = r0; r < min(rows, r0 + span); ++r) {
      const int v = cnt[r];
      cnt[r] = run;
      run += v;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < PER; ++k)
    if (my_row[k] >= 0) {
      const int at = cnt[my_row[k]] + my_pos[k];
      order[at] = (unsigned short)(threadIdx.x + k * 256);
      orow[at] = (unsigned short)my_row[k];
    }
  __syncthreads();
  const int valid = cnt[rows];
  const int c = threadIdx.x & ((1 << p.lgL) - 1), grp = threadIdx.x >> p.lgL, ngrp = blockDim.x >> p.lgL;
  if (c >= (p.D >> 2)) return;  // lanes past D/4 of a group (no barrier follows)
  const int per = (valid + ngrp - 1) / ngrp;
  const int k0 = grp * per, k1 = min(valid, k0 + per);
  int cur = -1;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  constexpr int U = 8;  // slices in flight per group (their addresses come from the sorted order: no prefetcher helps)
  for (int k = k0; k < k1; k += U) {
    int r[U];
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const bool on = k + u < k1;
      r[u] = on ? (int)orow[k + u] : -1;
      v[u] = on ? *reinterpret_cast<const float4*>(tb.grad + (b0 + order[k + u]) * p.D + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (r[u] < 0) continue;
      if (r[u] != cur) {
        if (cur >= 0) {
          red_add_v4(tb.dense + (long long)cur * p.D + 4 * c, acc);
          if (c == 0) tb.rep[cur] = 0;  // touched
        }
        cur = r[u];
        acc = v[u];
      } else {
        acc.x += v[u].x;
        acc.y += v[u].y;
        acc.z += v[u].z;
        acc.w += v[u].w;
      }
    }
  }
  if (cur >= 0) {
    red_add_v4(tb.dense + (long long)cur * p.D + 4 * c, acc);
    if (c == 0) tb.rep[cur] = 0;
  }
}

__global__ void sparse_scatter_mid_kernel(const __grid_constant__ SparseParams p) {
  const SparseTable& tb = p.t[blockIdx.y];
  const long long b = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> p.lgL;
  const int c = threadIdx.x & ((1 << p.lgL) - 1);
  if (b >= p.B || c >= (p.D >> 2)) return;
  const unsigned long long id = (unsigned long long)load_id(tb.ids, tb.idx_bytes, b);
  if (id >= (unsigned long long)tb.rows) return;
  const float4 v = *reinterpret_cast<const float4*>(tb.grad + b * p.D + 4 * c);
  red_add_v4(tb.dense + id * p.D + 4 * c, v);
  if (c == 0) tb.rep[id] = 0;
}

// one group of D/4 lanes per ROW of a dense-path table (rows of all such tables form one flattened index space: row_start
// holds the prefix sums): touched rows are updated from the accumulator, which is cleared
__global__ void sparse_apply_dense_kernel(const __grid_constant__ SparseParams p) {
  const long long fr = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> p.lgL;
  const int c = threadIdx.x & ((1 << p.lgL) - 1);
  if (fr >= p.row_start[p.n] || c >= (p.D >> 2)) return;
  int t = 0;
  while (fr >= p.row_start[t + 1]) ++t;
  const SparseTable& tb = p.t[t];
  const long long row = fr - p.row_start[t];
  // flag, accumulator, row and slots are requested together (tables on this path have nearly all rows touched)
  const long long off = row * p.D + 4 * c;
  const int flag = tb.rep[row];
  const float4 g = *reinterpret_cast<const float4*>(tb.dense + off);
  float4 w = *reinterpret_cast<float4*>(tb.w + off);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), v = a;
  if (p.opt != MM_OPT_SGD) a = *reinterpret_cast<float4*>(tb.s1 + off);
  if (p.opt == MM_OPT_ADAM) v = *reinterpret_cast<float4*>(tb.s2 + off);
  __syncwarp();
  if (flag != 0) return;
  *reinterpret_cast<float4*>(tb.dense + off) = make_float4(0.f, 0.f, 0.f, 0.f);
  const Hyper hy = load_hyper(p.hyper);
  w.x = upd(p.opt, w.x, g.x, a.x, v.x, hy);
  w.y = upd(p.opt, w.y, g.y, a.y, v.y, hy);
  w.z = upd(p.opt, w.z, g.z, a.z, v.z, hy);
  w.w = upd(p.opt, w.w, g.w, a.w, v.w, hy);
  *reinterpret_cast<float4*>(tb.w + off) = w;
  if (p.opt != MM_OPT_SGD) *reinterpret_cast<float4*>(tb.s1 + off) = a;
  if (p.opt == MM_OPT_ADAM) *reinterpret_cast<float4*>(tb.s2 + off) = v;
  if (tb.mirror) {
    uint32_t h0, l0, h1, l1;
    split_pair(w.x, w.y, h0, l0);
    split_pair(w.z, w.w, h1, l1);
    __nv_bfloat16* m = tb.mirror + row * 2 * p.D + 4 * c;
    *reinterpret_cast<uint2*>(m) = make_uint2(h0, h1);
    *reinterpret_cast<uint2*>(m + p.D) = make_uint2(l0, l1);
  }
  if (c == 0) tb.rep[row] = INT_MAX;
}

__global__ void dense_apply_kernel(int opt, float* __restrict__ w, float* __restrict__ g, float* __restrict__ s1,
                                   float* __restrict__ s2, long long n, const float* __restrict__ hyper, float grad_scale) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const Hyper hy = load_hyper(hyper);
  for (; i < n; i += stride) {
    float a = opt != MM_OPT_SGD ? s1[i] : 0.0f, v = opt == MM_OPT_ADAM ? s2[i] : 0.0f;
    w[i] = upd(opt, w[i], g[i] * grad_scale, a, v, hy);
    if (opt != MM_OPT_SGD) s1[i] = a;
    if (opt == MM_OPT_ADAM) s2[i] = v;
    g[i] = 0.0f;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Bag backward: the IndexedSlices values of a pooled (multi-hot) feature, out[i] = scale(bag(i)) * g[bag(i)].
// One warp per task; tasks 0..B-1 are the bags.  Ragged form: a bag is [off[b], off[b+1]) clamped to [0, nnz] (empty when
// decreasing), task B zero-fills [0, off[0]) and task B+1 [off[B], nnz).  Every position lies in one of these ranges
// (the first b with off[b+1] > i brackets i), so all nnz rows are written whatever the offsets hold.  Per bag: g[b] is
// read once (one float4 per lane), the ids are read 32 at a time (coalesced) for the count, then D/4 lanes per row
// write 32/(D/4) rows per vector store, zero where the id is outside [0, rows).  out_ids (nullable) receives the id of
// every row that carries a gradient and -1 for the others (uncovered positions, ids outside [0, rows)): the indices of
// the sparse update, which skips -1.
// ---------------------------------------------------------------------------------------------------------------
template <typename IT, typename OT, int D>
__global__ void __launch_bounds__(256)
bag_grad_rows_kernel(const float* __restrict__ g, long long g_stride, const IT* __restrict__ ids, const OT* __restrict__ offsets,
                     int L, long long B, long long nnz, long long rows, int combiner, float* __restrict__ out,
                     IT* __restrict__ out_ids) {
  constexpr int LR = D / 4;   // lanes per row
  constexpr int R = 32 / LR;  // rows per store instruction
  const int lane = threadIdx.x & 31, c = lane % LR, rl = lane / LR;
  const long long n_tasks = offsets ? B + 2 : B;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  auto clampn = [nnz](long long v) { return v < 0 ? 0 : (v > nnz ? nnz : v); };
  for (long long task = warp0; task < n_tasks; task += n_warps) {
    long long beg, end;
    const bool zero = task >= B;
    if (!offsets) {
      beg = task * L;
      end = beg + L;
    } else if (task < B) {
      beg = clampn((long long)offsets[task]);
      end = clampn((long long)offsets[task + 1]);
    } else if (task == B) {
      beg = 0;
      end = clampn((long long)offsets[0]);
    } else {
      beg = clampn((long long)offsets[B]);
      end = nnz;
    }
    if (beg >= end) continue;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!zero) {
      v = *reinterpret_cast<const float4*>(g + task * g_stride + 4 * c);
      if (combiner != MM_COMBINER_SUM) {
        float den = (float)L;  // fixed length: mean over all L positions, padding not masked
        if (offsets) {
          int cnt = 0;  // the ids gather_bag_kernel sums: those in [0, rows)
          for (long long i = beg; i < end; i += 32) {
            const long long id = i + lane < end ? (long long)ids[i + lane] : -1;
            cnt += __popc(__ballot_sync(0xffffffffu, id >= 0 && id < rows));
          }
          den = combiner == MM_COMBINER_SQRTN ? sqrtf((float)cnt) : (float)cnt;
        }
        if (den > 0.0f) {
          v.x = __fdiv_rn(v.x, den);
          v.y = __fdiv_rn(v.y, den);
          v.z = __fdiv_rn(v.z, den);
          v.w = __fdiv_rn(v.w, den);
        }
      }
    }
    for (long long i = beg; i < end; i += 32) {
      const int lim = (int)(end - i < 32 ? end - i : 32);  // positions of this chunk
      const long long id = (!zero && lane < lim) ? (long long)ids[i + lane] : -1;
      const bool mine = id >= 0 && id < rows;
      const unsigned ok = __ballot_sync(0xffffffffu, mine);
      if (out_ids && lane < lim) out_ids[i + lane] = mine ? (IT)id : (IT)-1;
      float* dst = out + (i + rl) * D + 4 * c;
#pragma unroll
      for (int r = 0; r < 32; r += R) {
        const int k = r + rl;
        const bool on = (ok >> k) & 1u;
        if (k < lim) *reinterpret_cast<float4*>(dst + r * D) = make_float4(on ? v.x : 0.f, on ? v.y : 0.f, on ? v.z : 0.f, on ? v.w : 0.f);
      }
    }
  }
}

template <typename IT, typename OT>
static void launch_bag_grad(unsigned blocks, cudaStream_t st, const float* g, long long g_stride, const void* ids, const void* offsets,
                            int L, long long B, long long nnz, long long rows, int combiner, int D, float* out, void* out_ids) {
  const IT* i = reinterpret_cast<const IT*>(ids);
  IT* oi = reinterpret_cast<IT*>(out_ids);
  const OT* o = reinterpret_cast<const OT*>(offsets);
  switch (D) {
    case 16: bag_grad_rows_kernel<IT, OT, 16><<<blocks, 256, 0, st>>>(g, g_stride, i, o, L, B, nnz, rows, combiner, out, oi); break;
    case 32: bag_grad_rows_kernel<IT, OT, 32><<<blocks, 256, 0, st>>>(g, g_stride, i, o, L, B, nnz, rows, combiner, out, oi); break;
    case 64: bag_grad_rows_kernel<IT, OT, 64><<<blocks, 256, 0, st>>>(g, g_stride, i, o, L, B, nnz, rows, combiner, out, oi); break;
    default: bag_grad_rows_kernel<IT, OT, 128><<<blocks, 256, 0, st>>>(g, g_stride, i, o, L, B, nnz, rows, combiner, out, oi); break;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Wide kernel of DeepFM (mm_wide_rows_apply): a (sum of cardinalities + n_cont, 1) Keras kernel whose feature blocks are
// disjoint row ranges; every block's gradient values are the one (B,) vector g (dloss/ds), so no (B, T) slice array exists.
// Scatter (blockIdx.y = block, CTAs stride chunks of WIDE_CHUNK samples): the lanes of a warp holding the same row are
// found with match.any and summed by their leader, which adds ONE value per row and warp:
//   small blocks (rows <= WIDE_SMALL_ROWS): into a per-CTA shared accumulator, flushed with one global add per touched row
//     and CTA at the end (a 4-row Criteo feature is hit 16 000 times per batch);
//   other blocks: straight into the (rows,) accumulator `acc`, and atomicMin(rep[row], b) elects the smallest sample.
// Apply: blocks of <= WIDE_DENSE_ROWS rows walk their rows (rep != INT_MAX marks a touched row); larger blocks walk the
// samples and the elected sample updates its row.  Either clears acc and rep.  The continuous rows and the bias are
// touched by every step and take the dense rule (wide_dense_apply_kernel).
// ---------------------------------------------------------------------------------------------------------------
constexpr int WIDE_MAX_BLOCKS = 64;
constexpr int WIDE_CHUNK = 2048;
constexpr int WIDE_SMALL_ROWS = 2048;
constexpr long long WIDE_DENSE_ROWS = 131072;
constexpr int WIDE_MAX_DENSE = 64;
struct WideBlock {
  const void* ids;
  long long rows;
  long long off;
  int idx_bytes;
};
struct WideParams {
  WideBlock blk[WIDE_MAX_BLOCKS];
  long long dense_off[WIDE_MAX_DENSE];
  int n_dense;
  float* w;
  float* s1;
  float* s2;
  float* acc;
  int* rep;
  const float* g;
  float* dgrad;  // (n_dense [+ 1 for the bias],)
  float* bias;
  float* bs1;
  float* bs2;
  long long B;
  int opt;
  const float* hyper;
};

__global__ void __launch_bounds__(256) wide_scatter_kernel(const __grid_constant__ WideParams p) {
  __shared__ float sacc[WIDE_SMALL_ROWS];
  __shared__ int stouch[WIDE_SMALL_ROWS];
  const WideBlock& bk = p.blk[blockIdx.y];
  const bool small = bk.rows <= WIDE_SMALL_ROWS;
  const int lane = threadIdx.x & 31;
  if (small) {
    for (int r = threadIdx.x; r < bk.rows; r += blockDim.x) {
      sacc[r] = 0.0f;
      stouch[r] = 0;
    }
    __syncthreads();
  }
  const long long n_chunks = (p.B + WIDE_CHUNK - 1) / WIDE_CHUNK;
  for (long long ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    for (int i = 0; i < WIDE_CHUNK; i += 256) {  // uniform trip count: every lane reaches match.any
      const long long b = ch * WIDE_CHUNK + i + threadIdx.x;
      long long row = -1;
      float v = 0.0f;
      if (b < p.B) {
        const unsigned long long id = (unsigned long long)load_id(bk.ids, bk.idx_bytes, b);
        if (id < (unsigned long long)bk.rows) {
          row = (long long)id;
          v = p.g[b];
        }
      }
      const unsigned grp = __match_any_sync(0xffffffffu, (unsigned long long)row);
      if (row < 0) continue;
      float s = 0.0f;
      for (unsigned m = grp; m; m &= m - 1) s += __shfl_sync(grp, v, __ffs(m) - 1);
      if (lane != __ffs(grp) - 1) continue;
      if (small) {
        atomicAdd(&sacc[row], s);
        stouch[row] = 1;
      } else {
        atomicAdd(p.acc + bk.off + row, s);
        atomicMin(p.rep + bk.off + row, (int)b);  // the leader is the group's smallest sample
      }
    }
  }
  if (small) {
    __syncthreads();
    for (int r = threadIdx.x; r < bk.rows; r += blockDim.x)
      if (stouch[r]) {
        atomicAdd(p.acc + bk.off + r, sacc[r]);
        atomicMin(p.rep + bk.off + r, 0);
      }
  }
}

__device__ __forceinline__ void wide_update(int opt, float* w, float* s1, float* s2, float g, const Hyper& hy) {
  float a = opt != MM_OPT_SGD ? *s1 : 0.0f, v = opt == MM_OPT_ADAM ? *s2 : 0.0f;
  *w = upd(opt, *w, g, a, v, hy);
  if (opt != MM_OPT_SGD) *s1 = a;
  if (opt == MM_OPT_ADAM) *s2 = v;
}

__global__ void __launch_bounds__(256) wide_apply_kernel(const __grid_constant__ WideParams p) {
  const WideBlock& bk = p.blk[blockIdx.y];
  const Hyper hy = load_hyper(p.hyper);
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if (bk.rows <= WIDE_DENSE_ROWS) {
    for (long long r = t0; r < bk.rows; r += stride) {
      const long long i = bk.off + r;
      if (p.rep[i] == INT_MAX) continue;
      wide_update(p.opt, p.w + i, p.s1 + i, p.s2 + i, p.acc[i], hy);
      p.acc[i] = 0.0f;
      p.rep[i] = INT_MAX;
    }
  } else {
    for (long long b = t0; b < p.B; b += stride) {
      const unsigned long long id = (unsigned long long)load_id(bk.ids, bk.idx_bytes, b);
      if (id >= (unsigned long long)bk.rows) continue;
      const long long i = bk.off + (long long)id;
      if (p.rep[i] != (int)b) continue;  // another sample holds the row (or already updated it: INT_MAX)
      wide_update(p.opt, p.w + i, p.s1 + i, p.s2 + i, p.acc[i], hy);
      p.acc[i] = 0.0f;
      p.rep[i] = INT_MAX;
    }
  }
}

// the continuous columns' rows and the bias: one thread each
__global__ void wide_dense_apply_kernel(const __grid_constant__ WideParams p) {
  const int t = threadIdx.x;
  const Hyper hy = load_hyper(p.hyper);
  if (t < p.n_dense) {
    const long long i = p.dense_off[t];
    wide_update(p.opt, p.w + i, p.s1 + i, p.s2 + i, p.dgrad[t], hy);
    p.dgrad[t] = 0.0f;
  } else if (t == p.n_dense && p.bias) {
    wide_update(p.opt, p.bias, p.bs1, p.bs2, p.dgrad[t], hy);
    p.dgrad[t] = 0.0f;
  }
}

__global__ void opt_tick_kernel(float* hyper) {
  const float t = hyper[MM_HYPER_STEP] + 1.0f;
  hyper[MM_HYPER_STEP] = t;
  const float b1 = hyper[MM_HYPER_BETA1], b2 = hyper[MM_HYPER_BETA2];
  hyper[MM_HYPER_LR_T] = hyper[MM_HYPER_LR] * sqrtf(1.0f - powf(b2, t)) / (1.0f - powf(b1, t));
}

// lr(s) of a K25 schedule, in fp32 and in the order of operations of tf.keras.optimizers.schedules (TF 2.9-2.12).
__device__ float schedule_lr(const float* sc, float s, float lr) {
  const int kind = (int)sc[MM_SCHED_KIND];
  const float init = sc[MM_SCHED_INIT], ds = sc[MM_SCHED_DECAY_STEPS], rate = sc[MM_SCHED_RATE];
  const bool flag = sc[MM_SCHED_FLAG] != 0.0f;
  switch (kind) {
    case MM_SCHED_EXPONENTIAL: {
      float p = s / ds;
      if (flag) p = floorf(p);
      return init * powf(rate, p);
    }
    case MM_SCHED_INVERSE_TIME: {
      float p = s / ds;
      if (flag) p = floorf(p);
      return init / (1.0f + rate * p);
    }
    case MM_SCHED_POLYNOMIAL: {
      float d = ds, sp = s;
      if (flag) {
        d = ds * (s == 0.0f ? 1.0f : ceilf(s / ds));
      } else {
        sp = fminf(s, ds);
      }
      return (init - rate) * powf(1.0f - sp / d, sc[MM_SCHED_POWER]) + rate;
    }
    case MM_SCHED_COSINE: {
      const float frac = fminf(s, ds) / ds;
      const float cd = 0.5f * (1.0f + cosf(3.14159265358979323846f * frac));
      return init * ((1.0f - rate) * cd + rate);
    }
    case MM_SCHED_PIECEWISE: {
      const int nb = (int)sc[MM_SCHED_NB];
      if (nb < 1 || nb > MM_SCHED_MAX_BOUNDARIES) return lr;
      int i = 0;
      while (i < nb && s > sc[MM_SCHED_BOUNDARIES + i]) ++i;
      return sc[MM_SCHED_VALUES + i];
    }
    default:
      return lr;
  }
}

__global__ void opt_tick_schedule_kernel(float* hyper, const float* sched) {
  const float s = hyper[MM_HYPER_STEP];
  const float lr = schedule_lr(sched, s, hyper[MM_HYPER_LR]);
  hyper[MM_HYPER_LR] = lr;
  const float t = s + 1.0f;
  hyper[MM_HYPER_STEP] = t;
  const float b1 = hyper[MM_HYPER_BETA1], b2 = hyper[MM_HYPER_BETA2];
  hyper[MM_HYPER_LR_T] = lr * sqrtf(1.0f - powf(b2, t)) / (1.0f - powf(b1, t));
}

__global__ void fill_i32_kernel(int* p, long long n, int v) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

}  // namespace trs
}  // namespace mm

extern "C" {

int mm_dlrm_interact_backward(const mm_lookup_table* tables_host, int n_tables, int64_t B, int D, const float* bottom,
                              int64_t bottom_stride, int bottom_slot, int P, const float* dA, int64_t dA_stride,
                              float* const* grad_rows_host, int64_t grad_stride, float* d_bottom, int64_t d_bottom_stride,
                              int mask_bottom, int row_format, void* stream) {
  using namespace mm;
  using namespace mm::trs;
  MM_REQUIRE(tables_host && n_tables > 0 && dA && grad_rows_host && B >= 0, MM_ERR_ARG, "mm_dlrm_interact_backward: null pointer");
  const int F = n_tables + (bottom ? 1 : 0);
  MM_REQUIRE(F >= 2 && F <= MM_LOOKUP_MAX_ROWS, MM_ERR_UNSUPPORTED, "mm_dlrm_interact_backward: F=%d outside [2, 32]", F);
  MM_REQUIRE(D == 16 || D == 32 || D == 64 || D == 128, MM_ERR_UNSUPPORTED, "mm_dlrm_interact_backward: D=%d not in {16,32,64,128}", D);
  MM_REQUIRE(P == 0 || (P == D && bottom), MM_ERR_ARG, "mm_dlrm_interact_backward: P must be 0 or D (with a bottom vector)");
  MM_REQUIRE(row_format == MM_ROWS_F32 || (row_format == MM_ROWS_OPERAND && D == 64), MM_ERR_UNSUPPORTED,
             "mm_dlrm_interact_backward: operand-format rows need D = 64");
  MM_REQUIRE(!bottom || (bottom_slot >= 0 && bottom_slot < F && bottom_stride >= D && (bottom_stride & 3) == 0 && ((uintptr_t)bottom & 15) == 0),
             MM_ERR_ARG, "mm_dlrm_interact_backward: bad bottom slot / stride / alignment");
  const int OW = P + F * (F - 1) / 2;
  MM_REQUIRE(dA_stride >= OW, MM_ERR_ARG, "mm_dlrm_interact_backward: dA_stride < %d", OW);
  MM_REQUIRE(grad_stride >= D && (grad_stride & 1) == 0, MM_ERR_ARG, "mm_dlrm_interact_backward: grad_stride must be even and >= D");
  MM_REQUIRE(!d_bottom || (d_bottom_stride >= D && (d_bottom_stride & 1) == 0 && ((uintptr_t)d_bottom & 7) == 0), MM_ERR_ALIGN,
             "mm_dlrm_interact_backward: d_bottom needs an even stride >= D and 8-byte alignment");
  if (B == 0) return MM_OK;
  LookupParams lk;
  memset(&lk, 0, sizeof(lk));
  lk.world = 1;
  IbwdParams p;
  memset(&p, 0, sizeof(p));
  if (const int rc = fill_lookup_params("mm_dlrm_interact_backward", tables_host, n_tables, F, bottom ? bottom_slot : -1, 0, false, lk))
    return rc;
  for (int i = 0; i < n_tables; ++i) {
    float* gr = grad_rows_host[i];
    MM_REQUIRE(!gr || ((uintptr_t)gr & 7) == 0, MM_ERR_ALIGN, "mm_dlrm_interact_backward: grad_rows[%d] must be 8-byte aligned", i);
    p.grad[tables_host[i].slot] = gr;
  }
  p.B = B;
  p.F = F;
  p.P = P;
  p.bottom_slot = bottom ? bottom_slot : -1;
  p.bottom = bottom;
  p.bottom_stride = bottom_stride;
  p.dA = dA;
  p.dA_stride = dA_stride;
  p.dA_vec = ((dA_stride & 3) == 0 && ((uintptr_t)dA & 15) == 0 && dA_stride >= ((OW + 3) & ~3)) ? 1 : 0;
  p.d_bottom = d_bottom;
  p.d_bottom_stride = d_bottom_stride;
  p.mask_bottom = mask_bottom;
  p.grad_stride = grad_stride;
  cudaStream_t st = (cudaStream_t)stream;
  if (row_format == MM_ROWS_OPERAND) return launch_ibwd_ps(lk, p, st);
  switch (D) {
    case 16: return launch_ibwd<16>(lk, p, st);
    case 32: return launch_ibwd<32>(lk, p, st);
    case 64: return launch_ibwd<64>(lk, p, st);
    default: return launch_ibwd<128>(lk, p, st);
  }
}

int mm_sparse_rows_apply(const mm_sparse_table* tables_host, int n_tables, int64_t B, int D, int opt, const float* hyper,
                         void* stream) {
  using namespace mm;
  using namespace mm::trs;
  MM_REQUIRE(tables_host && n_tables > 0 && n_tables <= MM_LOOKUP_MAX_ROWS && hyper && B >= 0, MM_ERR_ARG,
             "mm_sparse_rows_apply: null pointer or n_tables outside [1, %d]", MM_LOOKUP_MAX_ROWS);
  // a row is a group of L = next power of two >= D/4 lanes (one float4 each) inside one warp; lanes past D/4 are idle
  MM_REQUIRE(D >= 4 && D <= 128 && (D & 3) == 0, MM_ERR_UNSUPPORTED, "mm_sparse_rows_apply: D=%d (needs D %% 4 == 0, 4 <= D <= 128)", D);
  MM_REQUIRE(opt == MM_OPT_SGD || opt == MM_OPT_ADAGRAD || opt == MM_OPT_ADAM, MM_ERR_ARG, "mm_sparse_rows_apply: unknown optimizer %d", opt);
  MM_REQUIRE(B < (int64_t)INT_MAX, MM_ERR_UNSUPPORTED, "mm_sparse_rows_apply: batch too large for the int32 representative map");
  if (B == 0) return MM_OK;
  // three classes: election path (no dense accumulator), dense path small (private copy fits shared memory) / mid
  SparseParams pb, ps, pm, pd;
  memset(&pb, 0, sizeof(pb));
  memset(&ps, 0, sizeof(ps));
  memset(&pm, 0, sizeof(pm));
  memset(&pd, 0, sizeof(pd));
  int nb = 0, ns = 0, nm = 0, nd = 0;
  for (int i = 0; i < n_tables; ++i) {
    const mm_sparse_table& s = tables_host[i];
    MM_REQUIRE(s.weights && s.indices && s.grad_rows && s.rep_map && s.rows > 0, MM_ERR_ARG, "mm_sparse_rows_apply: table %d: null pointer", i);
    MM_REQUIRE(opt == MM_OPT_SGD || s.state1, MM_ERR_ARG, "mm_sparse_rows_apply: table %d: optimizer state missing", i);
    MM_REQUIRE(opt != MM_OPT_ADAM || s.state2, MM_ERR_ARG, "mm_sparse_rows_apply: table %d: second optimizer state missing", i);
    MM_REQUIRE(!s.mirror || D == 64, MM_ERR_ARG, "mm_sparse_rows_apply: table %d: an operand mirror needs D = 64", i);
    MM_REQUIRE((((uintptr_t)s.weights | (uintptr_t)s.grad_rows | (uintptr_t)s.state1 | (uintptr_t)s.state2 | (uintptr_t)s.dense_grad) & 15) == 0,
               MM_ERR_ALIGN, "mm_sparse_rows_apply: table %d: 16-byte alignment", i);
    if (const int rc = check_id_column("mm_sparse_rows_apply", i, s.indices, s.idx_bytes, s.rows)) return rc;
    SparseTable t;
    t.w = s.weights;
    t.rows = s.rows;
    t.ids = s.indices;
    t.idx_bytes = s.idx_bytes;
    t.grad = s.grad_rows;
    t.rep = s.rep_map;
    t.s1 = s.state1;
    t.s2 = s.state2;
    t.mirror = (__nv_bfloat16*)s.mirror;
    t.dense = s.dense_grad;
    if (!t.dense) {
      pb.t[nb++] = t;
      continue;
    }
    pd.row_start[nd + 1] = pd.row_start[nd] + s.rows;
    pd.t[nd++] = t;
    if (s.rows <= SMALL_MAX_ROWS) ps.t[ns++] = t;  // every id repeats many times per batch: sort + run sums
    else pm.t[nm++] = t;
  }
  pb.n = nb;
  ps.n = ns;
  pm.n = nm;
  pd.n = nd;
  for (SparseParams* q : {&pb, &ps, &pm, &pd}) {
    q->B = B;
    q->D = D;
    q->lgL = 0;
    while ((1 << q->lgL) < D / 4) ++q->lgL;
    q->opt = opt;
    q->hyper = hyper;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int L = 1 << pb.lgL;
  const unsigned bx1 = (unsigned)((B + 255) / 256), bxl = (unsigned)((B * L + 255) / 256);
  int rc = MM_OK;
  if (ns) {
    sparse_scatter_small_kernel<<<dim3((unsigned)((B + SMALL_CHUNK - 1) / SMALL_CHUNK), ns), 256, 0, st>>>(ps);
    if ((rc = check_launch("mm_sparse_rows_apply(scatter small)"))) return rc;
  }
  if (nm) {
    sparse_scatter_mid_kernel<<<dim3(bxl, nm), 256, 0, st>>>(pm);
    if ((rc = check_launch("mm_sparse_rows_apply(scatter mid)"))) return rc;
  }
  if (nd) {
    sparse_apply_dense_kernel<<<(unsigned)((pd.row_start[nd] * L + 255) / 256), 256, 0, st>>>(pd);
    if ((rc = check_launch("mm_sparse_rows_apply(apply dense)"))) return rc;
  }
  if (nb) {
    sparse_elect_kernel<<<dim3(bx1, nb), 256, 0, st>>>(pb);
    if ((rc = check_launch("mm_sparse_rows_apply(elect)"))) return rc;
    sparse_fold_kernel<<<dim3(bx1, nb), 256, 0, st>>>(pb);
    if ((rc = check_launch("mm_sparse_rows_apply(fold)"))) return rc;
    sparse_apply_kernel<<<dim3(bxl, nb), 256, 0, st>>>(pb);
    if ((rc = check_launch("mm_sparse_rows_apply(apply)"))) return rc;
  }
  return MM_OK;
}

int mm_dense_apply(int opt, float* w, float* grad, float* state1, float* state2, int64_t n, const float* hyper, float grad_scale,
                   void* stream) {
  MM_REQUIRE(w && grad && hyper && n >= 0, MM_ERR_ARG, "mm_dense_apply: null pointer");
  MM_REQUIRE(opt == MM_OPT_SGD || opt == MM_OPT_ADAGRAD || opt == MM_OPT_ADAM, MM_ERR_ARG, "mm_dense_apply: unknown optimizer %d", opt);
  MM_REQUIRE(opt == MM_OPT_SGD || state1, MM_ERR_ARG, "mm_dense_apply: optimizer state missing");
  MM_REQUIRE(opt != MM_OPT_ADAM || state2, MM_ERR_ARG, "mm_dense_apply: second optimizer state missing");
  if (n == 0) return MM_OK;
  long long blocks = (n + 255) / 256;
  const long long cap = 8LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  mm::trs::dense_apply_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(opt, w, grad, state1, state2, (long long)n, hyper, grad_scale);
  return mm::check_launch("mm_dense_apply");
}

int mm_opt_tick(float* hyper, void* stream) {
  MM_REQUIRE(hyper, MM_ERR_ARG, "mm_opt_tick: null pointer");
  mm::trs::opt_tick_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(hyper);
  return mm::check_launch("mm_opt_tick");
}

int mm_opt_tick_schedule(float* hyper, const float* sched, void* stream) {
  MM_REQUIRE(hyper && sched, MM_ERR_ARG, "mm_opt_tick_schedule: null pointer");
  mm::trs::opt_tick_schedule_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(hyper, sched);
  return mm::check_launch("mm_opt_tick_schedule");
}

int mm_bag_grad_rows(const float* g, int64_t B, int D, int64_t g_stride, const void* ids, int idx_dtype, const void* offsets,
                     int off_dtype, int L, int64_t nnz, int64_t rows, int combiner, float* out, void* out_ids, void* stream) {
  MM_REQUIRE(B >= 0 && nnz >= 0 && rows > 0 && (g || B == 0) && ((ids && out) || nnz == 0), MM_ERR_ARG,
             "mm_bag_grad_rows: null pointer or negative size");
  MM_REQUIRE(D == 16 || D == 32 || D == 64 || D == 128, MM_ERR_UNSUPPORTED, "mm_bag_grad_rows: D=%d not in {16,32,64,128}", D);
  MM_REQUIRE(idx_dtype == MM_I32 || idx_dtype == MM_I64, MM_ERR_ARG, "mm_bag_grad_rows: ids must be int32 or int64");
  if (offsets) {
    MM_REQUIRE(off_dtype == MM_I32 || off_dtype == MM_I64, MM_ERR_ARG, "mm_bag_grad_rows: offsets must be int32 or int64");
    MM_REQUIRE(combiner == MM_COMBINER_MEAN || combiner == MM_COMBINER_SUM || combiner == MM_COMBINER_SQRTN, MM_ERR_UNSUPPORTED,
               "mm_bag_grad_rows: ragged bags take the mean, sum or sqrtn combiner, got %d", combiner);
  } else {
    MM_REQUIRE(L > 0 && nnz == B * (int64_t)L, MM_ERR_ARG, "mm_bag_grad_rows: fixed-length bags need L > 0 and nnz = B * L");
    MM_REQUIRE(combiner == MM_COMBINER_MEAN || combiner == MM_COMBINER_SUM, MM_ERR_UNSUPPORTED,
               "mm_bag_grad_rows: fixed-length bags take the mean or sum combiner, got %d", combiner);
  }
  MM_REQUIRE(g_stride >= D && (g_stride & 3) == 0, MM_ERR_ARG, "mm_bag_grad_rows: g_stride must be a multiple of 4 and >= D");
  MM_REQUIRE((((uintptr_t)g | (uintptr_t)out) & 15) == 0, MM_ERR_ALIGN, "mm_bag_grad_rows: g and out must be 16-byte aligned");
  MM_REQUIRE(((uintptr_t)ids & (idx_dtype == MM_I64 ? 7 : 3)) == 0 &&
                 (!offsets || ((uintptr_t)offsets & (off_dtype == MM_I64 ? 7 : 3)) == 0) &&
                 ((uintptr_t)out_ids & (idx_dtype == MM_I64 ? 7 : 3)) == 0,
             MM_ERR_ALIGN, "mm_bag_grad_rows: ids / offsets / out_ids not aligned to their width");
  if (nnz == 0) return MM_OK;
  const long long tasks = offsets ? B + 2 : B;
  long long blocks = (tasks + 7) / 8;
  const long long cap = 64LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  cudaStream_t st = (cudaStream_t)stream;
  const bool i64 = idx_dtype == MM_I64, o64 = offsets && off_dtype == MM_I64;
  using mm::trs::launch_bag_grad;
  if (i64 && o64) launch_bag_grad<long long, long long>((unsigned)blocks, st, g, g_stride, ids, offsets, L, B, nnz, rows, combiner, D, out, out_ids);
  else if (i64) launch_bag_grad<long long, int>((unsigned)blocks, st, g, g_stride, ids, offsets, L, B, nnz, rows, combiner, D, out, out_ids);
  else if (o64) launch_bag_grad<int, long long>((unsigned)blocks, st, g, g_stride, ids, offsets, L, B, nnz, rows, combiner, D, out, out_ids);
  else launch_bag_grad<int, int>((unsigned)blocks, st, g, g_stride, ids, offsets, L, B, nnz, rows, combiner, D, out, out_ids);
  return mm::check_launch("mm_bag_grad_rows");
}

int mm_wide_rows_apply(float* wide, float* state1, float* state2, int64_t wide_rows, const mm_wide_block* blocks_host, int n_blocks,
                       int64_t B, const float* grad, float* acc, int32_t* rep_map, const int64_t* dense_offsets_host, int n_dense,
                       float* dense_grad, float* bias, float* bias_state1, float* bias_state2, int opt, const float* hyper, void* stream) {
  using namespace mm;
  using namespace mm::trs;
  MM_REQUIRE(wide && blocks_host && grad && acc && rep_map && hyper && B >= 0 && wide_rows > 0, MM_ERR_ARG,
             "mm_wide_rows_apply: null pointer or bad size");
  MM_REQUIRE(n_blocks >= 1 && n_blocks <= WIDE_MAX_BLOCKS && n_dense >= 0 && n_dense <= WIDE_MAX_DENSE, MM_ERR_UNSUPPORTED,
             "mm_wide_rows_apply: 1..%d feature blocks and 0..%d dense rows", WIDE_MAX_BLOCKS, WIDE_MAX_DENSE);
  MM_REQUIRE(opt == MM_OPT_SGD || opt == MM_OPT_ADAGRAD || opt == MM_OPT_ADAM, MM_ERR_ARG, "mm_wide_rows_apply: unknown optimizer %d", opt);
  MM_REQUIRE(opt == MM_OPT_SGD || (state1 && (!bias || bias_state1)), MM_ERR_ARG, "mm_wide_rows_apply: optimizer state missing");
  MM_REQUIRE(opt != MM_OPT_ADAM || (state2 && (!bias || bias_state2)), MM_ERR_ARG, "mm_wide_rows_apply: second optimizer state missing");
  MM_REQUIRE((n_dense == 0 && !bias) || (dense_grad && (n_dense == 0 || dense_offsets_host)), MM_ERR_ARG,
             "mm_wide_rows_apply: dense rows or a bias without dense_grad / offsets");
  MM_REQUIRE(B < (int64_t)INT_MAX, MM_ERR_UNSUPPORTED, "mm_wide_rows_apply: batch too large for the int32 representative map");
  WideParams p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < n_blocks; ++i) {
    const mm_wide_block& s = blocks_host[i];
    if (const int rc = check_id_column("mm_wide_rows_apply", i, s.indices, s.idx_bytes, s.rows)) return rc;
    MM_REQUIRE(s.offset >= 0 && s.offset + s.rows <= wide_rows, MM_ERR_ARG, "mm_wide_rows_apply: block %d: rows outside the wide kernel", i);
    for (int j = 0; j < i; ++j)
      MM_REQUIRE(s.offset >= blocks_host[j].offset + blocks_host[j].rows || blocks_host[j].offset >= s.offset + s.rows, MM_ERR_ARG,
                 "mm_wide_rows_apply: blocks %d and %d overlap", j, i);
    p.blk[i].ids = s.indices;
    p.blk[i].rows = s.rows;
    p.blk[i].off = s.offset;
    p.blk[i].idx_bytes = s.idx_bytes;
  }
  for (int c = 0; c < n_dense; ++c) {
    MM_REQUIRE(dense_offsets_host[c] >= 0 && dense_offsets_host[c] < wide_rows, MM_ERR_ARG, "mm_wide_rows_apply: dense row %d outside the wide kernel", c);
    for (int i = 0; i < n_blocks; ++i)
      MM_REQUIRE(dense_offsets_host[c] < blocks_host[i].offset || dense_offsets_host[c] >= blocks_host[i].offset + blocks_host[i].rows,
                 MM_ERR_ARG, "mm_wide_rows_apply: dense row %d lies in block %d", c, i);
    p.dense_off[c] = dense_offsets_host[c];
  }
  p.n_dense = n_dense;
  p.w = wide;
  p.s1 = state1;
  p.s2 = state2;
  p.acc = acc;
  p.rep = rep_map;
  p.g = grad;
  p.dgrad = dense_grad;
  p.bias = bias;
  p.bs1 = bias_state1;
  p.bs2 = bias_state2;
  p.B = B;
  p.opt = opt;
  p.hyper = hyper;
  cudaStream_t st = (cudaStream_t)stream;
  long long sx = (B + WIDE_CHUNK - 1) / WIDE_CHUNK;
  long long scap = 2LL * sm_count() / n_blocks;
  if (scap < 1) scap = 1;
  if (sx > scap) sx = scap;
  if (sx >= 1) {
    wide_scatter_kernel<<<dim3((unsigned)sx, (unsigned)n_blocks), 256, 0, st>>>(p);
    if (const int rc = check_launch("mm_wide_rows_apply(scatter)")) return rc;
  }
  long long span = B;
  for (int i = 0; i < n_blocks; ++i)
    if (blocks_host[i].rows <= WIDE_DENSE_ROWS && blocks_host[i].rows > span) span = blocks_host[i].rows;
  long long ax = (span + 255) / 256;
  long long acap = 4LL * sm_count() / n_blocks;
  if (acap < 1) acap = 1;
  if (ax > acap) ax = acap;
  if (ax < 1) ax = 1;
  wide_apply_kernel<<<dim3((unsigned)ax, (unsigned)n_blocks), 256, 0, st>>>(p);
  if (const int rc = check_launch("mm_wide_rows_apply(apply)")) return rc;
  if (n_dense == 0 && !bias) return MM_OK;
  wide_dense_apply_kernel<<<1, 96, 0, st>>>(p);
  return check_launch("mm_wide_rows_apply(dense rows)");
}

int mm_fill_i32(int32_t* p, int64_t n, int32_t value, void* stream) {
  MM_REQUIRE(p && n >= 0, MM_ERR_ARG, "mm_fill_i32: null pointer");
  if (n == 0) return MM_OK;
  long long blocks = (n + 255) / 256;
  const long long cap = 16LL * mm::sm_count();
  if (blocks > cap) blocks = cap;
  mm::trs::fill_i32_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(p, (long long)n, value);
  return mm::check_launch("mm_fill_i32");
}

}  // extern "C"
