// DLRM lookup + pairwise interaction on mma.sync, one warp per sample: the tensor-core path of
// mm_dlrm_lookup_interact and mm_dot_interaction (F <= 32, D in {16, 32, 64, 128}, P in {0, D}).
//
// The kernel is bound on the SM side, not by DRAM: serving the large tables' rows from L2 saves 1-3 % on H100 (DESIGN.md
// §4 has the measurements, phase by phase), so every phase is built to issue few instructions per sample:
//   * copy loop: 8 lanes move one 128-byte half row per LDGSTS, 4 rows per instruction.  Staged row r is
//     owned by lane r (tables arrive sorted by slot, so row == slot), a row's source pointer travels
//     with two shuffles, and because row = 4*i + lane/8 the XOR swizzle of a lane's destination does
//     not depend on i: every destination is `lane constant + immediate`.  7 iterations x (2 SHFL +
//     2 IADD + 2 LDGSTS) per sample at F = 27; the operand-format path runs all 8 without a branch.  Bad ids
//     read a zero row in global memory (no zero-fill operand, no predicates).
//   * fragment loads: the k index of a 16-wide k-step is permuted (lane t takes floats 4t..4t+3 and
//     calls them k = 2t, 2t+1, 2t+8, 2t+9).  A and B fragments are the same registers (B = X^T), so the
//     permutation cancels in the dot products and one LDS.128 replaces two LDS.64.
//   * the fp32 output row is staged INSIDE the sample buffer that was just consumed (the prefix row is
//     lifted into registers first), so a warp needs 2 x rows x D x 4 bytes and 16 warps fit in 227 KB.
//   * index arrays may be 1, 2, 3 (unsigned), 4 or 8 (signed) bytes wide PER TABLE — a host batch ships
//     52-60 B of ids per Criteo sample instead of 104 (PCIe is the end-to-end bound).
//   * a table may be ROW-SHARDED over the GPUs of an NVLink domain: row r lives on rank r % world at
//     local row r / world, and the owner lane takes the row's address from that rank's peer-mapped
//     shard — the cp.async reads the row over NVLink straight into this SM's shared memory.  Lookup,
//     all-to-all and interaction are ONE kernel: no index exchange, no send/receive buffers, no barrier
//     (tables are read-only in the forward pass).
//
// Replaces: T x Embedding lookups (inputs/embedding.py:401-471) or SOK's distributed lookup
// (distributed/embedding.py:75-84,144-148) + StackFeatures (core/aggregation.py:101-108) +
// DotProductInteraction (blocks/interaction.py:86-116) + shortcut concat (blocks/dlrm.py:126-130).
#include <cuda_bf16.h>

#include <cstring>

#include "mm_common.cuh"
#include "warp_mma.cuh"

namespace mm {
namespace imma2 {

__device__ __align__(16) float g_zero_row[128];  // zero-initialised: source of rows for out-of-range ids

// Sample buffers per warp: one sample in flight behind the one being computed, for local tables and for rows that come
// over NVLink alike.  Deeper pipelines do not pay for rows read over NVLink: remote latency is dominated by hot rows of
// tiny sharded tables serialising on single cache lines of the owner, which replicating those tables removes.
constexpr int NBUF = 2;

struct Params {
  const float* x;  // MODE 0: stacked input
  long long x_stride;
  const float* prefix;  // bottom vector (P == 0 or P == D)
  long long prefix_stride;
  int P;
  int bottom_slot;  // MODE 1: staged row of the bottom vector (-1: none)
  long long B;
  int F, D;
  int rows;  // rows staged per sample (F, or F+1 when MODE 0 carries a separate prefix row)
  float* out_f32;
  long long out_stride;
  __nv_bfloat16* out_split;
  int out_Kp;
  int* oob_count;
  int n_warps;
  unsigned buf_bytes;   // one sample buffer (>= rows*D*4 and >= the staged output row)
  unsigned stage_cols;  // floats of the staged output row (out_Kp, or OW rounded up to 4)
  unsigned peer_off;    // byte offset of the peer pointer table in shared memory
};

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

struct RawIdx {
  uint32_t a, b, sh;  // the aligned word(s) holding an id, and the bit offset of the id inside `a`
};

// Negative result kept as a note (the code is gone): issuing the Gram matrix as m16n8k8 MMAs.  With k16 every bf16x2
// register must sit both in an A quad {X[g],X[g+8]} x {k-lo,k-hi} and in a B pair {k-lo,k-hi} of one row — two
// incompatible adjacencies that cost many register moves per sample.  k8 operands are an A pair and a single
// B register: no moves, but twice as many MMAs, and HMMA.1688 occupies the legacy tensor pipe as long as HMMA.16816,
// so it was slower.
//
// PS ("pre-split", D = 64): the staged rows are split-bf16 rows [hi(0..D) | lo(0..D)] — the operand format of every
// tensor-core layer of this library (mm_split_rows) — read from a second copy of the tables in HBM; the bottom vector
// arrives in the same format from the tower kernel.  The rows land in shared memory with the 128-byte XOR swizzle
// (16-byte chunk c of row r at chunk c ^ (r & 7)) and the MMA fragments are loaded by ldmatrix.x4: per 16-wide k-step
// four loads give the A quads (hi and lo, two m-tiles), already in the register shape HMMA wants, and the B pairs of the
// four n-tiles are the same registers (B = X^T).  Per sample: 16 LDSM + 72 HMMA instead of 16 LDS.128 + 192 split
// instructions + ~180 operand moves + 72 HMMA.  Same values as the in-kernel split => bit-identical output.
// (A first attempt kept the lane-private LDS.128 scheme with hi and lo interleaved per chunk: fewer instructions, but
// the A quads still had to be assembled with moves and nothing overlapped the load -> HMMA latency: 0.116 ms vs 0.104.)
template <int MODE, int KD /* embedding dim: 16, 32, 64, 128 */, int NWARPS /* launch bound */, bool PS>
__global__ void __launch_bounds__(32 * NWARPS, 1)
interact_v2_kernel(const __grid_constant__ LookupParams lk, const Params p) {
  extern __shared__ __align__(256) uint8_t smem_raw[];
  constexpr int D = KD, KS = KD / 16;
  static_assert(!PS || KD == 64, "operand-format rows: D = 64");
  constexpr int C = KD / 4;           // 16-byte chunks per row
  constexpr int L = C < 8 ? C : 8;    // lanes per row in the copy loop
  constexpr int J = C / L;            // copies per lane and row
  constexpr int R = 32 / L;           // rows per copy instruction
  constexpr int IMAX = 32 / R;        // copy iterations for 32 rows
  constexpr bool SWZ = KD >= 32;      // chunk index XOR 4 on odd rows (bank-conflict-free LDS.128 of two rows)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int F = p.F;
  const int nw = p.n_warps;
  const uint32_t wbase = smem_u32(smem_raw) + (uint32_t)warp * (NBUF * p.buf_bytes);

  // ---- samples of this CTA: a contiguous range, interleaved over its warps (neighbouring warps read
  // neighbouring ids: the 32-byte index sectors are shared through L1 instead of being fetched 8 times).
  // Every warp runs the SAME number of iterations (a function of blockIdx only, so the loop and the shuffles
  // inside it are provably convergent); a warp whose last sample does not exist skips the work, not the loop.
  const long long begin = (long long)blockIdx.x * p.B / gridDim.x;
  const int n_cta = (int)((long long)(blockIdx.x + 1) * p.B / gridDim.x - begin);
  const int n_iter = (n_cta + nw - 1) / nw;
  const long long s0 = begin + warp;  // first sample of this warp

  // ---- owner role: lane r owns staged row r (MODE 1: a table, or the bottom vector)
  const bool is_table = MODE == 1 && lane < p.rows && lane != p.bottom_slot;
  const float* my_base = is_table ? lk.weights[lane] : nullptr;
  const unsigned long long my_rows = is_table ? (unsigned long long)lk.rows[lane] : 0ull;
  const int my_w = is_table ? lk.idx_bytes[lane] : 4;
  const bool my_sharded = is_table && lk.sharded[lane];
  const bool my_64 = my_w == 8;
  const uint32_t my_mask = my_w >= 4 ? 0xffffffffu : (0xffffffffu >> (32 - 8 * my_w));
  const uint8_t* id_ptr = is_table ? reinterpret_cast<const uint8_t*>(lk.indices[lane]) + (size_t)s0 * my_w : nullptr;
  const int id_step = nw * my_w;
  const float* const* peers = reinterpret_cast<const float* const*>(smem_raw + p.peer_off);
  if (MODE == 1 && lk.world > 1) {  // peer shard pointers: kernel parameters -> shared memory (indexed by lane AND owner)
    float const** dst = reinterpret_cast<float const**>(smem_raw + p.peer_off);
    for (int i = threadIdx.x; i < p.rows * lk.world; i += blockDim.x) dst[i] = lk.peers[i];
    __syncthreads();
  }
  // running source pointers of the non-table rows
  const uint8_t* pfx_ptr = p.prefix ? reinterpret_cast<const uint8_t*>(p.prefix + s0 * p.prefix_stride) : nullptr;
  const long long pfx_step = (long long)nw * p.prefix_stride * 4;

  // ids are fetched as the aligned 32-bit word(s) that contain them, one iteration before they are decoded
  int k_load = warp;  // index (inside the CTA's range) of the sample whose id is loaded next
  auto load_raw = [&]() -> RawIdx {
    RawIdx r{0u, 0u, 0u};
    if (MODE == 1 && is_table && k_load < n_cta) {
      const uintptr_t a = reinterpret_cast<uintptr_t>(id_ptr);
      const uint32_t* wp = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
      r.sh = 8u * (uint32_t)(a & 3);
      r.a = __ldg(wp);
      if (my_64 || (int)(a & 3) + my_w > 4) r.b = __ldg(wp + 1);
    }
    id_ptr += id_step;
    k_load += nw;
    return r;
  };

  // ---- copy-loop constants of this lane
  const int cl = lane & (L - 1), rl = lane / L;
  const uint32_t src_lane_off = (uint32_t)cl * 16u;
  // fp32 rows: chunk XOR 4 on odd rows; PS rows (row = 4i + rl, 8 lanes per 128-byte half): chunk ^ (row & 7) with
  // row & 7 = rl + 4 (i & 1) -> one constant for even i, one for odd i
  const uint32_t dst_lane_off =
      (uint32_t)rl * (D * 4) + (uint32_t)((PS ? (cl ^ rl) : SWZ ? (cl ^ ((rl & 1) << 2)) : cl) * 16);
  const uint32_t dst_lane_off_odd = (uint32_t)rl * (D * 4) + (uint32_t)((cl ^ (rl + 4)) * 16);  // PS, odd i
  const uint8_t* x_ptr = MODE == 0 ? reinterpret_cast<const uint8_t*>(p.x + s0 * p.x_stride) + (size_t)rl * (D * 4) + src_lane_off
                                   : nullptr;
  const long long x_step = (long long)nw * p.x_stride * 4;

  int k_issue = warp;
  uint32_t buf_issue = 0;  // byte offset (0 / buf_bytes) of the buffer the next sample is staged in
  auto issue = [&](RawIdx raw) {
    // The shuffles run unconditionally; past the end of this warp's samples the row count is 0 and nothing is copied.
    const int live_rows = k_issue < n_cta ? p.rows : 0;
    const uint32_t xs = wbase + buf_issue + dst_lane_off;
    if (MODE == 1) {
      const float* my_src = g_zero_row;
      if (is_table) {
        const uint32_t v = __funnelshift_r(raw.a, raw.b, raw.sh) & my_mask;
        const uint32_t hi = my_64 ? raw.b : (uint32_t)((int)v >> 31);
        const unsigned long long idx = ((unsigned long long)hi << 32) | v;
        if (idx < my_rows) {  // unsigned: negative ids are out of range too
          if (my_sharded) {
            unsigned long long lrow;
            int owner;
            if (lk.log2_world >= 0) {
              owner = (int)(idx & (unsigned)(lk.world - 1));
              lrow = idx >> lk.log2_world;
            } else {
              lrow = idx / (unsigned)lk.world;
              owner = (int)(idx - lrow * (unsigned)lk.world);
            }
            my_src = peers[lane * lk.world + owner] + lrow * D;
          } else {
            my_src = my_base + idx * D;
          }
        } else if (live_rows && p.oob_count) {
          atomicAdd(p.oob_count, 1);
        }
      } else if (lane == p.bottom_slot) {
        my_src = reinterpret_cast<const float*>(pfx_ptr);
      }
      const uint32_t src_lo = (uint32_t)(uintptr_t)my_src, src_hi = (uint32_t)((uintptr_t)my_src >> 32);
#pragma unroll
      for (int i = 0; i < IMAX; ++i) {
        // PS: all 8 iterations, the copies of rows past p.rows predicated off (no branch and divergence check per pair of
        // shuffles).  Otherwise a kernel parameter: uniform branch.
        if (PS || i * R < p.rows) {
          const int row = i * R + rl;
          const uint32_t lo = __shfl_sync(0xffffffffu, src_lo, row);
          const uint32_t hi = __shfl_sync(0xffffffffu, src_hi, row);
          const uint8_t* src = reinterpret_cast<const uint8_t*>(((uintptr_t)hi << 32) | lo) + src_lane_off;
          const bool on = row < live_rows;
          const uint32_t xd = (PS && (i & 1)) ? xs - dst_lane_off + dst_lane_off_odd : xs;
#pragma unroll
          for (int j = 0; j < J; ++j) cp_async16_if(on, xd + (uint32_t)(i * R * D * 4 + j * L * 16), src + j * L * 16);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < IMAX; ++i) {
        if (i * R < p.rows) {
          const int row = i * R + rl;
          const uint8_t* src = row < F ? x_ptr + (size_t)i * (R * D * 4) : pfx_ptr + src_lane_off;
          const bool on = row < live_rows;
#pragma unroll
          for (int j = 0; j < J; ++j) cp_async16_if(on, xs + (uint32_t)(i * R * D * 4 + j * L * 16), src + j * L * 16);
        }
      }
      x_ptr += x_step;
    }
    pfx_ptr += pfx_step;
    k_issue += nw;
    buf_issue += p.buf_bytes;
    if (buf_issue == NBUF * p.buf_bytes) buf_issue = 0;
    cp_async_commit();  // one group per sample (empty past the end keeps the group count in step)
  };

  // ---- fragment-load constants: rows q*8 + g (q = 0..3), clamped to staged rows; this lane reads floats
  // 4t..4t+3 of every 16-wide k-step.  Even k-steps sit at pe + 64*ks, odd ones at po + 64*ks (the XOR
  // swizzle of odd rows swaps neighbouring k-steps).
  uint32_t pe[4], po[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int r = min(8 * q + g, F - 1);
    const uint32_t base = (uint32_t)r * (D * 4) + (uint32_t)t * 16u;
    const uint32_t sb = (SWZ && (r & 1)) ? 64u : 0u;
    pe[q] = base + sb;
    po[q] = base - sb;
  }
  // ---- PS: ldmatrix row addresses.  Lane l supplies row (l & 7) of matrix (l >> 3).
  //   A quad of m-tile mt (rows 16mt..): matrices (rows +0..7, k-lo) (rows +8..15, k-lo) (rows +0..7, k-hi) (rows +8..15, k-hi)
  // k-lo / k-hi = chunks 2ks / 2ks+1 of the hi half (+128 bytes: lo half).  With 256-byte aligned buffers the byte offset
  // is row*256 | ((chunk ^ (row & 7)) << 4), and (2ks + b) ^ x = (2ks) ^ (b ^ x): one XOR with 32*ks per k-step.
  uint32_t la[2];
  {
    const int mi = lane >> 3, j = lane & 7;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int ra = min(16 * u + (mi & 1) * 8 + j, F - 1);
      la[u] = (uint32_t)ra * 256u | (uint32_t)((((mi >> 1) ^ ra) & 7) << 4);
    }
  }

  // ---- output constants: accumulator (i, j) with i = 8*qi + g, j = 8*nt + 2t + e lands at
  // P + i(2F-i-1)/2 + (j-i-1) = rb[qi] + 8*nt + e   (floats); valid iff i < j < F
  int rb[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = 8 * q + g;
    rb[q] = (p.P + i * (2 * F - i - 1) / 2 - i - 1 + 2 * t) * 4;  // bytes
  }
  const int jlim = F - 2 * t;        // j < F  <=>  8*nt + e < jlim
  const bool dg0 = g < 2 * t, dg1 = g < 2 * t + 1;  // diagonal tiles: i < j  <=>  g < 2t + e
  const int npairs = F * (F - 1) / 2;
  const int OW = p.P + npairs;
  const int prow = MODE == 1 ? p.bottom_slot : F;  // staged row holding the prefix
  const uint32_t pfx_off = (uint32_t)prow * (D * 4) + (uint32_t)((SWZ ? (lane ^ ((prow & 1) << 2)) : lane) * 16);
  // running output pointers
  __nv_bfloat16* osplit = p.out_split ? p.out_split + s0 * (2ll * p.out_Kp) : nullptr;
  float* of32 = p.out_f32 ? p.out_f32 + s0 * p.out_stride : nullptr;
  const bool f32_vec = ((p.out_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out_f32) & 15) == 0);

  // ---- software pipeline: NBUF-1 samples in flight behind the one being computed; ids one iteration ahead of their rows
  RawIdx raw_pref = load_raw();
#pragma unroll
  for (int i = 0; i < NBUF - 1; ++i) {
    const RawIdx cur = raw_pref;
    raw_pref = load_raw();
    issue(cur);
  }
  int k_cmp = warp;
  uint32_t buf_cmp = 0;
  for (int it = 0; it < n_iter; ++it) {
    const RawIdx cur = raw_pref;
    raw_pref = load_raw();
    issue(cur);  // refills the buffer consumed (and used as output stage) in the previous iteration
    cp_async_wait<NBUF - 1>();
    __syncwarp();
    const uint32_t xs = wbase + buf_cmp;
    buf_cmp += p.buf_bytes;
    if (buf_cmp == NBUF * p.buf_bytes) buf_cmp = 0;
    if (k_cmp < n_cta) {
      float acc[6][4];
#pragma unroll
      for (int ti = 0; ti < 6; ++ti)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[ti][c] = 0.0f;

      const uint32_t a0b = xs + la[0], a1b = xs + la[1];
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        // A quads of m-tiles 0, 1 and B pairs of n-tiles 0..3 (n-tile nt = rows 8nt + g), hi and lo
        uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
        if (PS) {
          const uint32_t kx = 32u * ks;
          ldsm_x4(a0b ^ kx, ah[0][0], ah[0][1], ah[0][2], ah[0][3]);
          ldsm_x4((a0b ^ kx) + 128u, al[0][0], al[0][1], al[0][2], al[0][3]);
          ldsm_x4(a1b ^ kx, ah[1][0], ah[1][1], ah[1][2], ah[1][3]);
          ldsm_x4((a1b ^ kx) + 128u, al[1][0], al[1][1], al[1][2], al[1][3]);
          // B = X^T: the B pairs of n-tiles 2mt, 2mt+1 are registers of the A quad of m-tile mt (same rows, same clamp)
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            bh[2 * mt][0] = ah[mt][0], bh[2 * mt][1] = ah[mt][2], bh[2 * mt + 1][0] = ah[mt][1], bh[2 * mt + 1][1] = ah[mt][3];
            bl[2 * mt][0] = al[mt][0], bl[2 * mt][1] = al[mt][2], bl[2 * mt + 1][0] = al[mt][1], bl[2 * mt + 1][1] = al[mt][3];
          }
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 v = lds128(xs + ((ks & 1) ? po[q] : pe[q]) + 64u * ks);
            split_pair(v.x, v.y, bh[q][0], bl[q][0]);
            split_pair(v.z, v.w, bh[q][1], bl[q][1]);
          }
          // the A quad of m-tile mt is made of the B pairs of rows q = 2mt, 2mt+1
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            ah[mt][0] = bh[2 * mt][0], ah[mt][1] = bh[2 * mt + 1][0], ah[mt][2] = bh[2 * mt][1], ah[mt][3] = bh[2 * mt + 1][1];
            al[mt][0] = bl[2 * mt][0], al[mt][1] = bl[2 * mt + 1][0], al[mt][2] = bl[2 * mt][1], al[mt][3] = bl[2 * mt + 1][1];
          }
        }
        // tile ti = (mt, nt).  Pass-major order: six independent accumulators between dependent MMAs.
#pragma unroll
        for (int ti = 0; ti < 6; ++ti) {
          const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
          mma16816(acc[ti], ah[mt], bl[nt][0], bl[nt][1]);
        }
#pragma unroll
        for (int ti = 0; ti < 6; ++ti) {
          const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
          mma16816(acc[ti], al[mt], bh[nt][0], bh[nt][1]);
        }
#pragma unroll
        for (int ti = 0; ti < 6; ++ti) {
          const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
          mma16816(acc[ti], ah[mt], bh[nt][0], bh[nt][1]);
        }
      }

      // ---- the prefix row leaves the buffer before the buffer becomes the output stage
      float4 pfx = make_float4(0.f, 0.f, 0.f, 0.f);
      if (PS) {  // chunk (lane & 7) of the hi (lanes 0-7) / lo (lanes 8-15) half of the bottom row, un-swizzled
        if (p.P > 0 && lane < 16)
          pfx = lds128(xs + (uint32_t)prow * 256u + ((uint32_t)(lane & 8) << 4) + (uint32_t)((((lane & 7) ^ prow) & 7) << 4));
      } else if (p.P > 0 && lane < C) pfx = lds128(xs + pfx_off);
      __syncwarp();  // every lane is done reading the sample
      if (PS) {
        // split-bf16 prefix: the hi and lo halves of the bottom row go straight to the hi / lo halves of the output row
        if (p.P > 0 && lane < 16)
          *reinterpret_cast<float4*>(osplit + ((lane & 8) ? p.out_Kp : 0) + 8 * (lane & 7)) = pfx;
      } else if (p.P > 0 && lane < C) {
        asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(xs + lane * 16u), "f"(pfx.x), "f"(pfx.y), "f"(pfx.z),
                     "f"(pfx.w)
                     : "memory");
      }
#pragma unroll
      for (int ti = 0; ti < 6; ++ti) {
        const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int qi = 2 * mt + (c >> 1), e = c & 1;
          if (qi > nt) continue;  // below the diagonal: never stored
          bool ok = (8 * nt + e) < jlim;
          if (qi == nt) ok = ok && (e ? dg1 : dg0);
          if (ok) sts32(xs + (uint32_t)(rb[qi] + (8 * nt + e) * 4), acc[ti][c]);
        }
      }
      for (int e = OW + lane; e < (int)p.stage_cols; e += 32) sts32(xs + (uint32_t)e * 4u, 0.0f);  // zero padding
      __syncwarp();

      // ---- coalesced row store
      if (p.out_split) {
        const int groups = p.out_Kp >> 3;  // 8 columns = one 16-byte bf16 store for hi and one for lo
        for (int gi = (PS ? (p.P >> 3) : 0) + lane; gi < groups; gi += 32) {  // PS: the prefix groups are already out
          const float4 a = lds128(xs + (uint32_t)gi * 32u), b = lds128(xs + (uint32_t)gi * 32u + 16u);
          uint32_t hh[4], ll[4];
          split_pair(a.x, a.y, hh[0], ll[0]);
          split_pair(a.z, a.w, hh[1], ll[1]);
          split_pair(b.x, b.y, hh[2], ll[2]);
          split_pair(b.z, b.w, hh[3], ll[3]);
          *reinterpret_cast<uint4*>(osplit + 8 * gi) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
          *reinterpret_cast<uint4*>(osplit + p.out_Kp + 8 * gi) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
        }
      } else {
        if (f32_vec) {
          const int n4 = OW >> 2;
          for (int e = lane; e < n4; e += 32) reinterpret_cast<float4*>(of32)[e] = lds128(xs + (uint32_t)e * 16u);
          for (int e = (n4 << 2) + lane; e < OW; e += 32) of32[e] = lds32(xs + (uint32_t)e * 4u);
        } else {
          for (int e = lane; e < OW; e += 32) of32[e] = lds32(xs + (uint32_t)e * 4u);
        }
      }
    }
    k_cmp += nw;
    if (osplit) osplit += (long long)nw * 2 * p.out_Kp;
    if (of32) of32 += (long long)nw * p.out_stride;
    __syncwarp();  // the buffer may be refilled by the next iteration's copies
  }
}

// Two launch bounds per shape: 16 warps when they fit, else the 12-warp variant (more registers per thread), which
// takes any smaller count (D = 128, F = 32: 32 KB per warp, 7 warps).
template <int MODE, int KD, bool PS>
static int launch_kd(const LookupParams& lk, const Params& p, size_t smem, unsigned grid, cudaStream_t st, const char* who) {
  const int wide = p.n_warps > 12;
  auto kern = wide ? interact_v2_kernel<MODE, KD, 16, PS> : interact_v2_kernel<MODE, KD, 12, PS>;
  static bool attr_set[2][64] = {};  // per device: function attributes belong to the device's copy of the kernel
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[wide][dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute failed: %s", who, cudaGetErrorString(e));
      return (int)e;
    }
    if (dev >= 0 && dev < 64) attr_set[wide][dev] = true;
  }
  kern<<<grid, 32 * p.n_warps, smem, st>>>(lk, p);
  return check_launch(who);
}

// Returns MM_ERR_UNSUPPORTED (without touching the error text) when the fast path does not apply.
// MODE 1: `lk` lists the tables BY STAGED ROW (= slot); the bottom row's entries are null.
template <int MODE>
int launch(const float* x, int64_t x_stride, const LookupParams& lk, const float* prefix, int64_t prefix_stride, int P,
           int bottom_slot, int64_t B, int F, int D, float* out_f32, int64_t out_stride, void* out_split, int out_Kp,
           int32_t* oob, cudaStream_t st, const char* who, bool presplit) {
  if (presplit && (MODE != 1 || !out_split || D != 64)) return MM_ERR_UNSUPPORTED;
  if (F < 2 || F > 32 || (D != 16 && D != 32 && D != 64 && D != 128)) return MM_ERR_UNSUPPORTED;
  if (P != 0 && P != D) return MM_ERR_UNSUPPORTED;
  if (out_f32 && out_split) return MM_ERR_UNSUPPORTED;
  const int rows = (MODE == 0 && P > 0) ? F + 1 : F;
  if (rows > 32) return MM_ERR_UNSUPPORTED;
  if (MODE == 0 && (((uintptr_t)x & 15) || (x_stride & 3))) return MM_ERR_UNSUPPORTED;
  if (P > 0 && (((uintptr_t)prefix & 15) || (prefix_stride & 3))) return MM_ERR_UNSUPPORTED;
  const int OW = P + F * (F - 1) / 2;
  Params p;
  memset(&p, 0, sizeof(p));
  p.x = x;
  p.x_stride = x_stride;
  p.prefix = prefix;
  p.prefix_stride = prefix_stride;
  p.P = P;
  p.bottom_slot = bottom_slot;
  p.B = B;
  p.F = F;
  p.D = D;
  p.rows = rows;
  p.out_f32 = out_f32;
  p.out_stride = out_stride;
  p.out_split = (__nv_bfloat16*)out_split;
  p.out_Kp = out_Kp;
  p.oob_count = oob;
  p.stage_cols = out_split ? (unsigned)out_Kp : (unsigned)((OW + 3) & ~3);
  const unsigned in_bytes = (unsigned)(rows * D * 4), stage_bytes = p.stage_cols * 4u;
  p.buf_bytes = ((in_bytes > stage_bytes ? in_bytes : stage_bytes) + 255u) & ~255u;  // 256-B aligned (ldmatrix address XOR)
  const unsigned per_warp = NBUF * p.buf_bytes;
  const unsigned peer_bytes = (MODE == 1 && lk.world > 1) ? (unsigned)(rows * lk.world * 8) : 0u;
  const unsigned budget = 227u * 1024u - peer_bytes;
  int warps = (int)(budget / per_warp);
  if (warps > 16) warps = 16;
  if (warps < 2) return MM_ERR_UNSUPPORTED;
  p.n_warps = warps;
  p.peer_off = (unsigned)warps * per_warp;
  const size_t smem = (size_t)p.peer_off + peer_bytes;
  const long long sms = sm_count();
  long long want = (B + warps - 1) / warps;
  const unsigned grid = (unsigned)(want < sms ? want : sms);
  if (presplit) return launch_kd<1, 64, true>(lk, p, smem, grid, st, who);  // MODE 1, D = 64 (checked above)
  switch (D) {
    case 16: return launch_kd<MODE, 16, false>(lk, p, smem, grid, st, who);
    case 32: return launch_kd<MODE, 32, false>(lk, p, smem, grid, st, who);
    case 64: return launch_kd<MODE, 64, false>(lk, p, smem, grid, st, who);
    default: return launch_kd<MODE, 128, false>(lk, p, smem, grid, st, who);
  }
}

template int launch<0>(const float*, int64_t, const LookupParams&, const float*, int64_t, int, int, int64_t, int, int,
                       float*, int64_t, void*, int, int32_t*, cudaStream_t, const char*, bool);
template int launch<1>(const float*, int64_t, const LookupParams&, const float*, int64_t, int, int, int64_t, int, int,
                       float*, int64_t, void*, int, int32_t*, cudaStream_t, const char*, bool);

}  // namespace imma2
}  // namespace mm
