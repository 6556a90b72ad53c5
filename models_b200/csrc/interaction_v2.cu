// DLRM lookup + pairwise interaction, one warp per sample (second generation of interaction_mma.cu).
//
// What changed against the first kernel (issue-bound, a large share of its instructions in the row-copy loop):
//   * copy loop: 8 lanes move one 128-byte half row per LDGSTS, 4 rows per instruction.  Staged row r is
//     owned by lane r (tables arrive sorted by slot, so row == slot), a row's source pointer travels
//     with two shuffles, and because row = 4*i + lane/8 the XOR swizzle of a lane's destination does
//     not depend on i: every destination is `lane constant + immediate`.  7 iterations x (2 SHFL +
//     2 IADD + 2 LDGSTS) per sample instead of 14 x 23 instructions.  Bad ids read a zero row in global
//     memory (no zero-fill operand, no predicates).
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

#include <cstdlib>
#include <cstring>

#include "mm_common.cuh"

namespace mm {
namespace imma2 {

__device__ __align__(16) float g_zero_row[128];  // zero-initialised: source of rows for out-of-range ids

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
  unsigned ids_off;     // byte offset of the per-warp id rings (NBUF > 2)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// predicated form: no branch / reconvergence bookkeeping around the copy
__device__ __forceinline__ void cp_async16_if(bool pred, uint32_t dst, const void* src) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p cp.async.cg.shared.global [%0], [%1], 16;\n\t}" ::"r"(dst),
      "l"(src), "r"((uint32_t)pred)
      : "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// (x, y) -> packed bf16x2 hi (x in the low half) and the bf16x2 of the residuals
__device__ __forceinline__ void split_pair(float x, float y, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  const float xh = __uint_as_float(hi << 16), yh = __uint_as_float(hi & 0xffff0000u);
  __nv_bfloat162 l = __floats2bfloat162_rn(x - xh, y - yh);
  lo = *reinterpret_cast<uint32_t*>(&l);
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
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
// four loads give the A quads (hi and lo, two m-tiles) and four the B pairs (hi and lo, four n-tiles), each already in the
// register shape HMMA wants.  Per sample: 32 LDSM + 16 LOP3 + 72 HMMA instead of 16 LDS.128 + 192 split instructions
// + ~180 operand moves + 72 HMMA.  Same values as the in-kernel split => bit-identical output.
// (A first attempt kept the lane-private LDS.128 scheme with hi and lo interleaved per chunk: fewer instructions, but
// the A quads still had to be assembled with moves and nothing overlapped the load -> HMMA latency: 0.116 ms vs 0.104.)
// NBUF sample buffers per warp: NBUF-1 samples in flight behind the one being computed.  The product uses 2 with
// 16 warps, for local tables and for rows that come over NVLink alike.  NBUF = 3 / 4 (10 / 7 warps, ids through a
// shared-memory ring) exist for experiments (MM_IMMA_NBUF): remote latency is dominated by hot rows of tiny
// sharded tables serialising on single cache lines of the owner, which replicating those tables removes.
template <int MODE, int KD /* embedding dim: 16, 32, 64, 128 */, int NWARPS /* launch bound */, bool PS, int NBUF>
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

  // ---- NBUF > 2 (rows over NVLink): ids travel through a per-warp shared-memory ring instead of registers.
  // A register prefetch one sample ahead is useless here: the id load queues in the memory pipeline behind
  // the row copies issued just before it and returns only after THEIR 10-20 us NVLink round trip, so every
  // sample would wait for the previous one (ncu, r2h: 49 % of the stall samples sat on the id decode).  Instead
  // the ids of sample j are copied (cp.async, 4-byte words) A = 2*NBUF-1 iterations before their rows are issued;
  // they ride in the same commit groups as the rows, so `wait_group` orders everything and no extra wait exists.
  constexpr bool IDS = NBUF > 2;
  constexpr int A = 2 * NBUF - 1, SLOTS = NBUF + 1;
  const uint32_t ring = smem_u32(smem_raw) + p.ids_off + (uint32_t)warp * (SLOTS * 256) + (uint32_t)lane * 8u;
  uint32_t slot_w = 0, slot_r = 0;  // byte offsets of the ring slots written / read next
  const uint8_t* idr_ptr = id_ptr;  // address of the id whose rows are issued next (bit offset inside its word)
  auto submit_ids = [&]() {
    if (MODE == 1 && is_table && k_load < n_cta) {
      const uintptr_t a = reinterpret_cast<uintptr_t>(id_ptr);
      const uint32_t* wp = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(ring + slot_w), "l"(wp) : "memory");
      if (my_64 || (int)(a & 3) + my_w > 4)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(ring + slot_w + 4u), "l"(wp + 1) : "memory");
    }
    id_ptr += id_step;
    k_load += nw;
    slot_w += 256u;
    if (slot_w == SLOTS * 256u) slot_w = 0;
  };
  auto read_ids = [&]() -> RawIdx {
    RawIdx r;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.a), "=r"(r.b) : "r"(ring + slot_r));
    r.sh = 8u * (uint32_t)(reinterpret_cast<uintptr_t>(idr_ptr) & 3);
    idr_ptr += id_step;
    slot_r += 256u;
    if (slot_r == SLOTS * 256u) slot_r = 0;
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
        if (i * R < p.rows) {  // kernel parameter: uniform branch
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
  //   B pairs of n-tiles 2u, 2u+1 (rows 16u..): matrices (rows +0..7, k-lo) (rows +0..7, k-hi) (rows +8..15, k-lo) (rows +8..15, k-hi)
  // k-lo / k-hi = chunks 2ks / 2ks+1 of the hi half (+128 bytes: lo half).  With 256-byte aligned buffers the byte offset
  // is row*256 | ((chunk ^ (row & 7)) << 4), and (2ks + b) ^ x = (2ks) ^ (b ^ x): one XOR with 32*ks per k-step.
  uint32_t la[2], lb[2];
  {
    const int mi = lane >> 3, j = lane & 7;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int ra = min(16 * u + (mi & 1) * 8 + j, F - 1), rbq = min(16 * u + (mi >> 1) * 8 + j, F - 1);
      la[u] = (uint32_t)ra * 256u | (uint32_t)((((mi >> 1) ^ ra) & 7) << 4);
      lb[u] = (uint32_t)rbq * 256u | (uint32_t)((((mi & 1) ^ rbq) & 7) << 4);
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

  // ---- software pipeline: NBUF-1 samples in flight behind the one being computed.
  // registers (NBUF == 2): ids one iteration ahead of their rows; ring (NBUF > 2): iteration `it` submits the ids
  // of sample it+A, issues the rows of sample it+NBUF-1, computes sample it — the first A iterations only fill.
  RawIdx raw_pref{0u, 0u, 0u};
  if (!IDS) {
    raw_pref = load_raw();
#pragma unroll
    for (int i = 0; i < NBUF - 1; ++i) {
      const RawIdx cur = raw_pref;
      raw_pref = load_raw();
      issue(cur);
    }
  }
  int k_cmp = warp;
  uint32_t buf_cmp = 0;
  for (int it = IDS ? -A : 0; it < n_iter; ++it) {
    if (IDS) {
      submit_ids();
      if (it + NBUF - 1 >= 0) issue(read_ids());
      else cp_async_commit();
    } else {
      const RawIdx cur = raw_pref;
      raw_pref = load_raw();
      issue(cur);  // refills the buffer consumed (and used as output stage) in the previous iteration
    }
    cp_async_wait<NBUF - 1>();
    __syncwarp();
    if (IDS && it < 0) continue;
    const uint32_t xs = wbase + buf_cmp;
    buf_cmp += p.buf_bytes;
    if (buf_cmp == NBUF * p.buf_bytes) buf_cmp = 0;
    if (k_cmp < n_cta) {
      float acc[6][4];
#pragma unroll
      for (int ti = 0; ti < 6; ++ti)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[ti][c] = 0.0f;

      if (PS) {
        const uint32_t a0b = xs + la[0], a1b = xs + la[1], b0b = xs + lb[0], b1b = xs + lb[1];
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
          const uint32_t kx = 32u * ks;
          ldsm_x4(a0b ^ kx, ah[0][0], ah[0][1], ah[0][2], ah[0][3]);
          ldsm_x4((a0b ^ kx) + 128u, al[0][0], al[0][1], al[0][2], al[0][3]);
          ldsm_x4(a1b ^ kx, ah[1][0], ah[1][1], ah[1][2], ah[1][3]);
          ldsm_x4((a1b ^ kx) + 128u, al[1][0], al[1][1], al[1][2], al[1][3]);
          ldsm_x4(b0b ^ kx, bh[0][0], bh[0][1], bh[1][0], bh[1][1]);
          ldsm_x4((b0b ^ kx) + 128u, bl[0][0], bl[0][1], bl[1][0], bl[1][1]);
          ldsm_x4(b1b ^ kx, bh[2][0], bh[2][1], bh[3][0], bh[3][1]);
          ldsm_x4((b1b ^ kx) + 128u, bl[2][0], bl[2][1], bl[3][0], bl[3][1]);
#pragma unroll
          for (int ti = 0; ti < 6; ++ti) {
            const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
            mma_bf16_16816(acc[ti], ah[mt][0], ah[mt][1], ah[mt][2], ah[mt][3], bl[nt][0], bl[nt][1]);
          }
#pragma unroll
          for (int ti = 0; ti < 6; ++ti) {
            const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
            mma_bf16_16816(acc[ti], al[mt][0], al[mt][1], al[mt][2], al[mt][3], bh[nt][0], bh[nt][1]);
          }
#pragma unroll
          for (int ti = 0; ti < 6; ++ti) {
            const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
            mma_bf16_16816(acc[ti], ah[mt][0], ah[mt][1], ah[mt][2], ah[mt][3], bh[nt][0], bh[nt][1]);
          }
        }
      } else {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        uint32_t h[4][2], l[4][2];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 v = lds128(xs + ((ks & 1) ? po[q] : pe[q]) + 64u * ks);
          split_pair(v.x, v.y, h[q][0], l[q][0]);
          split_pair(v.z, v.w, h[q][1], l[q][1]);
        }
        // tile (mt, nt): A = rows q = 2mt, 2mt+1; B (n-tile nt = rows 8nt + g) = the registers of q = nt.
        // Pass-major order: six independent accumulators between dependent MMAs.
#pragma unroll
        for (int ti = 0; ti < 6; ++ti) {
          const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
          mma_bf16_16816(acc[ti], h[2 * mt][0], h[2 * mt + 1][0], h[2 * mt][1], h[2 * mt + 1][1], l[nt][0], l[nt][1]);
        }
#pragma unroll
        for (int ti = 0; ti < 6; ++ti) {
          const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
          mma_bf16_16816(acc[ti], l[2 * mt][0], l[2 * mt + 1][0], l[2 * mt][1], l[2 * mt + 1][1], h[nt][0], h[nt][1]);
        }
#pragma unroll
        for (int ti = 0; ti < 6; ++ti) {
          const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
          mma_bf16_16816(acc[ti], h[2 * mt][0], h[2 * mt + 1][0], h[2 * mt][1], h[2 * mt + 1][1], h[nt][0], h[nt][1]);
        }
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
          for (int e = (n4 << 2) + lane; e < OW; e += 32) {
            float v;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(xs + (uint32_t)e * 4u));
            of32[e] = v;
          }
        } else {
          for (int e = lane; e < OW; e += 32) {
            float v;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(xs + (uint32_t)e * 4u));
            of32[e] = v;
          }
        }
      }
    }
    k_cmp += nw;
    if (osplit) osplit += (long long)nw * 2 * p.out_Kp;
    if (of32) of32 += (long long)nw * p.out_stride;
    __syncwarp();  // the buffer may be refilled by the next iteration's copies
  }
}

static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}

template <int MODE, int KD, int NWARPS, bool PS, int NBUF>
static int launch_kd(const LookupParams& lk, const Params& p, size_t smem, unsigned grid, cudaStream_t st, const char* who) {
  auto kern = interact_v2_kernel<MODE, KD, NWARPS, PS, NBUF>;
  static bool attr_set[64] = {};  // per device: function attributes belong to the device's copy of the kernel
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute failed: %s", who, cudaGetErrorString(e));
      return (int)e;
    }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
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
  bool remote = false;
  if (MODE == 1 && lk.world > 1)
    for (int r = 0; r < rows; ++r) remote = remote || lk.sharded[r];
  static int nbuf_env = -2;
  if (nbuf_env == -2) nbuf_env = env_int("MM_IMMA_NBUF", 0);
  const int nbuf = (nbuf_env >= 2 && nbuf_env <= 4) ? nbuf_env : 2;
  (void)remote;
  const unsigned ring_bytes = nbuf > 2 ? (unsigned)(nbuf + 1) * 256u : 0u;  // per-warp id ring
  const unsigned per_warp = (unsigned)nbuf * p.buf_bytes + ring_bytes;
  const unsigned peer_bytes = (MODE == 1 && lk.world > 1) ? (unsigned)(rows * lk.world * 8) : 0u;
  const unsigned budget = 227u * 1024u - peer_bytes;
  static int warps_env = -2;
  if (warps_env == -2) warps_env = env_int("MM_IMMA_WARPS", 0);
  const int want_warps = warps_env > 0 ? warps_env : (nbuf == 4 ? 8 : nbuf == 3 ? 10 : 16);
  int warps = (int)(budget / per_warp);
  if (warps > want_warps) warps = want_warps;
  if (warps > 16) warps = 16;
  if (nbuf > 2 && warps > 12) warps = 12;
  if (warps < 2) return MM_ERR_UNSUPPORTED;
  p.n_warps = warps;
  p.ids_off = (unsigned)warps * nbuf * p.buf_bytes;
  p.peer_off = (unsigned)warps * per_warp;
  const size_t smem = (size_t)p.peer_off + peer_bytes;
  const long long sms = sm_count();
  long long want = (B + warps - 1) / warps;
  const unsigned grid = (unsigned)(want < sms ? want : sms);
  // instantiated variants: 16 (or 12) warps x 2 buffers; operand-format rows (presplit) only with 2 buffers;
  // 3 / 4 buffers (id ring) for experiments
#define MM_V2_LAUNCH(KD)                                                                                                \
  (nbuf == 4 ? launch_kd<MODE, KD, 12, false, 4>(lk, p, smem, grid, st, who)                                            \
   : nbuf == 3 ? launch_kd<MODE, KD, 12, false, 3>(lk, p, smem, grid, st, who)                                          \
   : (presplit && MODE == 1 && KD == 64)                                                                                \
       ? (warps > 12 ? launch_kd<1, 64, 16, true, 2>(lk, p, smem, grid, st, who) : launch_kd<1, 64, 12, true, 2>(lk, p, smem, grid, st, who)) \
       : (warps > 12 ? launch_kd<MODE, KD, 16, false, 2>(lk, p, smem, grid, st, who)                                    \
                     : launch_kd<MODE, KD, 12, false, 2>(lk, p, smem, grid, st, who)))
  if (presplit && nbuf != 2) return MM_ERR_UNSUPPORTED;
  switch (D) {
    case 16: return MM_V2_LAUNCH(16);
    case 32: return MM_V2_LAUNCH(32);
    case 64: return MM_V2_LAUNCH(64);
    default: return MM_V2_LAUNCH(128);
  }
#undef MM_V2_LAUNCH
}

template int launch<0>(const float*, int64_t, const LookupParams&, const float*, int64_t, int, int, int64_t, int, int,
                       float*, int64_t, void*, int, int32_t*, cudaStream_t, const char*, bool);
template int launch<1>(const float*, int64_t, const LookupParams&, const float*, int64_t, int, int, int64_t, int, int,
                       float*, int64_t, void*, int, int32_t*, cudaStream_t, const char*, bool);

}  // namespace imma2
}  // namespace mm
