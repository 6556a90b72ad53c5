// DLRM pairwise interaction on tensor cores, one warp per sample — FIRST-GENERATION kernel, kept for A/B measurements
// (MM_IMMA_V1=1) and as the fallback of the legacy entry points; the product path is interaction_v2.cu.
//
// The per-sample Gram matrix X X^T (X = F x D, F <= 32) is far too small for wgmma (M >= 64 per
// instruction would waste > 4x on block-diagonal padding), so it runs on the warp-level
// mma.sync.m16n8k16 bf16 path with the same 3-pass split as the dense layers (hi*lo + lo*hi + hi*hi,
// fp32 accumulate).  It is NOT HBM-bound but instruction-issue bound — the v2 kernel cuts the instruction count in half.
//
// Data movement: rows go from the embedding tables — or the stacked (B,F,D) tensor — straight
// into a padded shared-memory tile with 16-byte cp.async (LDGSTS: no register staging, zero-fill
// for out-of-range ids), one commit group per sample; each warp keeps NBUF-1 samples in flight
// while it computes one.  (A first version issued one cp.async.bulk per row: UBLKCP takes uniform
// registers, so the compiler serialised the 27 per-lane copies through an ELECT/R2UR loop that
// cost a large share of the issue slots.)
// Because B = X^T, the B fragments of n-tile nt ARE registers of the A fragment of m-tile nt/2, so X
// is read from shared memory once per k-step.  The output row [prefix | upper triangle] is assembled
// in shared memory and written coalesced, either as fp32 or directly as the split-bf16 operand
// (M, 2*Kp) of the top MLP's first tensor-core layer.
//
// Replaces: StackFeatures + DotProductInteraction + shortcut concat
// (merlin/models/tf/core/aggregation.py:101-108, blocks/interaction.py:86-116, blocks/dlrm.py:126-130).
#include <cuda_bf16.h>

#include <cstdlib>
#include <cstring>

#include "mm_common.cuh"

namespace mm {
namespace imma {

constexpr int MAX_WARPS = 12;

struct Params {
  // MODE 0: stacked input
  const float* x;
  long long x_stride;
  // prefix / bottom vector (P == 0 or P == D)
  const float* prefix;
  long long prefix_stride;
  int P;
  int bottom_slot;  // MODE 1: slot of the bottom vector inside the stack (-1: none)
  long long B;
  int F, D, T;
  int rows;  // rows staged per sample (F, or F+1 when MODE 0 carries a separate prefix row)
  float* out_f32;
  long long out_stride;
  __nv_bfloat16* out_split;
  int out_Kp;
  int* oob_count;
  int n_warps;
  unsigned per_warp_bytes, in_bytes;
  int log2V, log2D;  // V = D/4 float4 per row
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// 16-byte global -> shared copy; src_bytes = 0 zero-fills the destination (out-of-range id)
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// (x, y) -> packed bf16x2 hi (x in the low half) and the bf16x2 of the residuals
__device__ __forceinline__ void split_pair(float2 v, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(v.x, v.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  const float xh = __uint_as_float(hi << 16), yh = __uint_as_float(hi & 0xffff0000u);
  __nv_bfloat162 l = __floats2bfloat162_rn(v.x - xh, v.y - yh);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

template <int MODE, typename IdxT, int KD /* compile-time D (0 = runtime) */, int NBUF /* sample buffers per warp */>
__global__ void __launch_bounds__(32 * MAX_WARPS, 1)
interact_mma_kernel(const __grid_constant__ GatherParams gp, const Params p) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  // rows are stored unpadded (D floats) with the 16-byte chunk index XOR-swizzled by ((row & 3) << 1):
  // the 8-byte fragment loads of 4 consecutive rows then hit 8 distinct chunks (conflict-free)
  const int F = p.F, D = KD > 0 ? KD : p.D, DS = D, KS = D >> 4;
  uint8_t* wbase = smem_raw + (size_t)warp * p.per_warp_bytes;
  uint8_t* ostage = wbase + (size_t)NBUF * p.in_bytes;
  const int npairs = F * (F - 1) / 2;
  const int OW = p.P + npairs;

  // ---- one-time per warp: zeroed output staging, output offsets of this lane's accumulators
  {
    const int stage_words = (int)((p.per_warp_bytes - NBUF * p.in_bytes) >> 2);
    for (int i = lane; i < stage_words; i += 32) reinterpret_cast<uint32_t*>(ostage)[i] = 0u;
  }
  // accumulator tiles: (mt, nt) in {(0,0),(0,1),(0,2),(0,3),(1,2),(1,3)}; c0..c3 = (g,2t),(g,2t+1),(g+8,2t),(g+8,2t+1)
  int off[6][4];
#pragma unroll
  for (int ti = 0; ti < 6; ++ti) {
    const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int i = 16 * mt + g + ((c & 2) ? 8 : 0), j = 8 * nt + 2 * t + (c & 1);
      off[ti][c] = (i < j && j < F) ? p.P + i * (2 * F - i - 1) / 2 + (j - i - 1) : -1;
    }
  }
  int ro[2][2];  // shared-memory row offsets (floats) of this lane's fragment rows, clamped to staged rows
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) ro[mt][h] = min(16 * mt + g + 8 * h, F - 1) * DS;
  int sw[2][2];  // chunk swizzle of those rows
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) sw[mt][h] = ((min(16 * mt + g + 8 * h, F - 1) & 3) << 1) & ((D >> 2) - 1);
  __syncwarp();

  const long long gw = (long long)blockIdx.x * p.n_warps + warp;
  const long long wstride = (long long)gridDim.x * p.n_warps;
  const long long n_mine = gw < p.B ? (p.B - gw + wstride - 1) / wstride : 0;

  // lane r < T holds the id of table r for the sample being issued (MODE 1)
  const IdxT* my_idx_ptr = (MODE == 1 && lane < p.T) ? reinterpret_cast<const IdxT*>(gp.t[lane].indices) : nullptr;
  const long long my_rows = (MODE == 1 && lane < p.T) ? gp.t[lane].rows : 0;
  const int V = D >> 2;

  // raw (un-widened) index prefetch: the value is not touched until the next iteration, so the
  // global-load latency is hidden behind a whole sample of compute
  auto load_index = [&](long long it) -> IdxT {
    if (MODE == 1 && lane < p.T && it < n_mine) return my_idx_ptr[gw + it * wstride];
    return (IdxT)0;
  };
  // Per-lane row constants: lane r (< rows) owns staged row r.  Its destination inside a sample
  // buffer (byte offset of the slot + the slot's chunk swizzle) never changes; its source pointer is
  // computed once per sample by the owner and broadcast with shuffles in the copy loop, so the loop
  // body is 3 shuffles + a few integer ops + one LDGSTS per 16 bytes.
  int my_slot = lane;
  const float* my_base = nullptr;  // table base (MODE 1) — row-invariant part of the source
  if (MODE == 1 && lane < p.T) {
    my_slot = gp.t[lane].out_col >> p.log2D;
    my_base = gp.t[lane].weights;
  } else if (MODE == 1 && lane == p.T) {
    my_slot = p.bottom_slot;
  }
  // destination descriptor: (slot * DS * 4 bytes) | swizzle (low 3 bits; the offset is a multiple of 64 B)
  const uint32_t my_dst = (uint32_t)(my_slot * DS * 4) | (uint32_t)(((my_slot & 3) << 1) & (V - 1));

  auto issue = [&](long long it, IdxT idx_raw) {
    if (it < n_mine) {
      const long long s = gw + it * wstride;
      const int buf = (int)(it % NBUF);
      const uint32_t xs_u32 = smem_u32(wbase + (size_t)buf * p.in_bytes);
      // owner lanes: source row pointer and copy size (0 = zero fill)
      const float* my_src = my_base;
      uint32_t my_bytes = 16;
      if (MODE == 1) {
        if (lane < p.T) {
          const long long idx = (long long)idx_raw;
          if (idx >= 0 && idx < my_rows) my_src = my_base + (idx << p.log2D);
          else {
            my_bytes = 0;
            if (p.oob_count) atomicAdd(p.oob_count, 1);
          }
        } else {
          my_src = p.prefix + s * p.prefix_stride;
        }
      } else {
        my_src = lane < F ? p.x + s * p.x_stride + ((long long)lane << p.log2D) : p.prefix + s * p.prefix_stride;
      }
      const uint32_t src_lo = (uint32_t)(uintptr_t)my_src, src_hi = (uint32_t)((uintptr_t)my_src >> 32);
      const uint32_t my_info = my_dst | (my_bytes << 24);  // dst offset < 2^24, bytes in the top byte
      const int total = p.rows << p.log2V;
      const int v = lane & (V - 1), rsub = lane >> p.log2V;  // rows per step = 32 / V
      const int rstep = 32 >> p.log2V;
      for (int r0 = 0; r0 < p.rows; r0 += rstep) {  // warp-uniform trip count (shuffles inside)
        const int r = r0 + rsub;
        const bool act = r < p.rows;
        const int rr = act ? r : 0;
        const uint32_t lo = __shfl_sync(0xffffffffu, src_lo, rr);
        const uint32_t hi = __shfl_sync(0xffffffffu, src_hi, rr);
        const uint32_t info = __shfl_sync(0xffffffffu, my_info, rr);
        const float* src = reinterpret_cast<const float*>(((uintptr_t)hi << 32) | lo) + v * 4;
        const uint32_t dst = xs_u32 + (info & 0x00fffff8u) + (((uint32_t)v ^ (info & 7u)) << 4);
        if (act) cp_async16_zfill(dst, src, info >> 24);
      }
      (void)total;
    }
    cp_async_commit();  // one group per sample (empty past the end keeps the group count in step)
  };

  // ---- software pipeline: NBUF-1 samples in flight; indices fetched one iteration ahead of their rows
  IdxT idx_pref = load_index(0);
  for (int i = 0; i < NBUF - 1; ++i) {
    const IdxT idx_cur = idx_pref;
    idx_pref = load_index(i + 1);
    issue(i, idx_cur);
  }
  for (long long it = 0; it < n_mine; ++it) {
    {
      const IdxT idx_cur = idx_pref;
      idx_pref = load_index(it + NBUF);
      issue(it + NBUF - 1, idx_cur);  // refills the buffer consumed in the previous iteration
    }
    const long long s = gw + it * wstride;
    const int buf = (int)(it % NBUF);
    const float* xs = reinterpret_cast<const float*>(wbase + (size_t)buf * p.in_bytes);
    cp_async_wait<NBUF - 1>();  // this sample's group (the oldest of NBUF pending) has landed
    __syncwarp();

    float acc[6][4];
#pragma unroll
    for (int ti = 0; ti < 6; ++ti)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[ti][c] = 0.0f;

#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        // logical column k0 = 16ks + 2t (+8): chunk c = k0/4, swizzled by the row's (r & 3) << 1
        const int c0 = 4 * ks + (t >> 1), w = (t & 1) * 2;
        split_pair(*reinterpret_cast<const float2*>(xs + ro[mt][0] + (((c0) ^ sw[mt][0]) << 2) + w), ah[mt][0], al[mt][0]);
        split_pair(*reinterpret_cast<const float2*>(xs + ro[mt][1] + (((c0) ^ sw[mt][1]) << 2) + w), ah[mt][1], al[mt][1]);
        split_pair(*reinterpret_cast<const float2*>(xs + ro[mt][0] + (((c0 + 2) ^ sw[mt][0]) << 2) + w), ah[mt][2], al[mt][2]);
        split_pair(*reinterpret_cast<const float2*>(xs + ro[mt][1] + (((c0 + 2) ^ sw[mt][1]) << 2) + w), ah[mt][3], al[mt][3]);
      }
      // B fragment of n-tile nt = registers {nt&1, 2+(nt&1)} of the A fragment of m-tile nt>>1.
      // Pass-major order: six independent accumulators between dependent MMAs.
#pragma unroll
      for (int ti = 0; ti < 6; ++ti) {
        const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
        mma_bf16_16816(acc[ti], ah[mt], al[nt >> 1][nt & 1], al[nt >> 1][2 + (nt & 1)]);
      }
#pragma unroll
      for (int ti = 0; ti < 6; ++ti) {
        const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
        mma_bf16_16816(acc[ti], al[mt], ah[nt >> 1][nt & 1], ah[nt >> 1][2 + (nt & 1)]);
      }
#pragma unroll
      for (int ti = 0; ti < 6; ++ti) {
        const int mt = ti < 4 ? 0 : 1, nt = ti < 4 ? ti : ti - 2;
        mma_bf16_16816(acc[ti], ah[mt], ah[nt >> 1][nt & 1], ah[nt >> 1][2 + (nt & 1)]);
      }
    }

    // ---- assemble the fp32 output row in shared memory (one predicated 4-byte store per accumulator);
    // the split into bf16 (hi, lo) happens in the coalesced store pass, 8 columns per lane at a time
    {
      float* os = reinterpret_cast<float*>(ostage);
      if (p.P > 0) {
        const int prow = MODE == 1 ? p.bottom_slot : F;
        const float* pr = xs + prow * DS;
        for (int e = lane; e < p.P; e += 32) os[e] = pr[((((e >> 2) ^ (((prow & 3) << 1) & ((D >> 2) - 1)))) << 2) + (e & 3)];
      }
#pragma unroll
      for (int ti = 0; ti < 6; ++ti)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (off[ti][c] >= 0) os[off[ti][c]] = acc[ti][c];
    }
    __syncwarp();  // staging complete; also: every lane is done reading xs[buf]

    // ---- coalesced row store
    if (p.out_split) {
      // staging holds out_Kp floats (columns >= OW are the zero padding written once at kernel start)
      const float4* src = reinterpret_cast<const float4*>(ostage);
      __nv_bfloat16* drow = p.out_split + s * (2ll * p.out_Kp);
      const int groups = p.out_Kp >> 3;  // 8 columns = one 16-byte bf16 store for hi and one for lo
      for (int gidx = lane; gidx < groups; gidx += 32) {
        const float4 a = src[2 * gidx], b = src[2 * gidx + 1];
        uint32_t h[4], l[4];
        split_pair(make_float2(a.x, a.y), h[0], l[0]);
        split_pair(make_float2(a.z, a.w), h[1], l[1]);
        split_pair(make_float2(b.x, b.y), h[2], l[2]);
        split_pair(make_float2(b.z, b.w), h[3], l[3]);
        *reinterpret_cast<uint4*>(drow + 8 * gidx) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(drow + p.out_Kp + 8 * gidx) = make_uint4(l[0], l[1], l[2], l[3]);
      }
    } else if (p.out_f32) {
      const float* os = reinterpret_cast<const float*>(ostage);
      float* dst = p.out_f32 + s * p.out_stride;
      if (((p.out_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out_f32) & 15) == 0)) {
        const int n4 = OW >> 2;
        for (int e = lane; e < n4; e += 32) reinterpret_cast<float4*>(dst)[e] = reinterpret_cast<const float4*>(os)[e];
        for (int e = (n4 << 2) + lane; e < OW; e += 32) dst[e] = os[e];
      } else {
        for (int e = lane; e < OW; e += 32) dst[e] = os[e];
      }
    }
    __syncwarp();  // staging may be overwritten by the next sample
  }
}

// Returns MM_ERR_UNSUPPORTED (without touching the error text) when the fast path does not apply.
template <int MODE, typename IdxT>
int launch(const float* x, int64_t x_stride, const GatherParams& gp, const float* prefix, int64_t prefix_stride,
           int P, int bottom_slot, int64_t B, int F, int D, float* out_f32, int64_t out_stride, void* out_split,
           int out_Kp, int32_t* oob, cudaStream_t st, const char* who) {
  if (F < 2 || F > 32 || (D != 16 && D != 32 && D != 64 && D != 128)) return MM_ERR_UNSUPPORTED;
  if (P != 0 && P != D) return MM_ERR_UNSUPPORTED;
  if (out_f32 && out_split) return MM_ERR_UNSUPPORTED;
  const int rows = (MODE == 0 && P > 0) ? F + 1 : F;
  if (rows > 32) return MM_ERR_UNSUPPORTED;
  if (MODE == 1 && gp.n_tables + (bottom_slot >= 0 ? 1 : 0) != F) return MM_ERR_UNSUPPORTED;
  if (MODE == 0 && (((uintptr_t)x & 15) || (x_stride & 3))) return MM_ERR_UNSUPPORTED;
  if (P > 0 && (((uintptr_t)prefix & 15) || (prefix_stride & 3))) return MM_ERR_UNSUPPORTED;
  const int OW = P + F * (F - 1) / 2;
  // buffers per warp: gathers of random rows want 2 samples in flight behind the one being computed;
  // MM_IMMA_NBUF overrides for tuning
  static int nbuf_env = -1;
  if (nbuf_env < 0) {
    const char* e = getenv("MM_IMMA_NBUF");
    nbuf_env = e ? atoi(e) : 0;
  }
  const int NBUF = (nbuf_env == 2 || nbuf_env == 3) ? nbuf_env : 2;
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
  p.T = MODE == 1 ? gp.n_tables : 0;
  p.rows = rows;
  p.out_f32 = out_f32;
  p.out_stride = out_stride;
  p.out_split = (__nv_bfloat16*)out_split;
  p.out_Kp = out_Kp;
  p.oob_count = oob;
  p.in_bytes = (unsigned)(rows * D * 4);
  const unsigned stage = out_split ? (unsigned)(out_Kp * 4) : (unsigned)(((OW + 3) & ~3) * 4);  // fp32 row (+ zero padding)
  p.per_warp_bytes = (NBUF * p.in_bytes + stage + 127u) & ~127u;
  int warps = (int)((226u * 1024u) / p.per_warp_bytes);
  if (warps > MAX_WARPS) warps = MAX_WARPS;
  if (warps < 2) return MM_ERR_UNSUPPORTED;
  p.n_warps = warps;
  p.log2D = D == 16 ? 4 : D == 32 ? 5 : D == 64 ? 6 : 7;
  p.log2V = p.log2D - 2;
  const size_t smem = (size_t)warps * p.per_warp_bytes;
  auto kern = D == 64 ? (NBUF == 3 ? interact_mma_kernel<MODE, IdxT, 64, 3> : interact_mma_kernel<MODE, IdxT, 64, 2>)
                      : (NBUF == 3 ? interact_mma_kernel<MODE, IdxT, 0, 3> : interact_mma_kernel<MODE, IdxT, 0, 2>);
  static bool attr_set[2][2] = {{false, false}, {false, false}};
  if (!attr_set[D == 64][NBUF == 3]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute failed: %s", who, cudaGetErrorString(e));
      return (int)e;
    }
    attr_set[D == 64][NBUF == 3] = true;
  }
  long long want = (B + warps - 1) / warps;
  const long long sms = sm_count();
  const unsigned grid = (unsigned)(want < sms ? want : sms);
  kern<<<grid, 32 * warps, smem, st>>>(gp, p);
  return check_launch(who);
}

template int launch<0, int32_t>(const float*, int64_t, const GatherParams&, const float*, int64_t, int, int, int64_t,
                                int, int, float*, int64_t, void*, int, int32_t*, cudaStream_t, const char*);
template int launch<1, int32_t>(const float*, int64_t, const GatherParams&, const float*, int64_t, int, int, int64_t,
                                int, int, float*, int64_t, void*, int, int32_t*, cudaStream_t, const char*);
template int launch<1, int64_t>(const float*, int64_t, const GatherParams&, const float*, int64_t, int, int, int64_t,
                                int, int, float*, int64_t, void*, int, int32_t*, cudaStream_t, const char*);

}  // namespace imma
}  // namespace mm
