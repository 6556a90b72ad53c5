// Shared helpers for the sm_90a kernels behind include/mm_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/mm_b200.h"

namespace mm {

// thread-local error text + process-wide launch counter (cabi.cu)
void set_error(const char* fmt, ...);
void count_launch(int n = 1);
int check_launch(const char* what);  // cudaGetLastError -> return code (0 or >0)
int sm_count();

#define MM_REQUIRE(cond, code, ...)  \
  do {                               \
    if (!(cond)) {                   \
      ::mm::set_error(__VA_ARGS__);  \
      return (code);                 \
    }                                \
  } while (0)

// ---- 128-bit streaming accesses (Guideline 13: vectorise; rows are touched once) -------
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void stg_stream(float4* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Keras activations (tf.keras.activations.*); exact (non-fast-math) forms.
// linear / relu are inlined; the transcendental ones live in ONE out-of-line function so that
// unrolled epilogues do not replicate ~3 KB of libm code per element (that blew the instruction
// cache: 110 KB of SASS and ~600 cycles per element in the first tensor-core epilogue).
static __device__ __noinline__ float apply_act_slow(float v, int act) {
  switch (act) {
    case MM_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
    case MM_ACT_TANH: return tanhf(v);
    case MM_ACT_SELU: {
      const float alpha = 1.6732632423543772f, scale = 1.0507009873554805f;
      return v > 0.0f ? scale * v : scale * alpha * expm1f(v);
    }
    case MM_ACT_ELU: return v > 0.0f ? v : expm1f(v);
    case MM_ACT_GELU: return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    default: return v;
  }
}
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == MM_ACT_RELU) return fmaxf(v, 0.0f);
  if (act == MM_ACT_LINEAR) return v;
  return apply_act_slow(v, act);
}

// Prediction of an output head from its logit z, as mm_heads_fwd_bwd writes it: z (MM_LOSS_MSE) or the |z|-stable sigmoid
// (MM_LOSS_BCE).  mm_metrics_update evaluates the same code, so its sigmoid is bit-identical to that forward's.
__device__ __forceinline__ float head_pred(int kind, float z) {
  if (kind == MM_LOSS_MSE) return z;
  const float e = expf(-fabsf(z));
  return z >= 0.0f ? 1.0f / (1.0f + e) : e / (1.0f + e);
}

// Loss term l and dloss/dz g of an output head from its logit z and target y, before the loss weight, the sample weight
// and 1/B: BCE on the logit (MM_LOSS_BCE, BinaryOutput) or squared error (MM_LOSS_MSE, RegressionOutput).  Every kernel
// that fuses a head's loss (mm_heads_fwd_bwd, the DeepFM, Wide&Deep and MMoE heads) evaluates this one code.
__device__ __forceinline__ void head_loss(int kind, float z, float y, float& l, float& g) {
  if (kind == MM_LOSS_MSE) {
    const float d = z - y;
    l = d * d;
    g = 2.0f * d;
  } else {
    const float e = expf(-fabsf(z));
    l = fmaxf(z, 0.0f) - z * y + log1pf(e);
    const float sig = z >= 0.0f ? 1.0f / (1.0f + e) : e / (1.0f + e);
    g = sig - y;
  }
}

// per-launch table list, passed by value in kernel parameter space (2 KB)
struct GatherParams {
  mm_gather_table t[MM_MAX_TABLES];
  int n_tables;
};

// Lookup descriptor of the fused lookup + interaction kernel (interaction_v2.cu), indexed by STAGED ROW
// (= feature slot); passed by value in kernel parameter space (2.9 KB)
constexpr int MM_LOOKUP_MAX_ROWS = 32;
constexpr int MM_LOOKUP_MAX_WORLD = 8;
struct LookupParams {
  const float* weights[MM_LOOKUP_MAX_ROWS];  // full table (replicated) or this rank's shard; null: not a table row
  const void* indices[MM_LOOKUP_MAX_ROWS];
  long long rows[MM_LOOKUP_MAX_ROWS];  // GLOBAL row count
  const float* peers[MM_LOOKUP_MAX_ROWS * MM_LOOKUP_MAX_WORLD];  // [row * world + rank] shard pointers (sharded rows)
  unsigned char idx_bytes[MM_LOOKUP_MAX_ROWS];  // 1, 2, 3 (unsigned), 4, 8 (signed)
  unsigned char sharded[MM_LOOKUP_MAX_ROWS];
  int world, log2_world;  // log2_world = -1: world is not a power of two
};

// Host checks of C-ABI input (cabi.cu).  Each returns MM_OK, or sets the error text (prefixed by `who`) and returns its code.
// One packed id column of table t: non-null, idx_bytes in {1, 2, 3, 4, 8}, rows > 0 and all addressable by a narrow
// width, 4- and 8-byte ids aligned to their width.
int check_id_column(const char* who, int t, const void* indices, int idx_bytes, long long rows);
// An mm_lookup_table array -> `lk` by staged row (= slot), on top of the caller's zeroed lk.world / lk.log2_world:
// slots in [0, F) and used once (with `bottom_slot`, -1: none), 16-byte aligned weights, check_id_column, and shard
// pointers for row-sharded tables (lk.world > 1 and sharded_ok; otherwise such a table is refused).
int fill_lookup_params(const char* who, const mm_lookup_table* tables, int n_tables, int F, int bottom_slot, int rank,
                       bool sharded_ok, LookupParams& lk);

template <typename T>
__device__ __forceinline__ long long load_index(const void* p, long long i) {
  return (long long)reinterpret_cast<const T*>(p)[i];
}

// Id s of a packed id column (mm_lookup_table.idx_bytes): 1, 2, 3 (unsigned, little-endian), 4 or 8 (signed) bytes.
__device__ __forceinline__ long long load_id(const void* base, int w, long long s) {
  switch (w) {
    case 1: return (long long)reinterpret_cast<const uint8_t*>(base)[s];
    case 2: return (long long)reinterpret_cast<const uint16_t*>(base)[s];
    case 3: {
      const uint8_t* b = reinterpret_cast<const uint8_t*>(base) + 3 * s;
      return (long long)b[0] | ((long long)b[1] << 8) | ((long long)b[2] << 16);
    }
    case 8: return reinterpret_cast<const long long*>(base)[s];
    default: return (long long)reinterpret_cast<const int32_t*>(base)[s];
  }
}

// Element i of an input column (mm_concat_piece.dtype, BCE targets) as fp32.  NC_F32: fp32 columns are read through the
// read-only data cache (__ldg).
template <bool NC_F32 = false>
__device__ __forceinline__ float load_as_f32(const void* src, long long i, int dtype) {
  switch (dtype) {
    case MM_I32: return (float)reinterpret_cast<const int32_t*>(src)[i];
    case MM_I64: return (float)reinterpret_cast<const long long*>(src)[i];
    case MM_F64: return (float)reinterpret_cast<const double*>(src)[i];
    default: return NC_F32 ? __ldg(reinterpret_cast<const float*>(src) + i) : reinterpret_cast<const float*>(src)[i];
  }
}

}  // namespace mm
