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

template <typename T>
__device__ __forceinline__ long long load_index(const void* p, long long i) {
  return (long long)reinterpret_cast<const T*>(p)[i];
}

}  // namespace mm
