// The dropout mask of a training step: one counter-based hash per element, so the forward's epilogue draws it with no
// state and no stored mask, and a CUDA-graph replay draws a fresh one from the device-resident step counter.
//
//   (w0, w1, w2, w3) = Philox4x32-10(counter = (col, row, layer, step), key = (seed & 0xffffffff, seed >> 32))
//   keep = w0 >= threshold,  threshold = min(round(rate * 2^32), 2^32 - 1)
//
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) is the generator cuRAND and
// TensorFlow's stateless ops use; tests/dropout_mask.py is its numpy port (checked against the paper's known-answer
// vectors) and the device masks are compared with it bit for bit.
#pragma once

#include <cstdint>

namespace mm {
namespace drop {

__host__ __device__ __forceinline__ void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
  const uint64_t p = (uint64_t)a * (uint64_t)b;
  hi = (uint32_t)(p >> 32);
  lo = (uint32_t)p;
}

// word 0 of Philox4x32-10(c, k)
__host__ __device__ __forceinline__ uint32_t philox_w0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                       uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, lo0, hi1, lo1;
    mulhilo(0xD2511F53u, c0, hi0, lo0);
    mulhilo(0xCD9E8D57u, c2, hi1, lo1);
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// what the epilogue needs: the key, the step's counter word, the layer and the threshold
struct Mask {
  uint32_t k0, k1, step, layer, threshold;
  __host__ __device__ __forceinline__ bool keep(uint32_t row, uint32_t col) const {
    return philox_w0(col, row, layer, step, k0, k1) >= threshold;
  }
};

__host__ __device__ __forceinline__ uint32_t threshold_of(float rate) {
  const double t = (double)rate * 4294967296.0 + 0.5;
  return t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
}

}  // namespace drop
}  // namespace mm
