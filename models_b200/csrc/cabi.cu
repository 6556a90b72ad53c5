// Library-wide state of the C-ABI (include/mm_b200.h): error text, launch counter, version,
// and the deterministic table initialiser.
#include <atomic>
#include <cstdarg>
#include <cstring>

#include "mm_common.cuh"

namespace mm {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
    return (int)e;
  }
  count_launch(1);
  return MM_OK;
}

int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 132;  // H100 SXM
  }
  return cached;
}

// splitmix64 finaliser over (seed, element index): identical integer arithmetic in
// oracle/oracle.py:hash_uniform, so any row of a 10 GiB table can be regenerated on the host.
__global__ void init_uniform_hash_kernel(float* __restrict__ w, long long n, unsigned long long seed,
                                         float lo, float span) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    unsigned long long z = seed + (unsigned long long)(i + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    const float u = (float)(unsigned int)(z >> 40) * (1.0f / 16777216.0f);  // exact
    w[i] = __fadd_rn(lo, __fmul_rn(span, u));                               // no FMA contraction
  }
}

}  // namespace mm

extern "C" {

int mm_version(void) { return 100; }
const char* mm_last_error(void) { return mm::g_err; }
int64_t mm_launch_count(void) { return (int64_t)mm::g_launches.load(); }

int mm_init_uniform_hash(float* w, int64_t n, uint64_t seed, float lo, float hi, void* stream) {
  MM_REQUIRE(w != nullptr && n >= 0, MM_ERR_ARG, "mm_init_uniform_hash: null buffer or n<0");
  if (n == 0) return MM_OK;
  const int threads = 256;
  long long blocks = (n + threads - 1) / threads;
  const long long cap = (long long)mm::sm_count() * 32;
  if (blocks > cap) blocks = cap;
  mm::init_uniform_hash_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
      w, (long long)n, (unsigned long long)seed, lo, hi - lo);
  return mm::check_launch("mm_init_uniform_hash");
}

}  // extern "C"
