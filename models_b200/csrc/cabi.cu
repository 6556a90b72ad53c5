// Library-wide state of the C-ABI (include/mm_b200.h): error text, launch counter, version,
// the checks of id columns and lookup-table descriptors shared by the entry points, and the
// deterministic table initialiser.
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

int check_id_column(const char* who, int t, const void* indices, int w, long long rows) {
  MM_REQUIRE(indices && rows > 0, MM_ERR_ARG, "%s: table %d: null ids or rows <= 0", who, t);
  MM_REQUIRE(w == 1 || w == 2 || w == 3 || w == 4 || w == 8, MM_ERR_ARG, "%s: table %d: idx_bytes must be 1, 2, 3, 4 or 8", who, t);
  MM_REQUIRE(w >= 4 || rows <= (1ll << (8 * w)), MM_ERR_ARG, "%s: table %d: %lld rows do not fit %d-byte ids", who, t, rows, w);
  MM_REQUIRE((w != 4 && w != 8) || ((uintptr_t)indices % w) == 0, MM_ERR_ALIGN, "%s: table %d: misaligned ids", who, t);
  return MM_OK;
}

int fill_lookup_params(const char* who, const mm_lookup_table* tables, int n_tables, int F, int bottom_slot, int rank,
                       bool sharded_ok, LookupParams& lk) {
  unsigned seen = bottom_slot >= 0 ? (1u << bottom_slot) : 0u;
  for (int t = 0; t < n_tables; ++t) {
    const mm_lookup_table& tb = tables[t];
    const int r = tb.slot;
    MM_REQUIRE(tb.weights && r >= 0 && r < F, MM_ERR_ARG, "%s: table %d: null weights or slot %d outside [0, %d)", who, t, r, F);
    MM_REQUIRE(!(seen & (1u << r)), MM_ERR_ARG, "%s: slot %d used twice", who, r);
    seen |= 1u << r;
    MM_REQUIRE(((uintptr_t)tb.weights % 16) == 0, MM_ERR_ALIGN, "%s: table %d: weights must be 16-byte aligned", who, t);
    if (const int rc = check_id_column(who, t, tb.indices, tb.idx_bytes, tb.rows)) return rc;
    lk.weights[r] = tb.weights;
    lk.indices[r] = tb.indices;
    lk.rows[r] = tb.rows;
    lk.idx_bytes[r] = (unsigned char)tb.idx_bytes;
    if (tb.peer_weights_host) {
      MM_REQUIRE(sharded_ok, MM_ERR_UNSUPPORTED, "%s: row-sharded tables are not supported", who);
      MM_REQUIRE(lk.world > 1, MM_ERR_ARG, "%s: table %d is sharded but world == 1", who, t);
      lk.sharded[r] = 1;
      for (int k = 0; k < lk.world; ++k) {
        MM_REQUIRE(tb.peer_weights_host[k] && ((uintptr_t)tb.peer_weights_host[k] % 16) == 0, MM_ERR_ARG,
                   "%s: table %d: null / misaligned shard pointer of rank %d", who, t, k);
        lk.peers[r * lk.world + k] = tb.peer_weights_host[k];
      }
      MM_REQUIRE(tb.peer_weights_host[rank] == tb.weights, MM_ERR_ARG, "%s: table %d: peer_weights_host[rank] != weights", who, t);
    }
  }
  return MM_OK;
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
