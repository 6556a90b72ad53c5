// IndexedSlices added into a dense (N, D) gradient: dense[ids[i]] += rows[i] for every i, duplicates folded in index order.
//
// The weight-tied catalog step's table gradient is the sum of the output side's dense dE (N, D) and the input side's
// IndexedSlices (one row per lookup, duplicates included).  Each row of `dense` must have ONE writer and its duplicates a
// fixed summation order, so that a repeated step (and a CUDA-graph replay) is bit-identical: the sparse update's election
// fold (train_sparse.cu) adds a row's third and later duplicates with float vector reds in whatever order warps arrive, so
// it does not fit here.  Instead the (id, index) pairs are put in id order by a stable LSD radix sort (8-bit digits, only
// as many passes as N needs), then each run of equal ids is summed in index order in fixed-size pieces whose partials are
// added in piece order, and the sum goes to its row of `dense`.  Integer shared-memory atomics count digits; no float atomics anywhere.
//
//   keys_init     key = id (N for an id outside [0, N): sorted last, never added), value = index
//   radix_hist    per 2048-entry tile and digit: the count           -> hist[digit][tile]
//   radix_scan    one CTA: exclusive scan of hist in digit-major order (stable across tiles)
//   radix_scatter per tile: each entry's rank among the tile's equal digits, in index order (__match_any_sync per warp,
//                 per-warp counts in shared memory), written to hist + rank
//   segment_sum   D/4 lanes per sorted position; runs of equal ids are cut into segments at fixed 256-position chunks of
//                 the sorted order, and the first position of each segment sums it in index order: a run inside one chunk
//                 updates its dense row, a longer one leaves one partial per chunk
//   chunk_combine the head chunk of each longer run adds its partials in chunk order and updates the dense row, so the
//                 serial work of a run of length r is at most 256 + r / 256 row additions (a padding id or a popular item
//                 does not serialise the merge)
#include <climits>

#include "mm_common.cuh"

namespace mm {
namespace sld {

constexpr int THREADS = 256;
constexpr int PER = 8;                     // entries per thread and tile
constexpr int TILE = THREADS * PER;        // entries per tile
constexpr int WARPS = THREADS / 32;
constexpr int CHUNK = 256;                 // sorted positions per segment: the longest serial sum of one group
constexpr int MAX_D = 128;

__global__ void keys_init_kernel(const void* __restrict__ ids, int idx_bytes, long long n, long long N, int* __restrict__ keys,
                                 int* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long id = load_id(ids, idx_bytes, i);
  keys[i] = (id >= 0 && id < N) ? (int)id : (int)N;
  vals[i] = (int)i;
}

__global__ void __launch_bounds__(THREADS) radix_hist_kernel(const int* __restrict__ keys, long long n, int shift,
                                                             int* __restrict__ hist, int ntiles) {
  __shared__ int cnt[256];
  cnt[threadIdx.x] = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * TILE;
#pragma unroll
  for (int r = 0; r < PER; ++r) {
    const long long i = base + r * THREADS + threadIdx.x;
    if (i < n) atomicAdd(&cnt[(keys[i] >> shift) & 255], 1);
  }
  __syncthreads();
  hist[(long long)threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
}

// Exclusive scan of m ints in place by one CTA of 1024 threads: each thread owns a contiguous span.
__global__ void __launch_bounds__(1024) radix_scan_kernel(int* __restrict__ hist, long long m) {
  __shared__ int part[1024];
  const long long span = (m + 1023) / 1024;
  const long long a = threadIdx.x * span, e = min(m, a + span);
  int s = 0;
  for (long long i = a; i < e; ++i) s += hist[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {  // inclusive Hillis-Steele scan of the partial sums
    const int v = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  int run = part[threadIdx.x] - s;
  for (long long i = a; i < e; ++i) {
    const int v = hist[i];
    hist[i] = run;
    run += v;
  }
}

__global__ void __launch_bounds__(THREADS) radix_scatter_kernel(const int* __restrict__ keys_in, const int* __restrict__ vals_in,
                                                                long long n, int shift, const int* __restrict__ hist, int ntiles,
                                                                int* __restrict__ keys_out, int* __restrict__ vals_out) {
  __shared__ int base[256];
  __shared__ int wcnt[WARPS][256];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  base[tid] = hist[(long long)tid * ntiles + blockIdx.x];
  const unsigned lt = (1u << lane) - 1u;
  const long long t0 = (long long)blockIdx.x * TILE;
  for (int r = 0; r < PER; ++r) {
#pragma unroll
    for (int w = 0; w < WARPS; ++w) wcnt[w][tid] = 0;
    const long long i = t0 + r * THREADS + tid;  // entries in index order: round, then warp, then lane
    const bool on = i < n;
    const int k = on ? keys_in[i] : 0;
    const int v = on ? vals_in[i] : 0;
    const int digit = on ? (k >> shift) & 255 : 256;  // past the end: a digit of its own, never written
    const unsigned peers = __match_any_sync(0xffffffffu, digit);
    const int rank = __popc(peers & lt);
    __syncthreads();  // wcnt cleared; base updated by the previous round
    if (on && rank == 0) wcnt[warp][digit] = __popc(peers);
    __syncthreads();
    if (on) {
      int pos = base[digit] + rank;
      for (int w = 0; w < warp; ++w) pos += wcnt[w][digit];
      keys_out[pos] = k;
      vals_out[pos] = v;
    }
    __syncthreads();
    int add = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) add += wcnt[w][tid];
    base[tid] += add;
  }
}

__device__ __forceinline__ void add4(float4& a, const float4& b) {
  a.x += b.x;
  a.y += b.y;
  a.z += b.z;
  a.w += b.w;
}

// One group of 2^lgL lanes (one float4 each, lanes past D/4 idle) per sorted position.  A segment is a run of equal ids cut
// at the CHUNK boundaries of the sorted order; its first position sums it (at most CHUNK rows, in index order).  A run
// inside one chunk goes straight to its dense row.  A run that crosses chunks leaves its head segment's sum in part_last
// of the head's chunk and each continuation segment's sum in part_first of its chunk, for chunk_combine_kernel.
__global__ void __launch_bounds__(THREADS) segment_sum_kernel(const int* __restrict__ keys, const int* __restrict__ vals,
                                                              long long n, long long N, const float* __restrict__ rows, int D,
                                                              int lgL, float* __restrict__ dense, float* __restrict__ part_first,
                                                              float* __restrict__ part_last) {
  const long long s = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> lgL;
  const int c = threadIdx.x & ((1 << lgL) - 1);
  if (s >= n || c >= (D >> 2)) return;
  const int k = keys[s];
  if (k >= N) return;  // an id outside [0, N)
  const bool run_head = s == 0 || keys[s - 1] != k;
  if (!run_head && s % CHUNK != 0) return;  // inside a segment
  const long long chunk = s / CHUNK, end = min(n, (chunk + 1) * CHUNK);
  float4 acc = *reinterpret_cast<const float4*>(rows + (long long)vals[s] * D + 4 * c);
  long long j = s + 1;
  for (; j < end && keys[j] == k; ++j) add4(acc, *reinterpret_cast<const float4*>(rows + (long long)vals[j] * D + 4 * c));
  const bool continues = j == end && end < n && keys[end] == k;
  if (run_head && !continues) {
    float4* out = reinterpret_cast<float4*>(dense + (long long)k * D + 4 * c);
    float4 d = *out;
    add4(d, acc);
    *out = d;
  } else {
    *reinterpret_cast<float4*>((run_head ? part_last : part_first) + chunk * D + 4 * c) = acc;
  }
}

// One group per chunk whose last run goes on into the next chunk and starts in this one: that run's head partial, then
// the continuation partials of the following chunks in chunk order, into its dense row (the run's only writer).
__global__ void __launch_bounds__(THREADS) chunk_combine_kernel(const int* __restrict__ keys, long long n, long long N, int D,
                                                                int lgL, const float* __restrict__ part_first,
                                                                const float* __restrict__ part_last, float* __restrict__ dense) {
  const long long ch = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> lgL;
  const int c = threadIdx.x & ((1 << lgL) - 1);
  const long long first = ch * CHUNK, last = min(n, first + CHUNK) - 1;
  if (first >= n || c >= (D >> 2) || last + 1 >= n) return;
  const int k = keys[last];
  if (k >= N || keys[last + 1] != k || (first > 0 && keys[first - 1] == k)) return;
  float4 acc = *reinterpret_cast<const float4*>(part_last + ch * D + 4 * c);
  for (long long c2 = ch + 1; c2 * CHUNK < n && keys[c2 * CHUNK] == k; ++c2)
    add4(acc, *reinterpret_cast<const float4*>(part_first + c2 * D + 4 * c));
  float4* out = reinterpret_cast<float4*>(dense + (long long)k * D + 4 * c);
  float4 d = *out;
  add4(d, acc);
  *out = d;
}

struct Layout {
  long long keys0, vals0, keys1, vals1, hist, part_first, part_last, total;
  int ntiles;
};
static Layout layout(long long n) {
  auto al = [](long long b) { return (b + 255) / 256 * 256; };
  Layout L;
  L.ntiles = (int)((n + TILE - 1) / TILE);
  const long long v = al(4 * n);
  L.keys0 = 0;
  L.vals0 = v;
  L.keys1 = 2 * v;
  L.vals1 = 3 * v;
  L.hist = 4 * v;
  const long long part = al(4LL * MAX_D * ((n + CHUNK - 1) / CHUNK));  // one partial row per chunk, sized for D <= 128
  L.part_first = L.hist + al(4LL * 256 * L.ntiles);
  L.part_last = L.part_first + part;
  L.total = L.part_last + part;
  return L;
}

}  // namespace sld
}  // namespace mm

extern "C" {

int64_t mm_slices_add_dense_workspace_bytes(int64_t n) { return n <= 0 ? 0 : (int64_t)mm::sld::layout(n).total; }

int mm_slices_add_dense(const void* ids, int idx_dtype, const float* rows, int64_t n, int D, float* dense, int64_t N,
                        void* workspace, int64_t workspace_bytes, void* stream) {
  using namespace mm;
  using namespace mm::sld;
  MM_REQUIRE(n >= 0 && N > 0 && dense && (n == 0 || (ids && rows && workspace)), MM_ERR_ARG,
             "mm_slices_add_dense: null pointer or negative size");
  MM_REQUIRE(idx_dtype == MM_I32 || idx_dtype == MM_I64, MM_ERR_ARG, "mm_slices_add_dense: ids must be int32 or int64");
  MM_REQUIRE(D >= 4 && D <= 128 && (D & 3) == 0, MM_ERR_UNSUPPORTED, "mm_slices_add_dense: D=%d (needs D %% 4 == 0, 4 <= D <= 128)", D);
  MM_REQUIRE(n < (int64_t)INT_MAX && N < (int64_t)INT_MAX, MM_ERR_UNSUPPORTED, "mm_slices_add_dense: n and N must be below 2^31");
  MM_REQUIRE((((uintptr_t)rows | (uintptr_t)dense | (uintptr_t)workspace) & 15) == 0, MM_ERR_ALIGN,
             "mm_slices_add_dense: 16-byte alignment");
  if (n == 0) return MM_OK;
  const Layout L = layout(n);
  MM_REQUIRE(workspace_bytes >= L.total, MM_ERR_ARG, "mm_slices_add_dense: workspace of %lld bytes, %lld needed",
             (long long)workspace_bytes, (long long)L.total);
  char* ws = static_cast<char*>(workspace);
  int* keys[2] = {reinterpret_cast<int*>(ws + L.keys0), reinterpret_cast<int*>(ws + L.keys1)};
  int* vals[2] = {reinterpret_cast<int*>(ws + L.vals0), reinterpret_cast<int*>(ws + L.vals1)};
  int* hist = reinterpret_cast<int*>(ws + L.hist);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  keys_init_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ids, idx_dtype == MM_I64 ? 8 : 4, n, N, keys[0], vals[0]);
  if ((rc = check_launch("mm_slices_add_dense(keys)"))) return rc;
  int bits = 1;  // keys lie in [0, N]
  while (bits < 31 && (1LL << bits) <= N) ++bits;
  int cur = 0;
  for (int shift = 0; shift < bits; shift += 8, cur ^= 1) {
    radix_hist_kernel<<<L.ntiles, THREADS, 0, st>>>(keys[cur], n, shift, hist, L.ntiles);
    if ((rc = check_launch("mm_slices_add_dense(hist)"))) return rc;
    radix_scan_kernel<<<1, 1024, 0, st>>>(hist, 256LL * L.ntiles);
    if ((rc = check_launch("mm_slices_add_dense(scan)"))) return rc;
    radix_scatter_kernel<<<L.ntiles, THREADS, 0, st>>>(keys[cur], vals[cur], n, shift, hist, L.ntiles, keys[cur ^ 1], vals[cur ^ 1]);
    if ((rc = check_launch("mm_slices_add_dense(scatter)"))) return rc;
  }
  int lgL = 0;
  while ((1 << lgL) < D / 4) ++lgL;
  float* part_first = reinterpret_cast<float*>(ws + L.part_first);
  float* part_last = reinterpret_cast<float*>(ws + L.part_last);
  segment_sum_kernel<<<(unsigned)((n * (1LL << lgL) + THREADS - 1) / THREADS), THREADS, 0, st>>>(keys[cur], vals[cur], n, N, rows,
                                                                                                D, lgL, dense, part_first, part_last);
  if ((rc = check_launch("mm_slices_add_dense(segments)"))) return rc;
  const long long chunks = (n + CHUNK - 1) / CHUNK;
  chunk_combine_kernel<<<(unsigned)((chunks * (1LL << lgL) + THREADS - 1) / THREADS), THREADS, 0, st>>>(keys[cur], n, N, D, lgL,
                                                                                                       part_first, part_last, dense);
  return check_launch("mm_slices_add_dense(combine)");
}

}  // extern "C"
