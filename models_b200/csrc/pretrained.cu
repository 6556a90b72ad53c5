// Pretrained embeddings (PretrainedEmbeddings, inputs/embedding.py:717-800, fed by the dataloader's EmbeddingOperator):
// rows of a device-resident (N, Dp) matrix looked up by a batch's ids, straight into their slot of the input block's
// concat x0, optionally through a trained Dense(d') projection in the same pass, and that projection's backward.
//   gather     one warp per sample row, 16-B loads and stores when everything is 4-float aligned
//   project    y = P[ids] W + b: 64x64 output tiles, the gathered rows staged 32 columns at a time in shared memory
//              (the (B, Dp) block never reaches HBM), fp32 FMAs in ascending k
//   backward   g = sum of the addends' slot columns (through the l2-norm backward when the slot is normalised), then
//              dW = P[ids]^T g over fixed row chunks into per-chunk partials, summed in chunk order with db = sum g
//              (no float atomics: repeats are bit-identical)
// A null `ids` reads row b of a dense (B, Dp) input instead of row ids[b].
#include "mm_common.cuh"

namespace mm {

constexpr int PT_BM = 64;  // output rows per tile (project) / weight rows per tile (backward)
constexpr int PT_BN = 64;  // output columns per tile
constexpr int PT_BK = 32;  // k (project) or samples (backward) staged per step
constexpr int PT_THREADS = 256;
constexpr int PT_MAX_ADDENDS = 4;

struct PtAddends {
  const float* p[PT_MAX_ADDENDS];
  long long stride[PT_MAX_ADDENDS];
  int n;
};

// Source row of sample b: ids[b] (-1 when out of range, counted once when `count`), or b itself without ids.
template <typename IdxT>
__device__ __forceinline__ long long pt_row(const IdxT* ids, long long b, long long rows, int* oob, bool count) {
  if (ids == nullptr) return b;
  const long long r = (long long)ids[b];
  if (r < 0 || r >= rows) {
    if (count && oob) atomicAdd(oob, 1);
    return -1;
  }
  return r;
}

template <typename IdxT, bool VEC>
__global__ void __launch_bounds__(PT_THREADS)
pretrained_gather_kernel(const float* __restrict__ P, long long rows, int Dp, long long p_stride,
                         const IdxT* __restrict__ ids, long long B, float* __restrict__ out, long long out_stride,
                         int* __restrict__ oob) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long b = warp0; b < B; b += n_warps) {
    const long long r = pt_row(ids, b, rows, oob, lane == 0);
    float* dst = out + b * out_stride;
    if (VEC) {
      const float4* src4 = reinterpret_cast<const float4*>(P + (r < 0 ? 0 : r) * p_stride);
      float4* dst4 = reinterpret_cast<float4*>(dst);
      for (int d = lane; d < (Dp >> 2); d += 32)
        stg_stream(dst4 + d, r >= 0 ? ldg_stream(src4 + d) : make_float4(0.f, 0.f, 0.f, 0.f));
    } else {
      for (int d = lane; d < Dp; d += 32) dst[d] = r >= 0 ? __ldg(P + r * p_stride + d) : 0.0f;
    }
  }
}

// y[b, n] = sum_k P[row(b), k] W[k, n] + bias[n] into out (B, N) at out_stride.  Tiles are visited row-tile major, so the
// column tiles of one row tile run on neighbouring CTAs and re-read the same gathered rows from L2.
template <typename IdxT>
__global__ void __launch_bounds__(PT_THREADS)
pretrained_project_kernel(const float* __restrict__ P, long long rows, int Dp, long long p_stride,
                          const IdxT* __restrict__ ids, long long B, const float* __restrict__ W,
                          const float* __restrict__ bias, int N, float* __restrict__ out, long long out_stride,
                          int* __restrict__ oob) {
  __shared__ __align__(16) float As[PT_BK][PT_BM + 4];  // As[k][m]: the gathered rows, transposed
  __shared__ __align__(16) float Ws[PT_BK][PT_BN];
  __shared__ long long rid[PT_BM];
  const int t = threadIdx.x;
  const int ty = t >> 4, tx = t & 15;  // this thread's 4x4 outputs: rows ty*4.., columns tx*4..
  const long long tiles_m = (B + PT_BM - 1) / PT_BM;
  const int tiles_n = (N + PT_BN - 1) / PT_BN;
  for (long long tile = blockIdx.x; tile < tiles_m * tiles_n; tile += gridDim.x) {
    const long long m0 = (tile / tiles_n) * PT_BM;
    const int tn = (int)(tile % tiles_n), n0 = tn * PT_BN;
    if (t < PT_BM) rid[t] = (m0 + t < B) ? pt_row(ids, m0 + t, rows, oob, tn == 0) : -1;
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    for (int k0 = 0; k0 < Dp; k0 += PT_BK) {
      const int kk = t & 31;
#pragma unroll
      for (int i = 0; i < 8; ++i) {  // a warp reads 32 consecutive floats of one row
        const int m = (t >> 5) + 8 * i;
        const long long r = rid[m];
        As[kk][m] = (r >= 0 && k0 + kk < Dp) ? __ldg(P + r * p_stride + k0 + kk) : 0.0f;
      }
      const int n = t & 63;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int k = (t >> 6) + 4 * i;
        Ws[k][n] = (k0 + k < Dp && n0 + n < N) ? __ldg(W + (long long)(k0 + k) * N + n0 + n) : 0.0f;
      }
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < PT_BK; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        const float4 w = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long b = m0 + ty * 4 + i;
      if (b >= B) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + tx * 4 + j;
        if (n < N) out[b * out_stride + n] = acc[i][j] + (bias ? __ldg(bias + n) : 0.0f);
      }
    }
  }
}

// g[b, :] = sum_a addend_a[b, :N] (the slot's columns), then through the l2-norm backward at the pre-norm y when given
// (the same rule as mm_l2_normalize_backward).  One warp per row.
__global__ void __launch_bounds__(PT_THREADS)
pretrained_grad_prep_kernel(const __grid_constant__ PtAddends ad, long long B, int N, const float* __restrict__ ypre,
                            long long y_stride, float* __restrict__ g) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long b = warp0; b < B; b += n_warps) {
    float* gr = g + b * N;
    for (int n = lane; n < N; n += 32) {
      float s = ad.p[0][b * ad.stride[0] + n];
      for (int a = 1; a < ad.n; ++a) s += ad.p[a][b * ad.stride[a] + n];
      gr[n] = s;
    }
    if (ypre == nullptr) continue;
    float ss = 0.0f, xg = 0.0f;
    for (int n = lane; n < N; n += 32) {
      const float v = ypre[b * y_stride + n];
      ss = fmaf(v, v, ss);
      xg = fmaf(v, gr[n], xg);
    }
    ss = warp_sum(ss);
    xg = warp_sum(xg);
    const bool on = ss >= 1e-12f;
    const float nrm = on ? sqrtf(ss) : 1e-6f;
    const float yg = on ? xg / nrm : 0.0f;
    for (int n = lane; n < N; n += 32) gr[n] = (gr[n] - (ypre[b * y_stride + n] / nrm) * yg) / nrm;
  }
}

// Partial dW of row chunk s for one (64 k) x (64 n) tile: ws[s, k, n] = sum over the chunk's samples, in order, of
// P[row(b), k] g[b, n]; the CTAs of k tile 0 also write the chunk's db partial wsb[s, n].
template <typename IdxT>
__global__ void __launch_bounds__(PT_THREADS)
pretrained_dw_kernel(const float* __restrict__ P, long long rows, int Dp, long long p_stride, const IdxT* __restrict__ ids,
                     long long B, const float* __restrict__ g, int N, long long chunk, int S, float* __restrict__ ws,
                     float* __restrict__ wsb) {
  __shared__ __align__(16) float As[PT_BK][PT_BM];  // As[b][k]
  __shared__ __align__(16) float Gs[PT_BK][PT_BN];  // Gs[b][n]
  __shared__ long long rid[PT_BK];
  const int t = threadIdx.x;
  const int ty = t >> 4, tx = t & 15;
  const int tiles_k = (Dp + PT_BM - 1) / PT_BM, tiles_n = (N + PT_BN - 1) / PT_BN;
  const long long tasks = (long long)tiles_k * tiles_n * S;
  for (long long task = blockIdx.x; task < tasks; task += gridDim.x) {
    const int s = (int)(task / (tiles_k * tiles_n));
    const int rem = (int)(task % (tiles_k * tiles_n));
    const int tk = rem / tiles_n, tn = rem % tiles_n;
    const int k0 = tk * PT_BM, n0 = tn * PT_BN;
    const long long b0 = (long long)s * chunk, b1 = b0 + chunk < B ? b0 + chunk : B;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    for (long long bb = b0; bb < b1; bb += PT_BK) {
      if (t < PT_BK) rid[t] = (bb + t < b1) ? pt_row(ids, bb + t, rows, (int*)nullptr, false) : -1;
      __syncthreads();
      const int c = t & 63;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int bi = (t >> 6) + 4 * i;
        const long long r = rid[bi];
        As[bi][c] = (r >= 0 && k0 + c < Dp) ? __ldg(P + r * p_stride + k0 + c) : 0.0f;
        Gs[bi][c] = (bb + bi < b1 && n0 + c < N) ? g[(bb + bi) * N + n0 + c] : 0.0f;
      }
      __syncthreads();
#pragma unroll 8
      for (int bi = 0; bi < PT_BK; ++bi) {
        const float4 a = *reinterpret_cast<const float4*>(&As[bi][ty * 4]);
        const float4 w = *reinterpret_cast<const float4*>(&Gs[bi][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
      }
      __syncthreads();
    }
    float* wsp = ws + (long long)s * Dp * N;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + ty * 4 + i;
      if (k >= Dp) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + tx * 4 + j;
        if (n < N) wsp[(long long)k * N + n] = acc[i][j];
      }
    }
    if (tk == 0 && t < PT_BN && n0 + t < N) {
      float sb = 0.0f;
      for (long long b = b0; b < b1; ++b) sb += g[b * N + n0 + t];
      wsb[(long long)s * N + n0 + t] = sb;
    }
  }
}

// dW[k, n] = sum_s ws[s, k, n] and db[n] = sum_s wsb[s, n], in chunk order.
__global__ void __launch_bounds__(PT_THREADS)
pretrained_dw_reduce_kernel(const float* __restrict__ ws, const float* __restrict__ wsb, int S, long long KN, int N,
                            float* __restrict__ dW, float* __restrict__ db) {
  const long long total = KN + (db ? N : 0);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.0f;
    if (i < KN) {
      for (int c = 0; c < S; ++c) s += ws[(long long)c * KN + i];
      dW[i] = s;
    } else {
      for (int c = 0; c < S; ++c) s += wsb[(long long)c * N + (i - KN)];
      db[i - KN] = s;
    }
  }
}

// Most row chunks the backward's partials take at B samples: enough (k, n, chunk) tasks to fill the GPU, at most 64, at
// most one per 32 rows.  Non-decreasing in B, so a workspace sized for B serves every smaller batch.
static long long pt_max_chunks(long long B, int Dp, int N) {
  const long long tiles = (long long)((Dp + PT_BM - 1) / PT_BM) * ((N + PT_BN - 1) / PT_BN);
  long long S = (512 + tiles - 1) / tiles;
  if (S > 64) S = 64;
  const long long max_s = (B + PT_BK - 1) / PT_BK;
  if (S > max_s) S = max_s;
  return S < 1 ? 1 : S;
}

// Row chunks of the backward's partials: chunks of a multiple of 32 rows, at most pt_max_chunks of them (rounding the
// chunk up only lowers their number).  A function of (B, Dp, N) only, so the summation order does not depend on the
// device.
static void pt_split(long long B, int Dp, int N, int* S_out, long long* chunk_out) {
  const long long S = pt_max_chunks(B, Dp, N);
  long long chunk = (B + S - 1) / S;
  chunk = (chunk + PT_BK - 1) / PT_BK * PT_BK;
  if (chunk < PT_BK) chunk = PT_BK;
  *chunk_out = chunk;
  *S_out = (int)((B + chunk - 1) / chunk);
}

static long long pt_grid(long long tasks, int per_sm) {
  const long long cap = (long long)sm_count() * per_sm;
  return tasks < cap ? (tasks < 1 ? 1 : tasks) : cap;
}

static int pt_check_source(const char* who, const float* P, long long rows, int Dp, long long p_stride, const void* ids,
                           int idx_dtype, long long B) {
  MM_REQUIRE(P != nullptr && B >= 0 && p_stride >= Dp, MM_ERR_ARG, "%s: null P, B < 0 or p_stride < Dp", who);
  MM_REQUIRE(Dp >= 1 && Dp <= MM_PRETRAINED_MAX_DIM, MM_ERR_UNSUPPORTED, "%s: Dp=%d outside 1..%d", who, Dp,
             MM_PRETRAINED_MAX_DIM);
  MM_REQUIRE(ids == nullptr || idx_dtype == MM_I32 || idx_dtype == MM_I64, MM_ERR_ARG,
             "%s: idx_dtype must be MM_I32 or MM_I64", who);
  MM_REQUIRE(ids != nullptr ? rows > 0 : rows >= B, MM_ERR_ARG,
             "%s: rows must be > 0 (ids given) or >= B (a dense (B, Dp) input)", who);
  return MM_OK;
}

}  // namespace mm

extern "C" {

int mm_pretrained_gather(const float* P, int64_t rows, int Dp, int64_t p_stride, const void* ids, int idx_dtype, int64_t B,
                         float* out, int64_t out_stride, int32_t* oob_count, void* stream) {
  int rc = mm::pt_check_source("mm_pretrained_gather", P, rows, Dp, p_stride, ids, idx_dtype, B);
  if (rc) return rc;
  MM_REQUIRE(out != nullptr && out_stride >= Dp, MM_ERR_ARG, "mm_pretrained_gather: null out or out_stride < Dp");
  if (B == 0) return MM_OK;
  const bool vec = Dp % 4 == 0 && p_stride % 4 == 0 && out_stride % 4 == 0 && (uintptr_t)P % 16 == 0 &&
                   (uintptr_t)out % 16 == 0;
  const unsigned blocks = (unsigned)mm::pt_grid((B * 32 + mm::PT_THREADS - 1) / mm::PT_THREADS, 8);
  cudaStream_t st = (cudaStream_t)stream;
#define MM_PT_GATHER(IT, V)                                                                                     \
  mm::pretrained_gather_kernel<IT, V><<<blocks, mm::PT_THREADS, 0, st>>>(P, rows, Dp, p_stride, (const IT*)ids, \
                                                                         B, out, out_stride, oob_count)
  if (idx_dtype == MM_I64 && ids) {
    if (vec) MM_PT_GATHER(int64_t, true); else MM_PT_GATHER(int64_t, false);
  } else {
    if (vec) MM_PT_GATHER(int32_t, true); else MM_PT_GATHER(int32_t, false);
  }
#undef MM_PT_GATHER
  return mm::check_launch("mm_pretrained_gather");
}

int mm_pretrained_project(const float* P, int64_t rows, int Dp, int64_t p_stride, const void* ids, int idx_dtype, int64_t B,
                          const float* W, const float* bias, int N, float* out, int64_t out_stride, int32_t* oob_count,
                          void* stream) {
  int rc = mm::pt_check_source("mm_pretrained_project", P, rows, Dp, p_stride, ids, idx_dtype, B);
  if (rc) return rc;
  MM_REQUIRE(W != nullptr && out != nullptr, MM_ERR_ARG, "mm_pretrained_project: null W or out");
  MM_REQUIRE(N >= 1 && N <= MM_PRETRAINED_MAX_OUT, MM_ERR_UNSUPPORTED, "mm_pretrained_project: N=%d outside 1..%d", N,
             MM_PRETRAINED_MAX_OUT);
  MM_REQUIRE(out_stride >= N, MM_ERR_ARG, "mm_pretrained_project: out_stride < N");
  if (B == 0) return MM_OK;
  const long long tiles = ((B + mm::PT_BM - 1) / mm::PT_BM) * ((N + mm::PT_BN - 1) / mm::PT_BN);
  const unsigned blocks = (unsigned)mm::pt_grid(tiles, MM_PRETRAINED_CTAS_PER_SM);
  cudaStream_t st = (cudaStream_t)stream;
  if (idx_dtype == MM_I64 && ids)
    mm::pretrained_project_kernel<int64_t><<<blocks, mm::PT_THREADS, 0, st>>>(P, rows, Dp, p_stride, (const int64_t*)ids, B, W,
                                                                            bias, N, out, out_stride, oob_count);
  else
    mm::pretrained_project_kernel<int32_t><<<blocks, mm::PT_THREADS, 0, st>>>(P, rows, Dp, p_stride, (const int32_t*)ids, B, W,
                                                                            bias, N, out, out_stride, oob_count);
  return mm::check_launch("mm_pretrained_project");
}

int64_t mm_pretrained_backward_workspace_bytes(int64_t B, int Dp, int N) {
  if (B <= 0 || Dp <= 0 || N <= 0) return 0;
  const long long S = mm::pt_max_chunks(B, Dp, N);
  return (int64_t)(B * N + S * ((long long)Dp * N + N)) * (int64_t)sizeof(float);
}

int mm_pretrained_project_backward(const float* P, int64_t rows, int Dp, int64_t p_stride, const void* ids, int idx_dtype,
                                   int64_t B, const float* const* addends, const int64_t* addend_strides, int n_addends,
                                   const float* ypre, int64_t y_stride, int N, float* dW, float* db, void* workspace,
                                   int64_t workspace_bytes, void* stream) {
  int rc = mm::pt_check_source("mm_pretrained_project_backward", P, rows, Dp, p_stride, ids, idx_dtype, B);
  if (rc) return rc;
  MM_REQUIRE(N >= 1 && N <= MM_PRETRAINED_MAX_OUT, MM_ERR_UNSUPPORTED, "mm_pretrained_project_backward: N=%d outside 1..%d",
             N, MM_PRETRAINED_MAX_OUT);
  MM_REQUIRE(dW != nullptr && addends != nullptr && addend_strides != nullptr && n_addends >= 1 &&
                 n_addends <= mm::PT_MAX_ADDENDS,
             MM_ERR_ARG, "mm_pretrained_project_backward: null dW / addends or n_addends outside 1..%d", mm::PT_MAX_ADDENDS);
  MM_REQUIRE(ypre == nullptr || y_stride >= N, MM_ERR_ARG, "mm_pretrained_project_backward: y_stride < N");
  mm::PtAddends ad;
  ad.n = n_addends;
  for (int a = 0; a < mm::PT_MAX_ADDENDS; ++a) {
    ad.p[a] = a < n_addends ? addends[a] : nullptr;
    ad.stride[a] = a < n_addends ? addend_strides[a] : 0;
    if (a < n_addends)
      MM_REQUIRE(ad.p[a] != nullptr && ad.stride[a] >= N, MM_ERR_ARG,
                 "mm_pretrained_project_backward: addend %d is null or its stride < N", a);
  }
  if (B == 0) return MM_OK;
  MM_REQUIRE(workspace != nullptr && workspace_bytes >= mm_pretrained_backward_workspace_bytes(B, Dp, N) &&
                 (uintptr_t)workspace % 16 == 0,
             MM_ERR_ARG, "mm_pretrained_project_backward: workspace null, misaligned or smaller than "
                         "mm_pretrained_backward_workspace_bytes");
  int S;
  long long chunk;
  mm::pt_split(B, Dp, N, &S, &chunk);
  float* g = (float*)workspace;
  float* ws = g + B * N;
  float* wsb = ws + (long long)S * Dp * N;
  cudaStream_t st = (cudaStream_t)stream;
  mm::pretrained_grad_prep_kernel<<<(unsigned)mm::pt_grid((B * 32 + mm::PT_THREADS - 1) / mm::PT_THREADS, 8), mm::PT_THREADS, 0,
                                    st>>>(ad, B, N, ypre, y_stride, g);
  const long long tasks = (long long)((Dp + mm::PT_BM - 1) / mm::PT_BM) * ((N + mm::PT_BN - 1) / mm::PT_BN) * S;
  const unsigned blocks = (unsigned)mm::pt_grid(tasks, MM_PRETRAINED_CTAS_PER_SM);
  if (idx_dtype == MM_I64 && ids)
    mm::pretrained_dw_kernel<int64_t><<<blocks, mm::PT_THREADS, 0, st>>>(P, rows, Dp, p_stride, (const int64_t*)ids, B, g, N,
                                                                       chunk, S, ws, wsb);
  else
    mm::pretrained_dw_kernel<int32_t><<<blocks, mm::PT_THREADS, 0, st>>>(P, rows, Dp, p_stride, (const int32_t*)ids, B, g, N,
                                                                       chunk, S, ws, wsb);
  const long long KN = (long long)Dp * N;
  mm::pretrained_dw_reduce_kernel<<<(unsigned)mm::pt_grid((KN + N + mm::PT_THREADS - 1) / mm::PT_THREADS, 8), mm::PT_THREADS, 0,
                                    st>>>(ws, wsb, S, KN, N, dW, db);
  mm::count_launch(2);
  return mm::check_launch("mm_pretrained_project_backward");
}

}  // extern "C"
