// Evaluation metrics of the ranking outputs, accumulated on the device (mm_metrics_update, include/mm_b200.h): the
// loss, the Keras AUC histogram, confusion counts at up to 4 decision thresholds (Precision / Recall / BinaryAccuracy) and
// the squared-error sums of RootMeanSquaredError, read from the logits z (H, M) the evaluation forward wrote.
//
// One CTA walks its share of the batch head by head (grid-stride, whole warps, so __match_any_sync sees every lane):
//   * per-thread fp64 accumulators for the scalars; reduced by shuffles, then across warps in warp order, into one
//     partial per CTA in the workspace; metrics_fold_kernel adds the partials into the state in CTA order.  With null
//     metric weights every value is an integer or a fixed-order sum: two passes over the same batches are bit-identical;
//   * the histogram in shared memory: lanes of a warp that share a bucket are merged first (__match_any_sync: a trained
//     model puts most predictions in a few buckets), the leader adds the group's count / weight with one shared fp64
//     atomic, and the CTA adds its non-zero buckets into the state with global fp64 atomics.  Counts are integers, so their
//     sums do not depend on the order; weighted buckets may differ across runs in the last bits.
#include "mm_common.cuh"

namespace mm {
namespace met {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int S = MM_METRICS_SCALARS;
constexpr int SETS = 2;

struct Params {
  const float* z;
  long long M;
  int H, T, n_sets;
  mm_metrics_head head[MM_METRICS_MAX_HEADS];
  double* state;     // H x (S + 4T)
  double* partials;  // gridDim.x x H x S
};

__global__ void __launch_bounds__(THREADS) metrics_update_kernel(const Params p) {
  extern __shared__ double hist[];  // n_sets x [pos T | neg T]
  __shared__ double wbuf[WARPS][32];
  __shared__ double red[WARPS][S];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long stride = (long long)gridDim.x * THREADS;
  const int nh = p.n_sets * 2 * p.T;
  const float tm1 = (float)(p.T - 1);
  for (int h = 0; h < p.H; ++h) {
    const mm_metrics_head& hd = p.head[h];
    const bool binary = hd.loss_kind == MM_LOSS_BCE;
    double acc[S];
#pragma unroll
    for (int k = 0; k < S; ++k) acc[k] = 0.0;
    if (binary) {
      for (int i = threadIdx.x; i < nh; i += THREADS) hist[i] = 0.0;
      __syncthreads();
    }
    for (long long m0 = (long long)blockIdx.x * THREADS + (threadIdx.x & ~31); m0 < p.M; m0 += stride) {
      const long long m = m0 + lane;
      bool ok = m < p.M;
      float z = 0.0f, y = 0.0f, pr = 0.0f;
      if (ok) {
        z = p.z[(long long)h * p.M + m];
        y = load_as_f32(hd.targets, m, hd.target_dtype);
        const bool bad = z != z || y != y || (binary && y != 0.0f && y != 1.0f);
        acc[MM_METRICS_INVALID] += bad ? 1.0 : 0.0;
        ok = !bad;
      }
      int bucket = 0;
      if (ok) {
        const float sw = hd.sample_weight ? hd.sample_weight[m] : 1.0f;
        float l;
        if (binary) {
          const float e = expf(-fabsf(z));
          l = fmaxf(z, 0.0f) - z * y + log1pf(e);
          pr = hd.pred_form == MM_PRED_HEAD ? head_pred(MM_LOSS_BCE, z) : apply_act_slow(z, MM_ACT_SIGMOID);
          bucket = max((int)ceilf(__fmul_rn(pr, tm1)) - 1, 0);
        } else {
          const float d = z - y;
          l = d * d;
        }
        acc[MM_METRICS_LOSS] += (double)sw * (double)l;
        acc[MM_METRICS_COUNT] += 1.0;
      }
#pragma unroll
      for (int s = 0; s < SETS; ++s) {
        if (s >= p.n_sets) break;
        const float* mw = hd.metric_weights[s];
        const double w = ok ? (mw ? (double)mw[m] : 1.0) : 0.0;
        double* a = acc + MM_METRICS_SET0 + s * MM_METRICS_SET_STRIDE;
        if (!binary) {
          const double d = (double)z - (double)y;
          a[MM_METRICS_SQ_ERR] += w * d * d;
          a[MM_METRICS_W_SUM] += w;
          continue;
        }
        // constant indices only: acc stays in registers
        const bool pos = y == 1.0f;
        const double wp = pos ? w : 0.0, wn = pos ? 0.0 : w;
        a[MM_METRICS_POS] += wp;
        a[MM_METRICS_NEG] += wn;
#pragma unroll
        for (int i = 0; i < MM_METRICS_MAX_THRESHOLDS; ++i) {
          const bool above = i < hd.n_thresholds && pr > hd.thresholds[i];
          a[MM_METRICS_TP + i] += above ? wp : 0.0;
          a[MM_METRICS_FP + i] += above ? wn : 0.0;
        }
        // histogram: merge the lanes of one bucket, then one shared atomic per group
        const int key = ok ? (pos ? 0 : p.T) + bucket : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        const int leader = __ffs(peers) - 1;
        double v;
        if (mw) {
          wbuf[wid][lane] = w;
          __syncwarp();
          v = 0.0;
          if (lane == leader)
            for (unsigned r = peers; r; r &= r - 1) v += wbuf[wid][__ffs(r) - 1];
          __syncwarp();
        } else {
          v = (double)__popc(peers);
        }
        if (lane == leader && key >= 0) atomicAdd(&hist[s * 2 * p.T + key], v);
      }
    }
    // scalars: warp butterfly, then warps in order -> this CTA's partial
#pragma unroll
    for (int k = 0; k < S; ++k) {
      double v = acc[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[wid][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < S) {
      double v = 0.0;
      for (int w = 0; w < WARPS; ++w) v += red[w][threadIdx.x];
      p.partials[((long long)blockIdx.x * p.H + h) * S + threadIdx.x] = v;
    }
    if (binary) {
      double* st = p.state + (long long)h * (S + 4 * p.T) + S;
      for (int i = threadIdx.x; i < nh; i += THREADS)
        if (hist[i] != 0.0) atomicAdd(st + i, hist[i]);
    }
    __syncthreads();  // red / hist are reused by the next head
  }
}

// state[h][k] += sum over CTAs (in CTA order) of the partials
__global__ void metrics_fold_kernel(const double* __restrict__ partials, int G, int H, int T, double* __restrict__ state) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * S) return;
  double v = 0.0;
  for (int g = 0; g < G; ++g) v += partials[(long long)g * H * S + i];
  state[(long long)(i / S) * (S + 4 * T) + i % S] += v;
}

static int grid_for(long long M) {
  const long long g = (M + THREADS - 1) / THREADS;
  return (int)(g < sm_count() ? g : sm_count());
}

}  // namespace met
}  // namespace mm

extern "C" {

int64_t mm_metrics_workspace_bytes(int64_t M, int H) {
  if (M <= 0 || H <= 0) return 0;
  return (int64_t)mm::met::grid_for(M) * H * MM_METRICS_SCALARS * (int64_t)sizeof(double);
}

int mm_metrics_update(const float* logits, int64_t M, int H, const mm_metrics_head* heads_host, int num_buckets, int n_sets,
                      double* state, void* workspace, int64_t workspace_bytes, void* stream) {
  using namespace mm::met;
  MM_REQUIRE(logits && heads_host && state && M >= 0, MM_ERR_ARG, "mm_metrics_update: null pointer or M < 0");
  MM_REQUIRE(H >= 1 && H <= MM_METRICS_MAX_HEADS, MM_ERR_ARG, "mm_metrics_update: H = %d outside [1, %d]", H, MM_METRICS_MAX_HEADS);
  MM_REQUIRE(num_buckets >= 2 && num_buckets <= MM_METRICS_MAX_BUCKETS, MM_ERR_ARG,
             "mm_metrics_update: num_buckets = %d outside [2, %d]", num_buckets, MM_METRICS_MAX_BUCKETS);
  MM_REQUIRE(n_sets == 1 || n_sets == 2, MM_ERR_ARG, "mm_metrics_update: n_sets must be 1 or 2");
  Params p{};
  p.z = logits;
  p.M = M;
  p.H = H;
  p.T = num_buckets;
  p.n_sets = n_sets;
  p.state = state;
  for (int h = 0; h < H; ++h) {
    const mm_metrics_head& hd = heads_host[h];
    MM_REQUIRE(hd.targets, MM_ERR_ARG, "mm_metrics_update: head %d: null targets", h);
    MM_REQUIRE(hd.target_dtype >= MM_I32 && hd.target_dtype <= MM_F64, MM_ERR_ARG, "mm_metrics_update: head %d: bad target dtype", h);
    MM_REQUIRE(hd.loss_kind == MM_LOSS_BCE || hd.loss_kind == MM_LOSS_MSE, MM_ERR_ARG, "mm_metrics_update: head %d: bad loss kind", h);
    MM_REQUIRE(hd.pred_form == MM_PRED_ACT || hd.pred_form == MM_PRED_HEAD, MM_ERR_ARG, "mm_metrics_update: head %d: bad pred_form", h);
    MM_REQUIRE(hd.n_thresholds >= 0 && hd.n_thresholds <= MM_METRICS_MAX_THRESHOLDS, MM_ERR_ARG,
               "mm_metrics_update: head %d: n_thresholds outside [0, %d]", h, MM_METRICS_MAX_THRESHOLDS);
    p.head[h] = hd;
  }
  if (M == 0) return MM_OK;
  const int G = grid_for(M);
  MM_REQUIRE(workspace && workspace_bytes >= mm_metrics_workspace_bytes(M, H), MM_ERR_ARG,
             "mm_metrics_update: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
             (long long)mm_metrics_workspace_bytes(M, H));
  p.partials = static_cast<double*>(workspace);
  const size_t smem = (size_t)n_sets * 2 * num_buckets * sizeof(double);
  metrics_update_kernel<<<G, THREADS, smem, (cudaStream_t)stream>>>(p);
  if (const int rc = mm::check_launch("mm_metrics_update")) return rc;
  const int n = H * MM_METRICS_SCALARS;
  metrics_fold_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p.partials, G, H, num_buckets, state);
  return mm::check_launch("mm_metrics_update (fold)");
}

}  // extern "C"
