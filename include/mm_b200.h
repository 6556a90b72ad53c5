/*
 * mm_b200.h — C-ABI of the H100-native (sm_90a) hot path of NVIDIA-Merlin/models:
 *             embedding lookup -> MLP tower -> interaction / scoring.
 *
 * The reference (/root/reference, merlin/models/tf) has no FFI layer: every byte on this
 * path is moved by TensorFlow ops called from Python.  This header declares the entry
 * points a maintainer would bind (ctypes stub shown in INTEGRATION.md) to replace those op
 * call sites.  Each declaration cites the reference call site it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the parameter name ends in `_host`;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - nothing is allocated or freed inside the library; the caller owns every buffer;
 *   - return value: 0 = ok, <0 = argument error (MM_ERR_*), >0 = cudaError_t of the launch;
 *     `mm_last_error()` returns a thread-local human-readable message for the last failure;
 *   - all matrices are row-major fp32 unless stated; strides are in ELEMENTS.
 */
#ifndef MM_B200_H_
#define MM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MM_OK 0
#define MM_ERR_ARG (-1)        /* null pointer / negative size / bad enum */
#define MM_ERR_UNSUPPORTED (-2) /* shape outside what the kernels implement */
#define MM_ERR_ALIGN (-3)      /* pointer / stride alignment requirement violated */
#define MM_ERR_DRIVER (-4)     /* driver entry point (tensor map encode) unavailable */

#define MM_MAX_TABLES 64 /* tables per fused gather launch */

/* index dtypes */
#define MM_I32 0
#define MM_I64 1

/* activations (Keras names; merlin/models/tf/blocks/mlp.py:97-127 passes them to Dense) */
#define MM_ACT_LINEAR 0
#define MM_ACT_RELU 1
#define MM_ACT_SIGMOID 2
#define MM_ACT_TANH 3
#define MM_ACT_SELU 4
#define MM_ACT_ELU 5
#define MM_ACT_GELU 6 /* exact erf form (Keras default approximate=False) */

/* bag combiners (tf.nn.safe_embedding_lookup_sparse; inputs/embedding.py:432-441) */
#define MM_COMBINER_MEAN 0
#define MM_COMBINER_SUM 1
#define MM_COMBINER_SQRTN 2
#define MM_COMBINER_MAX 3 /* dense-sequence combiner only (inputs/embedding.py:1545-1587) */

int mm_version(void);
const char* mm_last_error(void);
/* number of kernel launches issued through this library by the calling process */
int64_t mm_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * Deterministic table initialiser: w[i] = lo + (hi-lo) * u24(hash(seed, i)) with
 * u24 in [0,1) on a 2^-24 grid; bit-reproducible on the CPU (oracle/oracle.py:hash_uniform).
 * Stands in for Keras `embeddings_initializer="uniform"` (inputs/embedding.py:205) at sizes
 * (10.9 GiB of tables) that cannot be generated on the host and shipped.
 * ------------------------------------------------------------------------------------- */
int mm_init_uniform_hash(float* w, int64_t n, uint64_t seed, float lo, float hi, void* stream);

/* ---------------------------------------------------------------------------------------
 * K1/K3/K5  Fused multi-table one-hot gather.
 * Replaces T x tf.keras.layers.Embedding / tf.gather  (inputs/embedding.py:452,460,:1142,1146)
 * + tf.stack / tf.concat of the results (core/aggregation.py:64,108).
 *   out[b * out_stride + out_col[t] + d] = weights[t][ idx[t][b] * dim[t] + d ]
 * With out_col[t] = slot(t)*D this IS StackFeatures' (B,F,D) layout; with a running sum of
 * dims it is ConcatFeatures' layout.  Rows are copied bit-exactly.
 * An index outside [0, rows) writes a zero row and increments *oob_count (if non-null) —
 * TF-GPU semantics for gather; the Python wrapper turns a non-zero count into the
 * InvalidArgumentError that TF-CPU raises.
 * ------------------------------------------------------------------------------------- */
typedef struct {
  const float* weights; /* (rows, dim) */
  const void* indices;  /* (B,) int32 or int64 */
  int64_t rows;
  int32_t dim;
  int32_t out_col; /* column offset (floats) of this feature inside an output row */
} mm_gather_table;

int mm_gather_multi(const mm_gather_table* tables_host, int n_tables, int idx_dtype, int64_t B,
                    float* out, int64_t out_stride, int32_t* oob_count, void* stream);

/* ---------------------------------------------------------------------------------------
 * K2  Multi-hot bag lookup (ragged `name__values` + `name__offsets`).
 * Replaces tf.nn.safe_embedding_lookup_sparse (inputs/embedding.py:432-441,:1139):
 * ids < 0 are dropped, an empty bag yields zeros, mean = sum/count, sqrtn = sum/sqrt(count).
 * Summation order inside a bag is left-to-right (sequential fp32 adds), as TF's
 * segment_sum on CPU does.
 * ------------------------------------------------------------------------------------- */
int mm_gather_bag(const float* weights, int64_t rows, int dim, const void* values, int idx_dtype,
                  const void* offsets, int off_dtype, int64_t B, int combiner, float* out,
                  int64_t out_stride, int out_col, int32_t* oob_count, void* stream);

/* Dense (B, L) sequence lookup + combiner over axis 1 (padding NOT masked);
 * replaces Embedding + process_sequence_combiner (inputs/embedding.py:457-461,:1556-1587). */
int mm_gather_seq(const float* weights, int64_t rows, int dim, const void* ids, int idx_dtype,
                  int64_t B, int L, int combiner, float* out, int64_t out_stride, int out_col,
                  int32_t* oob_count, void* stream);

/* ---------------------------------------------------------------------------------------
 * K3  Column concat with cast to fp32.
 * Replaces ConcatFeatures (core/aggregation.py:54-66: sorted-key tf.concat + cast to float32)
 * and ContinuousFeatures' (B,) -> (B,1) expand (inputs/continuous.py:134-138).  The caller
 * lists the pieces in the reference's sorted-name order with running out_col offsets.
 *   out[b, out_col[i] + c] = (float) src_i[b * src_stride_i + c],  c < width_i
 * ------------------------------------------------------------------------------------- */
#define MM_F32 2
#define MM_F64 3
typedef struct {
  const void* src;
  int64_t src_stride; /* elements between consecutive rows of this piece */
  int32_t width;
  int32_t dtype; /* MM_I32, MM_I64, MM_F32, MM_F64 */
  int32_t out_col;
  int32_t reserved;
} mm_concat_piece;

int mm_concat_columns(const mm_concat_piece* pieces_host, int n_pieces, int64_t B, float* out,
                      int64_t out_stride, void* stream);

/* mm_concat_columns fused with mm_split_rows: the concatenated row leaves directly as the
 * split-bf16 operand (B, 2*Kp) [hi | lo] of mm_dense_tc / mm_mlp_tc, zero padded to Kp
 * (ConcatFeatures core/aggregation.py:54-66 feeding the first Dense of an MLPBlock, blocks/mlp.py:275-277).
 * Pieces as above (out_col + width <= Kp, at most 64 pieces, Kp <= 320). */
int mm_concat_split(const mm_concat_piece* pieces_host, int n_pieces, int64_t B, void* out_split, int Kp,
                    void* stream);

/* L2Norm (transforms/regularization.py:27-82): x / sqrt(max(sum(x^2, -1), 1e-12)); in place ok */
int mm_l2_normalize(const float* x, int64_t B, int D, int64_t x_stride, float* out,
                    int64_t out_stride, void* stream);

/* BatchNormalization at inference (MLPBlock(normalization="batch_norm"), blocks/mlp.py:131-135; Keras epsilon 1e-3):
 * out = x * scale + shift per column, scale = gamma / sqrt(moving_var + eps), shift = beta - moving_mean * scale.
 * The host folds every normalization that is followed by a Dense into that Dense's kernel and bias; this entry
 * point serves the one at the end of a block.  In place ok. */
int mm_scale_shift(const float* x, int64_t B, int D, int64_t x_stride, const float* scale, const float* shift,
                   float* out, int64_t out_stride, void* stream);

/* DCN-v2 cross combine out = x0 * proj + x (blocks/cross.py:196-198) for projections that do not come out of a
 * GEMM with the fused cross epilogue (CrossBlock(low_rank_dim=...) on the exact-fp32 engine). */
int mm_cross_combine(const float* x0, const float* proj, const float* x, int64_t B, int D, int64_t x0_stride,
                     int64_t proj_stride, int64_t x_stride, float* out, int64_t out_stride, void* stream);

/* ---------------------------------------------------------------------------------------
 * K6 (+K3)  Pairwise dot-product interaction.
 * Replaces tf.matmul(x, x, transpose_b=True) + band_part + boolean_mask
 * (blocks/interaction.py:102,107-112) and the shortcut concat (blocks/dlrm.py:126-130).
 *   out[b, 0:P]      = prefix[b, 0:P]                  (P = 0 / prefix NULL: no prefix)
 *   out[b, P + p(i,j)] = sum_d x[b,i,d] * x[b,j,d]      i<j (or i<=j if self_interaction),
 * pairs enumerated row-major over the upper triangle.  Dots accumulate in fp32.
 * Output: either fp32 `out` (B, >= P+pairs) or `out_split`, the split-bf16 operand (B, 2*out_Kp)
 * = [hi | lo] of the next tensor-core dense layer (out_Kp = mm_tc_padded_k(P+pairs), padding
 * columns written as zeros) — exactly one of the two must be non-null.
 * Tensor-core path (mma.sync bf16, 3-pass split, one warp per sample, 16-byte cp.async row staging)
 * when F <= 32, D in {16, 32, 64, 128}, P in {0, D}, no self interaction; CUDA-core path otherwise.
 * ------------------------------------------------------------------------------------- */
int mm_dot_interaction(const float* x, int64_t B, int F, int D, int64_t x_stride,
                       const float* prefix, int P, int64_t prefix_stride, int self_interaction,
                       float* out, int64_t out_stride, void* out_split, int out_Kp, void* stream);

/* Fused K1+K5+K6+K3 for DLRM: look up one row per table and sample straight into shared memory,
 * place the bottom-MLP vector at slot `bottom_slot`, write [bottom | interactions] as mm_dot_interaction
 * does (fp32 `out` or split-bf16 `out_split`); the (B,F,D) stack never touches HBM.  All rows are D wide.
 * Table descriptor:
 *   - per-table id width: idx_bytes = 1, 2, 3 (unsigned little-endian — what a loader ships when the
 *     table has <= 2^8 / 2^16 / 2^24 rows), 4 (int32) or 8 (int64).  Narrow arrays need no alignment;
 *     the kernel reads the aligned 32-bit words that contain an id, so the array must be readable up
 *     to the next 4-byte boundary after its last id.  (loader hand-off: merlin/models/tf/loader.py:135-420)
 *   - placement: peer_weights_host == NULL: `weights` is the whole (rows, D) table (replicated);
 *     otherwise the table is ROW-SHARDED over `world` GPUs of one NVLink domain — global row r lives on
 *     rank r % world at local row r / world — `weights` is this rank's shard and peer_weights_host[k]
 *     the shard of rank k as mapped into this process (peer access / symmetric memory;
 *     peer_weights_host[rank] == weights).  A row owned by another rank is read over NVLink straight
 *     into the consuming SM's shared memory: the distributed lookup (SOK `lookup_sparse` on a distributed
 *     variable, merlin/models/tf/distributed/embedding.py:75-84,144-148: all-to-all of keys, local
 *     lookup, all-to-all of vectors) is part of the same kernel as the interaction.  No collective,
 *     no barrier: tables are read-only in the forward pass.
 * `rows` is always the GLOBAL row count; ids outside [0, rows) give a zero row and bump *oob_count.
 * F = n_tables + (bottom ? 1 : 0) <= 32, D in {16, 32, 64, 128}, world <= 8.
 * Id columns (indices, idx_bytes, rows) of mm_lookup_table and mm_sparse_table are checked alike by every entry point
 * that takes them (mm_dlrm_lookup_interact, mm_dlrm_interact_backward, mm_deepfm_head, mm_sparse_rows_apply), before
 * any launch: null indices, rows <= 0, idx_bytes outside {1, 2, 3, 4, 8} or a 1-, 2- or 3-byte width that cannot
 * address every row (rows > 2^(8 idx_bytes)) return MM_ERR_ARG; 4- and 8-byte id arrays not aligned to their width
 * return MM_ERR_ALIGN.  mm_dlrm_interact_backward, mm_deepfm_head and mm_sparse_rows_apply return these codes where
 * they used to launch with such a column; weights that are not 16-byte aligned now return MM_ERR_ALIGN from both
 * mm_dlrm_lookup_interact (formerly MM_ERR_ARG) and mm_dlrm_interact_backward.
 * The earlier fused entry point over mm_gather_table descriptors (int32 / int64 ids only) is removed.  Its callers pass the
 * same tables here as mm_lookup_table with idx_bytes 4 or 8; for shapes outside this kernel they gather the (B,F,D) stack
 * with mm_gather_multi and call mm_dot_interaction. */
typedef struct {
  const float* weights;
  const void* indices; /* (B,) ids of this feature, idx_bytes each */
  int64_t rows;
  int32_t slot;      /* position of this feature in the sorted (B,F,D) stack */
  int32_t idx_bytes; /* 1, 2, 3, 4, 8 */
  const float* const* peer_weights_host; /* NULL, or `world` shard pointers (host array) */
} mm_lookup_table;

/* row_format: MM_ROWS_F32 — `weights` / `bottom` are fp32 rows; MM_ROWS_OPERAND (D = 64) — they are split-bf16 rows
 * [hi(0..D) | lo(0..D)] (mm_split_rows with Kp = D: the operand format of every tensor-core layer here; same row size),
 * so the kernel loads its MMA fragments with ldmatrix and the per-sample bf16 split and operand moves (more than a
 * third of its instructions) disappear.  Needs the split-bf16 output (`out_split`); same arithmetic as MM_ROWS_F32
 * (the k order inside an MMA differs, so results agree to fp32 rounding, not bit for bit).  The price is a second
 * copy of the tables in HBM (bottom: mm_mlp_tc_operand_out writes it directly). */
#define MM_ROWS_F32 0
#define MM_ROWS_OPERAND 1
/* MM_ROWS_OPERAND_PAIRS: as MM_ROWS_OPERAND (a bottom vector is required), but the output row carries the pairs only:
 * out_split (B, 2*out_Kp) = [hi(pairs) | lo(pairs)] with out_Kp a multiple of 8 >= F(F-1)/2 (Criteo: 352, 1 408-B rows);
 * columns past the pairs are zeros.  The bottom vector is not copied out: mm_mlp_tc_pairs reads it from the bottom
 * tower's own operand rows. */
#define MM_ROWS_OPERAND_PAIRS 2
int mm_dlrm_lookup_interact(const mm_lookup_table* tables_host, int n_tables, int64_t B, int D, int rank, int world,
                            const float* bottom, int64_t bottom_stride, int bottom_slot, float* out,
                            int64_t out_stride, void* out_split, int out_Kp, int32_t* oob_count, int row_format,
                            void* stream);

/* ---------------------------------------------------------------------------------------
 * K4  Dense layer, exact fp32 on CUDA cores:  out = act(x @ W + bias).
 * Replaces tf.keras.layers.Dense (blocks/mlp.py:275-280); W is the Keras kernel (K, N).
 * If x0 is non-null the epilogue is the DCN-v2 cross:  out = x0 * (x @ W + bias) + x
 * (blocks/cross.py:196-198; requires N == K, act ignored).
 * ------------------------------------------------------------------------------------- */
int mm_dense_fp32(const float* x, int64_t B, int K, int64_t x_stride, const float* W,
                  const float* bias, int N, int act, const float* x0, int64_t x0_stride,
                  float* out, int64_t out_stride, void* stream);

/* ---------------------------------------------------------------------------------------
 * K4/K7  Tensor-core dense layer (wgmma bf16, TMA-fed, fp32 register accumulators).
 * fp32 operands are carried as split-bf16 pairs (hi, lo): x ~ hi + lo with
 * hi = bf16(x), lo = bf16(x - hi).  passes = 3 computes hi*hi + hi*lo + lo*hi in one
 * fp32 accumulator (|err| ~ 2^-16 relative: fp32-grade, holds the 1e-3 logit tolerance);
 * passes = 1 is plain bf16.
 *   a_split : (M, 2*Kp) bf16, row = [hi(0..Kp) | lo(0..Kp)], Kp = K padded to 64
 *   w_split : (Np, 2*Kp) bf16, K-major transpose of the Keras kernel, same split, Np = N
 *             padded to 16 — produced once by mm_split_weights
 *   out_f32 : (M, N) fp32 (nullable);  out_split : (M, 2*Kp(N)) bf16 for the next layer
 *             (nullable; its padding columns N..Kp(N) of hi and lo are written as zeros)
 *   x0/xres : fp32 (M, N) operands of the cross epilogue (nullable, both or none)
 * ------------------------------------------------------------------------------------- */
/* padded operand sizes used by the tensor-core path: Kp = ceil64(K); Np = ceil16(N) (N<=128) or ceil128(N) */
int mm_tc_padded_k(int K);
int mm_tc_padded_n(int N);
int mm_split_rows(const float* x, int64_t M, int K, int64_t x_stride, void* out_split, int Kp,
                  void* stream);
int mm_split_weights(const float* W, int K, int N, void* w_split, int Kp, int Np, void* stream);
int mm_dense_tc(const void* a_split, int64_t M, int K, int Kp, const void* w_split, int N, int Np,
                const float* bias, int act, int passes, const float* x0, const float* xres,
                int64_t x_stride, float* out_f32, int64_t out_stride, void* out_split,
                int out_Kp, void* stream);

/* mm_dense_tc followed by Keras Dropout(rate) in training (the weight-tied next-item step's MLP): after the activation,
 * v = keep(row, col) ? v / (1 - rate) : 0 into out_f32 and out_split alike, keep = Philox4x32-10 of (col, row, layer,
 * step) under key `seed`, word 0 >= round(rate 2^32) (csrc/dropout.cuh).  step: ONE device float, the optimizer's
 * MM_HYPER_STEP counter (mm_opt_tick advances it every step), read by the kernel so graph replays draw fresh masks.
 * A compile-time epilogue variant (dense_tc_kernel<true>): mm_dense_tc's kernel is unchanged.  No cross / scorer / head
 * epilogue.  Errors: mm_dense_tc's, and MM_ERR_ARG for rate outside [0, 1), a null or unaligned step, layer < 0. */
int mm_dense_tc_dropout(const void* a_split, int64_t M, int K, int Kp, const void* w_split, int N, int Np, const float* bias,
                        int act, int passes, float* out_f32, int64_t out_stride, void* out_split, int out_Kp, float rate,
                        uint64_t seed, const float* step, int layer, void* stream);
/* mm_dense_tc with a fused output head: out_head[m] = head_act( act(x W + b)[m,:] . head_w + head_b ),
 * i.e. the layer followed by Dense(N -> 1) (BinaryOutput's Dense(1, sigmoid),
 * outputs/classification.py:114) evaluated in the GEMM epilogue; N <= 32.  head_w: (N,) device. */
int mm_dense_tc_head(const void* a_split, int64_t M, int K, int Kp, const void* w_split, int N, int Np,
                     const float* bias, int act, int passes, const float* head_w, float head_b,
                     int head_act, float* head_out, void* stream);

/* Whole MLP tower in ONE launch (MLPBlock = SequentialBlock of Dense layers, blocks/mlp.py:97-139,
 * `_Dense.call` :275-280; optionally followed by BinaryOutput's Dense(1), outputs/classification.py:114):
 *   h_1 = act_1(x W_1 + b_1); h_l = act_l(h_{l-1} W_l + b_l), l = 2..n_layers (n_layers <= 4);
 *   out (M, widths[n-1]) fp32 rows (or null) and/or head_out[m] = head_act(h_n[m,:] . head_w + head_b).
 * Layer 1 is the TMA-fed wgmma GEMM of mm_dense_tc (any K); layers 2..n run on chip: the
 * activations stay in registers (bias, activation, bf16 split) and are the register A operand of the
 * next wgmma, the weights of layers 2..n stay resident in shared memory.  Every width must be
 * <= 128 (README towers: 13->128->64 and 415->128->64->32->1); fp32 parity by 3-pass split-bf16.
 * a_split: mm_split_rows layout (M, 2*Kp(K)); w_split[l]: mm_split_weights layout of layer l;
 * bias[l]: (widths[l],) device or null; acts[l]: MM_ACT_*; the head needs widths[n-1] <= 32.
 * Returns MM_ERR_UNSUPPORTED when the tower does not fit (caller then chains mm_dense_tc);
 * mm_mlp_tc_supported(K, n_layers, widths, with_head) answers that question (1 / 0) without launching:
 * 2..4 layers, widths <= 128, head only after <= 32 units, resident weights + two pipeline stages
 * within 227 KB of shared memory (with_head = 2: the multi-head epilogue of mm_mlp_tc_heads). */
int mm_mlp_tc_supported(int K, int n_layers, const int* widths, int with_head);
int mm_mlp_tc(const void* a_split, int64_t M, int K, int n_layers, const void* const* w_split,
              const int* widths, const float* const* bias, const int* acts, float* out,
              int64_t out_stride, const float* head_w, float head_b, int head_act, float* head_out,
              void* stream);

/* mm_mlp_tc with n_heads <= 8 fused output heads instead of one (OutputBlock's BinaryOutput / RegressionOutput heads,
 * outputs/block.py:32-131, outputs/regression.py:35-58, on the same tower output):
 *   heads_out[h * M + m] = heads_act[h](h_n[m,:] . heads_w[:, h] + heads_b[h])
 * heads_w (widths[n-1], n_heads) Keras layout, heads_b (n_heads,) device or null (read on the device, so a captured graph
 * follows training), heads_act: host array of MM_ACT_*; heads_out (n_heads, M): each head's (M, 1) is a contiguous slice.
 * widths[n-1] <= 32; mm_mlp_tc_supported(K, n_layers, widths, 2) says whether the tower fits with this epilogue.  Only the
 * heads are written (no fp32 rows). */
int mm_mlp_tc_heads(const void* a_split, int64_t M, int K, int n_layers, const void* const* w_split, const int* widths,
                    const float* const* bias, const int* acts, int n_heads, const float* heads_w, const float* heads_b,
                    const int* heads_act, float* heads_out, void* stream);

/* mm_mlp_tc (n_heads = 0) or mm_mlp_tc_heads (n_heads >= 1: head_w / head_out are heads_w / heads_out, out must be NULL)
 * over a layer-1 input held in two buffers, the hand-off of mm_dlrm_lookup_interact(row_format = MM_ROWS_OPERAND_PAIRS):
 *   bottom_split (M, 2*64) bf16 [hi | lo] = input columns 0..63 (the bottom tower's operand rows);
 *   pairs_split  (M, 2*Kq) bf16 [hi(Kq) | lo(Kq)] = input columns 64..K-1, Kq = K - 64 rounded up to 8.
 * Same k-blocks, MMAs and order as mm_mlp_tc over the concatenated row: results are bit-identical.  Columns of pairs_split
 * past K - 64 are never read.  K > 64. */
int mm_mlp_tc_pairs(const void* bottom_split, const void* pairs_split, int64_t M, int K, int n_layers, const void* const* w_split,
                    const int* widths, const float* const* bias, const int* acts, float* out, int64_t out_stride,
                    const float* head_w, float head_b, int head_act, float* head_out, int n_heads, const float* heads_b,
                    const int* heads_act, void* stream);

/* mm_mlp_tc whose last layer also (or only: out may be NULL) leaves its rows as split-bf16 rows
 * out_operand (M, 2 * widths[n-1]) bf16 = [hi | lo] per row (widths[n-1] % 4 == 0; the mm_split_rows layout when the
 * width is a multiple of 64) — the bottom tower of a DLRM hands its vector to
 * mm_dlrm_lookup_interact(row_format = MM_ROWS_OPERAND) this way, without a fp32 round trip. */
int mm_mlp_tc_operand_out(const void* a_split, int64_t M, int K, int n_layers, const void* const* w_split,
                          const int* widths, const float* const* bias, const int* acts, float* out,
                          int64_t out_stride, void* out_operand, void* stream);

/* Narrow-input two-layer tower in ONE launch: out = act2(act1(concat(pieces) W1 + b1) W2 + b2), K = total piece width
 * <= 16, N1 in {32, 64, 128}, N2 in {16, 32, 64} (mm_tower2_small_supported) — the DLRM bottom tower over the continuous
 * columns: ContinuousFeatures + ConcatFeatures (inputs/continuous.py:117-138, core/aggregation.py:54-66: pieces in
 * sorted-name order, cast to fp32) feeding MLPBlock([N1, N2]) (blocks/mlp.py:97-139).  One warp per 16 samples on
 * mma.sync (3-pass split-bf16, fp32 accumulate), hidden activations stay in registers, both weight matrices
 * (mm_split_weights layouts) in shared memory.  out: (B, N2) fp32 (nullable); out_split: (B, 2*N2) bf16 [hi | lo]
 * (nullable) — the operand format of mm_dlrm_lookup_interact(row_format = MM_ROWS_OPERAND).  pieces: as
 * mm_concat_columns, listed in column order (out_col = running sum of widths). */
int mm_tower2_small_supported(int K, int N1, int N2);
int mm_tower2_small(const mm_concat_piece* pieces_host, int n_pieces, int64_t B, const void* w1_split, int N1,
                    const float* bias1, int act1, const void* w2_split, int N2, const float* bias2, int act2, float* out,
                    int64_t out_stride, void* out_split, void* stream);

/* ---------------------------------------------------------------------------------------
 * K8/K9  Two-tower scoring.
 * mm_rowwise_dot: inference scorer  s[b] = sum_d q[b,d]*i[b,d]
 *   (blocks/retrieval/base.py:278-281; outputs/contrastive.py:305-307).
 * mm_inbatch_scores: training/testing logits
 *   out[b,0]   = q[b].pos[b]  (- log(pos_prob[b]+1e-16))
 *   out[b,1+n] = (pos_id[b]==neg_id[n] && downscore) ? false_neg_score
 *                                                    : q[b].neg[n] (- log(neg_prob[n]+1e-16))
 *   then every element is divided by `temperature`
 *   (blocks/retrieval/base.py:339-343,373-396; utils/tf_utils.py:126-154;
 *    outputs/contrastive.py:303-326; prediction_tasks/retrieval.py:135-136).
 * ------------------------------------------------------------------------------------- */
int mm_rowwise_dot(const float* q, const float* items, int64_t B, int D, int64_t q_stride,
                   int64_t i_stride, float* out, void* stream);
int mm_inbatch_scores(const float* q, const float* pos, const float* neg, int64_t B, int64_t N,
                      int D, const void* pos_ids, const void* neg_ids, int id_dtype, int downscore,
                      float false_neg_score, const float* pos_prob, const float* neg_prob,
                      float temperature, float* out, int64_t out_stride, void* stream);
/* Tensor-core version of the same logits, in two calls:
 *   mm_positive_scores   : column 0   (row-wise dot, logQ, temperature)
 *   mm_inbatch_scores_tc : columns 1..N — wgmma GEMM Q.N^T on split-bf16 operands
 *                          (q_split (B, 2*Kp) and neg_split (N, 2*Kp), both from mm_split_rows,
 *                          Kp = mm_tc_padded_k(D)) with mask / logQ / temperature in the epilogue. */
int mm_positive_scores(const float* q, const float* pos, int64_t B, int D, const float* pos_prob,
                       float temperature, float* out, int64_t out_stride, void* stream);
int mm_inbatch_scores_tc(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D,
                         const void* pos_ids, const void* neg_ids, int id_dtype, int downscore,
                         float false_neg_score, const float* neg_prob, float temperature, float* out,
                         int64_t out_stride, void* stream);

/* ---------------------------------------------------------------------------------------
 * K10  Query x catalog scoring without materialising (B, N_I):
 *   logits[b,i] = q[b].E[i] (+ bias[i])   (outputs/classification.py:347-357 EmbeddingTablePrediction;
 *   blocks/retrieval/base.py:431-438; outputs/topk.py:221-223 BruteForce; core/index.py:236-237)
 * One wgmma GEMM pass over the catalog whose epilogue folds every logits tile into per-row
 *   out_stats (B,3) = [max, log-sum-exp, logit[target]]   — the inputs of
 *                     CategoricalCrossEntropy(from_logits=True) (losses/listwise.py:38-50); nullable
 *   topk_scores/topk_ids (B,k): tf.math.top_k order (descending, ties -> lower id), k <= 32; k = 0: off
 * q_split (B, 2*Kp) and e_split (I, 2*Kp) are split-bf16 operands from mm_split_rows
 * (Kp = mm_tc_padded_k(D), D <= 128; the catalog is split once and reused).  `workspace` must hold
 * mm_catalog_workspace_bytes(B, I, k) bytes (per-row partials of the item-range splits).
 * ------------------------------------------------------------------------------------- */
int64_t mm_catalog_workspace_bytes(int64_t B, int64_t I, int k);
int mm_catalog_score(const void* q_split, int64_t B, int D, const void* e_split, int64_t I,
                     const float* bias, const void* targets, int id_dtype, float* out_stats, int k,
                     float* topk_scores, int64_t* topk_ids, void* workspace, int64_t workspace_bytes,
                     void* stream);

/* In-batch contrastive soft-max cross-entropy WITHOUT the (B, 1+N) logits: the same logits as
 * mm_positive_scores + mm_inbatch_scores_tc (blocks/retrieval/base.py:339-396, outputs/contrastive.py:303-326,
 * utils/tf_utils.py:126-154) folded straight into the inputs of CategoricalCrossEntropy(from_logits=True) against the
 * one-hot target on column 0 (losses/listwise.py:38-50):
 *   out_stats (B,3) = [row max, log-sum-exp over {pos} U {negatives}, pos]   ->  loss[b] = out_stats[b,1] - out_stats[b,2]
 * pos_logit (B,): column 0 as mm_positive_scores writes it (logQ and temperature already applied);
 * negatives: (pos_ids[b] == neg_ids[n] && downscore ? false_neg_score : q[b].neg[n] - log(neg_prob[n] + 1e-16)) / temperature.
 * One wgmma pass of the catalog-scoring kernel (its epilogue with the id mask) + the merge kernel; 1.07 GB of
 * logits at B = N = 16 384 never exist.  workspace: mm_catalog_workspace_bytes(B, N, 0). */
int mm_inbatch_softmax_ce(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                          const void* neg_ids, int id_dtype, int downscore, float false_neg_score, const float* pos_logit,
                          const float* neg_prob, float temperature, float* out_stats, void* workspace,
                          int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * K13  Row-sharded tables over the GPUs of one NVLink domain: row r of every table lives on
 * rank r % world at local row r / world (the reference's counterpart is SOK's distributed
 * variable, distributed/embedding.py:75-84,144-148).  Owner-computes push = gather + all-to-all
 * in ONE kernel: each rank scans the GLOBAL index list (B_global = world * B_local samples,
 * replicated by an all-gather of 4 B/feature/sample) and, for the rows it owns, copies the row
 * from its local shard straight into the destination rank's (B_local, out_stride) stack through
 * peer-mapped memory (dst_ptrs_host[r] = that buffer as mapped in this process; NVLink stores).
 *   tables_host[t].weights = local shard (local_rows, D);  .rows = GLOBAL row count;
 *   .indices = global (B_global,) index array of feature t;  .out_col = slot*D.
 * Out-of-range ids write a zero row (by the rank idx mod world) and bump *oob_count.
 * A cross-rank barrier must follow before the stacks are read (torch.distributed / symmetric
 * memory barrier on the same stream).
 * mm_init_uniform_hash_rows initialises a shard so that local row l equals global row
 * row0 + l*row_step of the table mm_init_uniform_hash would produce.
 * ------------------------------------------------------------------------------------- */
int mm_shard_gather_push(const mm_gather_table* tables_host, int n_tables, int idx_dtype,
                         int64_t B_global, int64_t B_local, int D, int rank, int world,
                         void* const* dst_ptrs_host, int64_t out_stride, int32_t* oob_count,
                         void* stream);
int mm_init_uniform_hash_rows(float* w, int64_t local_rows, int D, uint64_t seed, float lo, float hi,
                              int64_t row0, int64_t row_step, void* stream);

/* ---------------------------------------------------------------------------------------
 * K14  Training step of the DLRM path (SURVEY §8(f)-4): the backward of the same kernels and the optimizer,
 * i.e. what `Model.train_step` (merlin/models/tf/models/base.py:1121-1231) obtains from tf.GradientTape +
 * `optimizer.apply_gradients` for DLRMBlock (blocks/dlrm.py:32-133) + BinaryOutput (outputs/classification.py:114):
 *
 *   mm_heads_fwd_bwd          H <= 8 BinaryOutput / RegressionOutput heads Dense(K -> 1) with loss weights, forward AND
 *                             backward in one pass over x (M, K), K <= 256 (see below).
 *   mm_dense_wgrad            dW (K, N) += X^T dZ,  db (N) += column sums of dZ   (db nullable; accumulated)
 *   mm_dense_dgrad            dX (M, K) = dZ (M, N) W^T, W the Keras kernel (K, N), N <= 128; `mask` (M, K) nullable:
 *                             dX is zeroed where mask <= 0 (mask = the layer's input = the previous layer's relu
 *                             output, so dX is that layer's pre-activation gradient)
 *   mm_dlrm_interact_backward backward of mm_dlrm_lookup_interact (fp32 rows, replicated tables): dA (B, P + F(F-1)/2)
 *                             -> grad_rows_host[t] (B, D): the IndexedSlices values of table t (indices = the
 *                             batch's ids; duplicates NOT yet summed), and d_bottom (B, D) = gradient of the bottom
 *                             vector (interaction rows + the shortcut dA[:, :P]; zeroed where bottom <= 0 when
 *                             mask_bottom).  The table rows are looked up again (tables_host as in the forward call).
 *                             row_format MM_ROWS_OPERAND (D = 64): `weights` and `bottom` are the split-bf16 rows of
 *                             mm_dlrm_lookup_interact's operand format (mirrors kept in step by mm_sparse_rows_apply).
 *   mm_sparse_rows_apply      optimizer step on IndexedSlices with duplicate ids as Keras applies it: duplicates are
 *                             summed, then ONE update per unique row (OptimizerV2._resource_apply_sparse_duplicate_
 *                             indices; Adam on touched rows only = LazyAdam, blocks/optimizer.py:342).  rep_map:
 *                             (rows,) int32 scratch per table, all INT32_MAX between calls (mm_fill_i32 once);
 *                             grad_rows is clobbered (duplicates are folded into the first occurrence's slice);
 *                             `mirror`: operand-format copy of the table (mm_dlrm_lookup_interact MM_ROWS_OPERAND)
 *                             kept in step with the weights, nullable.
 *   mm_bag_grad_rows          backward of one pooled multi-hot feature (mm_gather_bag / mm_gather_seq): the pooled-row
 *                             gradient g (B, D) -> out (nnz, D), row i = scale(i) * g[bag(i)] — the IndexedSlices values
 *                             TF's gradient of safe_embedding_lookup_sparse / the (B, L) lookup + reduce produces; they go
 *                             to mm_sparse_rows_apply with the bag's ids as indices and B = nnz.
 *                               ragged (offsets non-null, (B+1,) int32 / int64; ids (nnz,)): mean 1/cnt, sum 1,
 *                               sqrtn 1/sqrt(cnt), cnt = ids of the bag in [0, rows) (what mm_gather_bag divides by);
 *                               fixed length (offsets null, ids (B, L), nnz = B*L): mean 1/L (padding not masked), sum 1.
 *                             Ids outside [0, rows) get a zero row.  All nnz rows are written on every call: each bag's
 *                             range is clamped to [0, nnz] and positions no bag covers get zeros, so malformed offsets
 *                             never read or write outside ids / out.  D in {16, 32, 64, 128}; g (stride a multiple of 4)
 *                             and out 16-byte aligned.  out_ids (nullable, nnz ids of the ids' dtype) receives the id of
 *                             every row that carries a gradient and -1 for the others (positions no bag covers, ids
 *                             outside [0, rows)): passed as the indices of mm_sparse_rows_apply, only rows some bag
 *                             really holds are updated (with Adam, a zero-gradient row would still move).  The max
 *                             combiner (and sqrtn on fixed-length bags) returns MM_ERR_UNSUPPORTED.
 *   mm_dense_apply            the same update rules over a flat fp32 arena; g is scaled by grad_scale and CLEARED.
 *   mm_opt_tick               step counter += 1 and the Adam bias-corrected rate (once per step, before the applies);
 *                             the counter is fp32, exact up to 2^24 steps (K25's mm_opt_tick_schedule also sets lr)
 * Update rules (hyper: device float[MM_HYPER_COUNT], so a captured CUDA graph follows a learning-rate schedule):
 *   MM_OPT_SGD      w -= lr g
 *   MM_OPT_ADAGRAD  a += g^2;  w -= lr g / (sqrt(a) + eps)                       (a starts at 0.1 in Keras)
 *   MM_OPT_ADAM     m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  w -= lr_t m / (sqrt(v) + eps),
 *                   lr_t = lr sqrt(1 - b2^t) / (1 - b1^t)
 * ------------------------------------------------------------------------------------- */
#define MM_OPT_SGD 0
#define MM_OPT_ADAGRAD 1
#define MM_OPT_ADAM 2
#define MM_HYPER_LR 0
#define MM_HYPER_BETA1 1
#define MM_HYPER_BETA2 2
#define MM_HYPER_EPS 3
#define MM_HYPER_STEP 4
#define MM_HYPER_LR_T 5
#define MM_HYPER_COUNT 8
typedef struct {
  float* weights; /* (rows, D) */
  int64_t rows;
  const void* indices; /* (B,) ids, idx_bytes each (1, 2, 3, 4, 8) */
  int32_t idx_bytes;
  int32_t reserved;
  float* grad_rows; /* (B, D) */
  int32_t* rep_map; /* (rows,) */
  float* state1;    /* Adagrad accumulator / Adam m, (rows, D); null for SGD */
  float* state2;    /* Adam v; null otherwise */
  void* mirror;     /* (rows, 2*D) bf16 [hi | lo] or null */
  float* dense_grad; /* (rows, D) fp32, all zero between calls, or null.  Non-null selects the dense path for tables with
                      * few rows (every id repeated many times per batch): slices are summed into this accumulator (rows
                      * <= 1024: each CTA first sorts its samples by row and sums the runs in registers), rep_map only
                      * flags the touched rows, and the update walks the rows.  Null: the election path (rows >> batch: duplicates are rare). */
} mm_sparse_table;

/* Loss kinds of mm_heads_fwd_bwd: BinaryOutput (sigmoid + binary cross-entropy on the logits) and RegressionOutput
 * (linear + squared error). */
#define MM_LOSS_BCE 0
#define MM_LOSS_MSE 1
/* H <= 8 output heads Dense(K -> 1) on the same x (M, K), K <= 256 (OutputBlock, outputs/block.py:32-131; BinaryOutput
 * outputs/classification.py:114, RegressionOutput outputs/regression.py:35-58; Keras compile(loss_weights) sums the
 * weighted per-output losses), forward AND backward in one pass over x:
 *   z_h = x . W[:, h] + b_h                 W (K, H) Keras layout, b (H,) device or null
 *   l_h,i = BCE: max(z,0) - z y + log(1 + e^-|z|)  |  MSE: (z - y)^2          (loss_kind[h] = MM_LOSS_BCE / MM_LOSS_MSE)
 *   loss_h = sum_i sw_i l_h,i / M;  loss (1 + H) += [sum_h lambda_h loss_h, loss_0 .. loss_{H-1}]   (lambda = loss_weight)
 *   dz_h = lambda_h sw_i (sigmoid(z_h) - y) / M  |  lambda_h sw_i 2 (z_h - y) / M
 *   dx = sum_h dz_h W[:, h]^T (written once; zeroed where x <= 0 when mask_relu);  dW[:, h] += x^T dz_h;  db_h += sum dz_h
 *   logits (H, M) nullable: z_h.  loss / dW / db are ACCUMULATED (zero them first).
 * loss_kind, loss_weight, targets, target_dtypes, sample_weights are HOST arrays of H entries; targets[h] is (M,) of
 * target_dtypes[h] (MM_I32 .. MM_F64); sample_weights (nullable array, entries nullable) holds (M,) fp32 per head — the
 * same pointer for every head when the weights are shared.  targets == NULL: forward only — logits (H, M) receives the
 * activated predictions (sigmoid(z) / z) and nothing else is read or written. */
int mm_heads_fwd_bwd(const float* x, int64_t M, int K, int64_t x_stride, int H, const float* w, const float* bias,
                     const int* loss_kind, const float* loss_weight, const void* const* targets, const int* target_dtypes,
                     const float* const* sample_weights, float* logits, float* loss, float* dx, int64_t dx_stride,
                     int mask_relu, float* dw, float* db, void* stream);
int mm_dense_wgrad(const float* x, int64_t M, int K, int64_t x_stride, const float* dz, int N, int64_t dz_stride,
                   float* dw, float* db, void* stream);
/* mm_dense_wgrad with X given as split-bf16 rows (M, 2*Kp) = [hi | lo] (mm_split_rows layout, Kp = mm_tc_padded_k(K)): the
 * operand the forward layer consumed — e.g. the interaction kernel's split output — so no fp32 copy of X has to exist. */
int mm_dense_wgrad_split(const void* x_split, int64_t M, int K, int Kp, const float* dz, int N, int64_t dz_stride,
                         float* dw, float* db, void* stream);
int mm_dense_dgrad(const float* dz, int64_t M, int N, int64_t dz_stride, const float* w, int K, const float* mask,
                   int64_t mask_stride, float* dx, int64_t dx_stride, void* stream);
/* x (B, D) = mask > 0 ? x : 0, in place: the relu derivative on a gradient that did not come out of mm_dense_dgrad (layers
 * wider than 128 units take dX = dZ W^T through mm_dense_tc on the transposed kernel). */
int mm_relu_mask(float* x, int64_t B, int D, int64_t x_stride, const float* mask, int64_t mask_stride, void* stream);
int mm_dlrm_interact_backward(const mm_lookup_table* tables_host, int n_tables, int64_t B, int D, const float* bottom,
                              int64_t bottom_stride, int bottom_slot, int P, const float* dA, int64_t dA_stride,
                              float* const* grad_rows_host, int64_t grad_stride, float* d_bottom,
                              int64_t d_bottom_stride, int mask_bottom, int row_format, void* stream);
int mm_sparse_rows_apply(const mm_sparse_table* tables_host, int n_tables, int64_t B, int D, int opt,
                         const float* hyper, void* stream);
/* Added with multi-hot training (DLRM features given as ragged bags or (B, L) id matrices); no existing entry point changed. */
int mm_bag_grad_rows(const float* g, int64_t B, int D, int64_t g_stride, const void* ids, int idx_dtype, const void* offsets,
                     int off_dtype, int L, int64_t nnz, int64_t rows, int combiner, float* out, void* out_ids, void* stream);
int mm_dense_apply(int opt, float* w, float* grad, float* state1, float* state2, int64_t n, const float* hyper,
                   float grad_scale, void* stream);
int mm_opt_tick(float* hyper, void* stream);
int mm_fill_i32(int32_t* p, int64_t n, int32_t value, void* stream);

/* Added with DCN-v2 training; no existing entry point changed, except that mm_sparse_rows_apply now also takes every
 * D with D % 4 == 0 and 4 <= D <= 128 (formerly D/4 had to divide 32; those widths run exactly as before) and returns
 * MM_ERR_ARG for a non-null mirror when D != 64.
 *   mm_cross_backward   one cross layer l of the backward of x_{l+1} = x0 * z_l + x_l, z_l = x_l W_l + b_l, in one pass:
 *                       g += p (in place; p = dz_{l+1} W_{l+1}^T, null for the top layer), dz = g * x0 written as fp32 (the
 *                       dz of mm_dense_wgrad[_split]) and as split-bf16 rows dz_split (B, 2*Kp) (mm_split_rows layout,
 *                       Kp = mm_tc_padded_k(d), padding written as zeros: the operand of the transposed-kernel
 *                       mm_dense_tc), and acc = g * z (acc_init) or acc += g * z.  Any d >= 1; fp32 row strides multiples
 *                       of 4, every buffer 16-byte aligned.
 *   mm_concat_backward  backward of a concatenated input block: for each slice t, dst_t[b, 0:width_t] = sum over the
 *                       n_addends <= 4 (B, d) addends of addend[b, col_t : col_t + width_t].  Columns of no slice are not
 *                       read.  col arbitrary, width a positive multiple of 4, dst 16-byte aligned with a row stride that is a
 *                       multiple of 4; n_slices <= 64.  addends_host / addend_strides_host / slices_host are HOST arrays. */
typedef struct {
  float* dst;         /* (B, width) rows, dst_stride floats apart */
  int64_t dst_stride;
  int32_t col;        /* first column of the slice in the addends */
  int32_t width;
} mm_column_slice;
int mm_cross_backward(const float* x0, int64_t x0_stride, const float* z, int64_t z_stride, float* g, int64_t g_stride,
                      const float* p, int64_t p_stride, float* acc, int64_t acc_stride, int acc_init, int64_t B, int d, float* dz,
                      int64_t dz_stride, void* dz_split, int Kp, void* stream);
int mm_concat_backward(const float* const* addends_host, const int64_t* addend_strides_host, int n_addends, int64_t B, int d,
                       const mm_column_slice* slices_host, int n_slices, void* stream);

/* Added with matrix factorization training; no existing entry point changed.
 *   mm_concat_backward_l2  mm_concat_backward plus the gradient of the embeddings' L2 penalty
 *                          reg = sum_t l2_t sum_b ||x0[b, col_t : col_t + width_t]||^2 (the reference's embeddings_l2_reg on
 *                          the batch's looked-up, pooled rows): dst_t[b, :] = sum_a addend_a[b, col_t : +width_t]
 *                          + 2 l2_t x0[b, col_t : +width_t], and loss[0] += reg, loss[1] += reg (loss: 2 device floats,
 *                          [total, regularization]).  The arguments and rules of mm_concat_backward, plus x0 (B, d) fp32
 *                          rows x0_stride >= d apart (no alignment beyond fp32), l2_host: n_slices HOST floats, each finite
 *                          and >= 0, and a device workspace `partials` of n_partials >= n_slices * MM_CONCAT_L2_CTAS floats.
 *                          reg is reduced in a fixed order (per-CTA partials, then one fold): equal inputs give equal bits. */
#define MM_CONCAT_L2_CTAS 512
int mm_concat_backward_l2(const float* const* addends_host, const int64_t* addend_strides_host, int n_addends, int64_t B, int d,
                          const mm_column_slice* slices_host, int n_slices, const float* x0, int64_t x0_stride,
                          const float* l2_host, float* partials, int64_t n_partials, float* loss, void* stream);

/* ---------------------------------------------------------------------------------------
 * K15  Factorization-machine heads (blocks/interaction.py:205-332; DeepFMModel models/ranking.py:171-279).
 *   mm_fm_pairwise   FMPairwiseInteraction.call: x (B, A, K) -> out (B, K) = 0.5 ((sum_a x)^2 - sum_a x^2)
 *   mm_deepfm_head   everything DeepFMModel does after its deep tower, one pass over the batch:
 *       pairwise = sum_f 0.5 ((sum_d e_f[d])^2 - sum_d e_f[d]^2)   — FMBlock stacks the embeddings on the LAST axis, so
 *                  FMPairwiseInteraction reduces over the D components of each feature (interaction.py:323-328);
 *       wide     = sum_f wide_kernel[wide_offsets[f] + id_f] + sum_c wide_kernel[cont_offsets[c]] x_c + *wide_bias
 *                  (Dense(1) over concat(one-hot categorical, continuous), :307-316: a row lookup in the Keras kernel);
 *       z = pairwise + wide + addend[b]  (addend: the deep tower's logit, nullable);
 *       out[b] = out_w ? act(z * *out_w + *out_b) : z       (BinaryOutput's Dense(1) on the 1-wide sum).
 *   tables_host[f]: weights (rows, D) fp32, ids (B,) of idx_bytes each (slot / peers unused; one-hot features only);
 *   cont_host[c]: one (B,) column (width 1, any mm_concat_piece dtype).  Ids outside [0, rows) contribute nothing and
 *   bump *oob_count.  wide_bias / out_w / out_b are DEVICE scalars (a captured graph follows weight updates).
 * ------------------------------------------------------------------------------------- */
int mm_fm_pairwise(const float* x, int64_t B, int A, int K, float* out, void* stream);
int mm_deepfm_head(const mm_lookup_table* tables_host, const int64_t* wide_offsets_host, int n_tables, int64_t B, int D,
                   const mm_concat_piece* cont_host, const int64_t* cont_offsets_host, int n_cont,
                   const float* wide_kernel, const float* wide_bias, const float* addend, int64_t addend_stride,
                   const float* out_w, const float* out_b, int out_act, float* out, int32_t* oob_count, void* stream);

/* Added with DeepFM training; no existing entry point changed.  With the forward's notation, u = h.w_dl + b_dl the deep
 * logit's pre-activation, s = pairwise + wide + act_dl(u), z = s * out_w + out_b and delta = dloss/dz (as
 * mm_heads_fwd_bwd: BCE sw (sigmoid(z) - y) / B, MSE sw 2 (z - y) / B):
 *   mm_deepfm_head_fwd_bwd  forward, loss and backward of the head in one pass over the batch.  The embedding rows are read
 *       from the gathered x0 (B, x0_stride) at emb_cols_host[f] (no second lookup); tables_host[f] gives feature f's ids
 *       (idx_bytes 1, 2, 3, 4, 8), its rows and its block's first row in the wide kernel.  Writes logits (B,) = z,
 *       ds (B,) = delta out_w, dh (B, units) = du w_dl (zeroed where h <= 0 when mask_h), du = ds act_dl'(u);
 *       ACCUMULATES loss (2,) += [loss, loss] (total and the one output's), *dw_out += sum delta s, *db_out += sum delta,
 *       dw_dl (units,) += sum du h, *db_dl += sum du, *d_wide_bias += sum ds, d_cont (n_cont,) += sum ds x_c (each of
 *       these nullable).  An id outside [0, rows) adds no wide term and bumps *oob_count (its x0 row is the gather's zero
 *       row).  out_w / out_b / wide_bias / b_dl: DEVICE scalars.  units <= 512; act_dl linear or relu.
 *   mm_fm_concat_backward   the FM term's gradient into the embedding rows, added to mm_concat_backward's sum:
 *       dst_t[b, :] = sum_a addend_a[b, col_t : col_t + D] + ds[b] (S_t,b - x0[b, col_t : col_t + D]), S_t,b the sum of
 *       that x0 slice.  Every slice has the same width D (1..128); 0..4 addends; no alignment beyond fp32.
 *   mm_wide_rows_apply      optimizer step of DeepFM's wide kernel (wide_rows, 1) by the rule of mm_sparse_rows_apply:
 *       block i covers rows [offset, offset + rows) and is addressed by the batch's ids of feature i; every block's gradient
 *       values are grad (B,) (the ds of mm_deepfm_head_fwd_bwd).  Duplicates are summed, each touched row gets one
 *       update, untouched rows and their slots do not move (LazyAdam), ids outside [0, rows) are dropped.  acc (wide_rows,)
 *       fp32 all zero and rep_map (wide_rows,) int32 all INT32_MAX between calls.  The n_dense rows at dense_offsets_host
 *       (the continuous columns' rows) and the bias (nullable; its slots bias_state1 / bias_state2) take the dense rule
 *       with the gradients dense_grad (n_dense [+ 1],), which are then cleared.  Blocks must not overlap. */
typedef struct {
  const void* indices; /* (B,) ids, idx_bytes each (1, 2, 3, 4, 8) */
  int64_t rows;
  int64_t offset;      /* first row of the block in the wide kernel */
  int32_t idx_bytes;
  int32_t reserved;
} mm_wide_block;
int mm_deepfm_head_fwd_bwd(const float* x0, int64_t x0_stride, const int64_t* emb_cols_host, int D, const mm_wide_block* tables_host,
                           int n_tables, const mm_concat_piece* cont_host, const int64_t* cont_offsets_host, int n_cont,
                           const float* wide_kernel, const float* wide_bias, const float* h, int64_t h_stride, int units, int mask_h,
                           const float* w_dl, const float* b_dl, int act_dl, const float* out_w, const float* out_b, int loss_kind,
                           const void* targets, int target_dtype, const float* sample_weight, int64_t B, float* logits, float* loss,
                           float* ds, float* dh, int64_t dh_stride, float* dw_out, float* db_out, float* dw_dl, float* db_dl,
                           float* d_wide_bias, float* d_cont, int32_t* oob_count, void* stream);
int mm_fm_concat_backward(const float* const* addends_host, const int64_t* addend_strides_host, int n_addends, int64_t B, int d,
                          const float* x0, int64_t x0_stride, const float* ds, const mm_column_slice* slices_host, int n_slices,
                          void* stream);
int mm_wide_rows_apply(float* wide, float* state1, float* state2, int64_t wide_rows, const mm_wide_block* blocks_host, int n_blocks,
                       int64_t B, const float* grad, float* acc, int32_t* rep_map, const int64_t* dense_offsets_host, int n_dense,
                       float* dense_grad, float* bias, float* bias_state1, float* bias_state2, int opt, const float* hyper, void* stream);

/* ---------------------------------------------------------------------------------------
 * K16  Training step of the two-tower path (TwoTowerModel + ItemRetrievalTask, prediction_tasks/retrieval.py:33-191;
 * CategoricalCrossentropy(from_logits=True) against the one-hot on column 0, losses/listwise.py:38-50).  Added with
 * two-tower training; no existing entry point changed.
 *   mm_inbatch_softmax_ce_backward  backward of mm_inbatch_softmax_ce without the (B, 1+N) logits.  With s the logits of
 *       that call (s[b,0] = pos_logit[b]; s[b,1+n] = masked ? false_neg_score/T : (q_b.neg_n - log(neg_prob[n]+1e-16))/T,
 *       masked = downscore && pos_ids[b] == neg_ids[n]), lse[b] = stats[b,1] and p = exp(s - lse)
 *       (false_neg_score is taken for symmetry with the forward and not read: a masked logit is a constant):
 *         g[b,0] = c[b] (p[b,0] - 1) / T;  g[b,1+n] = masked ? 0 : c[b] p[b,1+n] / T   (the masked logits are constants)
 *         dq[b] = g[b,0] pos[b] + sum_n g[b,1+n] neg[n];  dpos[b] = g[b,0] q[b];  dneg[n] = sum_b g[b,1+n] q[b]
 *         *loss += sum_b c[b] (lse[b] - s[b,0])        (loss nullable; accumulated: zero it first)
 *       c = row_scale: (B,) device floats, or ONE device float when row_scale_is_scalar (1/B: Keras' mean).
 *       q_split / neg_split: the operands the forward read (mm_split_rows, Kp = mm_tc_padded_k(D) <= 128, 16-B aligned);
 *       stats (B,3): mm_inbatch_softmax_ce's output; q, pos (B, D), dq, dpos (B, D), dneg (N, D): contiguous fp32.
 *       dpos may alias dneg when the negatives are the positives (in-batch, N == B): the sum is written.  dq aliases
 *       neither.  Two wgmma kernels recompute the logits tile by tile (inbatch_flash_kernel<SoftmaxCE, DQ>: one CTA per
 *       128 queries; <SoftmaxCE, DN>: one CTA per 128 negatives), each output row is written by one CTA: deterministic.
 *       Errors before any launch: MM_ERR_ARG (null pointer, T <= 0, N <= 0, ids missing for down-scoring, dpos == dneg with
 *       N != B), MM_ERR_UNSUPPORTED (D > 128, sizes >= 2^31), MM_ERR_ALIGN (split operands not 16-B aligned, an fp32
 *       buffer not 4-B aligned).  Arguments that break several rules get the code of one of them, not a fixed one.
 *   mm_l2_normalize_backward  backward of mm_l2_normalize from its INPUT x: s = sum(x^2), n = sqrt(s), y = x / n;
 *       s >= 1e-12: dx = (dy - y (y.dy)) / n, else dx = dy / 1e-6 (TF's gradient of maximum(s, 1e-12) flows to s only
 *       where s >= 1e-12).  dx may alias x or dy.
 * ------------------------------------------------------------------------------------- */
int mm_inbatch_softmax_ce_backward(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                                   const void* neg_ids, int id_dtype, int downscore, float false_neg_score, const float* neg_prob,
                                   float temperature, const float* stats, const float* q, const float* pos, const float* row_scale,
                                   int row_scale_is_scalar, float* dq, float* dpos, float* dneg, float* loss, void* stream);
int mm_l2_normalize_backward(const float* x, const float* dy, int64_t B, int D, int64_t x_stride, int64_t dy_stride, float* dx,
                             int64_t dx_stride, void* stream);

/* ---------------------------------------------------------------------------------------
 * K17  Evaluation metrics of the ranking outputs (Keras metrics of BinaryOutput / RegressionOutput: AUC, Precision,
 * Recall, BinaryAccuracy, RootMeanSquaredError, and the compiled loss), accumulated on the device.  Added with
 * RankingModel.evaluate; no existing entry point changed.
 *   mm_metrics_update  reads the LOGITS z (H, M) of H <= 8 heads (the (H, M) layout of mm_heads_fwd_bwd / mm_mlp_tc_heads)
 *       and ADDS this batch into state, H blocks of MM_METRICS_SCALARS + 4 * num_buckets fp64 values (zero it first):
 *         [MM_METRICS_LOSS]    sum sample_weight * l,  l = BCE max(z,0) - z y + log(1 + e^-|z|) | MSE (z - y)^2
 *         [MM_METRICS_COUNT]   samples;   [MM_METRICS_INVALID]  samples with a NaN z / y or a binary target outside {0, 1}
 *                              (they add nothing else)
 *         metric set s (0, 1 < n_sets) at MM_METRICS_SET0 + s * MM_METRICS_SET_STRIDE, w = metric_weights[s][i] or 1:
 *           binary heads: +POS / +NEG sum w of y = 1 / y = 0, +TP + t / +FP + t sum w of y = 1 / y = 0 with p > thresholds[t];
 *           regression heads: +SQ_ERR sum w (z - y)^2, +W_SUM sum w
 *         binary heads, after the scalars: per set [pos | neg] num_buckets each: sum w of y = 1 / y = 0 in bucket
 *           max(ceil(fp32(p) * fp32(num_buckets - 1)) - 1, 0)   (the evenly spaced thresholds of Keras' AUC)
 *       p = sigmoid(z) by pred_form: MM_PRED_ACT 1 / (1 + expf(-z)) (the epilogues that take MM_ACT_SIGMOID) or MM_PRED_HEAD
 *       the |z|-stable form of mm_heads_fwd_bwd; either is bit-identical to the forward that produced z.  heads_host is a HOST
 *       array.  workspace: mm_metrics_workspace_bytes(M, H) bytes of device scratch (one partial per CTA, added in CTA order:
 *       with null metric weights the result does not depend on scheduling; weighted buckets use fp64 atomics).
 *       2 <= num_buckets <= MM_METRICS_MAX_BUCKETS, n_sets 1 or 2.
 * ------------------------------------------------------------------------------------- */
#define MM_METRICS_MAX_HEADS 8
#define MM_METRICS_MAX_THRESHOLDS 4
#define MM_METRICS_MAX_BUCKETS 1024
#define MM_METRICS_LOSS 0
#define MM_METRICS_COUNT 1
#define MM_METRICS_INVALID 2
#define MM_METRICS_SET0 3
#define MM_METRICS_SET_STRIDE 12
#define MM_METRICS_POS 0
#define MM_METRICS_NEG 1
#define MM_METRICS_SQ_ERR 2
#define MM_METRICS_W_SUM 3
#define MM_METRICS_TP 4
#define MM_METRICS_FP 8
#define MM_METRICS_SCALARS 27
#define MM_PRED_ACT 0
#define MM_PRED_HEAD 1
typedef struct {
  const void* targets;              /* (M,) of target_dtype (MM_I32 .. MM_F64) */
  const float* sample_weight;       /* (M,) weights of the loss, nullable */
  const float* metric_weights[2];   /* (M,) weights of metric set 0 / 1, nullable */
  int32_t target_dtype;
  int32_t loss_kind;                /* MM_LOSS_BCE / MM_LOSS_MSE */
  int32_t pred_form;                /* MM_PRED_ACT / MM_PRED_HEAD */
  int32_t n_thresholds;             /* 0 .. MM_METRICS_MAX_THRESHOLDS */
  float thresholds[4];
} mm_metrics_head;
int64_t mm_metrics_workspace_bytes(int64_t M, int H);
int mm_metrics_update(const float* logits, int64_t M, int H, const mm_metrics_head* heads_host, int num_buckets, int n_sets,
                      double* state, void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * K18  Wide&Deep head (WideAndDeepModel, models/ranking.py:276-570; CategoryEncoding, transforms/features.py:473-612).
 * Added with WideAndDeepModel; no existing entry point changed.  The wide branch is Dense(1) over the concatenated
 * CategoryEncoding of each wide feature: a block of (int_domain.max + 1) rows of the wide kernel per feature.
 *   mm_wide_bag: one bag (list) feature of the wide branch.  values (nnz,) ids of idx_bytes (1, 2, 3, 4, 8); offsets
 *       (B + 1,) of off_dtype (MM_I32 / MM_I64): bag b = positions [offsets[b], offsets[b+1]) clamped to [0, nnz] (an end
 *       below the start is an empty bag; positions no bag covers are ignored), or offsets null: fixed length, bag b =
 *       [b length, (b + 1) length) and nnz = B length.  mode MM_WIDE_MULTI_HOT: each distinct id of a bag counts once
 *       (Keras bincount(binary_output=True)); MM_WIDE_COUNT: every occurrence counts.  Deduplication compares each
 *       position with the earlier positions of its bag (quadratic in the bag length).  The gradient matches the forward
 *       when the offsets are non-decreasing; other offsets are never read or written outside their arrays.
 *   mm_wide_deep_head_fwd_bwd  one pass over the batch:
 *       wide = sum over one-hot blocks wide_kernel[offset + id] + sum over bags (by mode) wide_kernel[offset + id] + *wide_bias
 *       u = h . w_dl + *b_dl;  s = wide + act_dl(u);  z = s *out_w + *out_b
 *       h null: no deep part (s = wide); no blocks: no wide part (s = act_dl(u) + *wide_bias).
 *     targets null: forward only, out (B,) = out_act(z); loss_kind, ds, dh and the gradients are not read.
 *     otherwise out (B,) = z, delta = dloss/dz as mm_heads_fwd_bwd (BCE sw (sigmoid(z) - y) / B | MSE sw 2 (z - y) / B),
 *       ds (B,) = delta *out_w, du = ds act_dl'(u), dh (B, units) = du w_dl (zeroed where h <= 0 when mask_h);
 *       ACCUMULATES loss (2,) += [loss, loss], *dw_out += sum delta s, *db_out += sum delta, dw_dl (units,) += sum du h,
 *       *db_dl += sum du, *d_wide_bias += sum ds (each nullable).
 *     Ids outside [0, rows) add nothing and bump *oob_count.  out_w / out_b / wide_bias / b_dl: DEVICE scalars (nullable
 *     but out_w).  units <= 512; act_dl linear or relu; <= 64 one-hot blocks and <= 32 bags.
 *   mm_wide_bag_grad  one bag feature's gradient as nnz pairs: out_ids[i] = values[i] and out_values[i] = ds[bag(i)] for
 *       every position that adds a term in the forward (MM_WIDE_COUNT: every in-range id; MM_WIDE_MULTI_HOT: the first
 *       occurrence of each id in its bag), out_ids[i] = -1 and out_values[i] = 0 for repeated occurrences, ids outside
 *       [0, rows) and positions no bag covers.  Passed to mm_wide_rows_apply as one block of B = nnz samples with int64
 *       ids (idx_bytes 8), the block's rows / offset and grad = out_values.
 * ------------------------------------------------------------------------------------- */
#define MM_WIDE_MULTI_HOT 0
#define MM_WIDE_COUNT 1
typedef struct {
  const void* values;  /* (nnz,) ids, idx_bytes each */
  const void* offsets; /* (B + 1,) or null: fixed length */
  int64_t rows;
  int64_t offset;      /* first row of the block in the wide kernel */
  int64_t nnz;
  int32_t idx_bytes;
  int32_t off_dtype;
  int32_t length;      /* ids per sample when offsets is null */
  int32_t mode;        /* MM_WIDE_MULTI_HOT / MM_WIDE_COUNT */
} mm_wide_bag;
int mm_wide_deep_head_fwd_bwd(const mm_wide_block* onehot_host, int n_onehot, const mm_wide_bag* bags_host, int n_bags,
                              const float* wide_kernel, const float* wide_bias, const float* h, int64_t h_stride, int units,
                              int mask_h, const float* w_dl, const float* b_dl, int act_dl, const float* out_w, const float* out_b,
                              int out_act, int loss_kind, const void* targets, int target_dtype, const float* sample_weight,
                              int64_t B, float* out, float* loss, float* ds, float* dh, int64_t dh_stride, float* dw_out,
                              float* db_out, float* dw_dl, float* db_dl, float* d_wide_bias, int32_t* oob_count, void* stream);
int mm_wide_bag_grad(const mm_wide_bag* bag_host, int64_t B, const float* ds, int64_t* out_ids, float* out_values, void* stream);

/* ---------------------------------------------------------------------------------------
 * K19  MMoE gates, expert mixture and output heads (MMOEBlock, blocks/experts.py:37-208; OutputBlock, outputs/block.py).
 * Added with MMOEBlock; no existing entry point changed.
 *   mm_mmoe_heads_fwd_bwd  one pass over the batch.  x (B, E U): the E experts' last-layer outputs side by side (expert e
 *       at columns [e U, (e + 1) U)); gate_logits_host[t] (B, E) with row stride gate_strides_host[t]: task t's gate logits
 *       (host arrays of H device pointers / strides).  w (U, H) Keras layout, bias (H,) nullable; losses, loss weights,
 *       targets, sample weights and the loss vector as mm_heads_fwd_bwd.
 *       p_t = softmax(L_t / temperature),  m_t = sum_e p_t,e x_e,  z_t = m_t . w[:, t] + bias[t]   (m_t is never stored)
 *     targets null: forward only, logits (H, B) = the activated predictions (mm_heads_fwd_bwd's sigmoid form, or z for MSE);
 *       loss_weight, dx, the gate-logit gradients and dw / db are not read.
 *     otherwise logits (H, B) = z, delta_t = dloss/dz_t as mm_heads_fwd_bwd, dm_t = delta_t w[:, t];
 *       dx (B, E U) = sum_t p_t,e dm_t (zeroed where x <= 0 when mask_relu), d_gate_logits_host[t] (B, E) =
 *       p_t (dg_t - <p_t, dg_t>) / temperature with dg_t,e = <dm_t, x_e>; ACCUMULATES loss (1 + H), dw (U, H) += m_t delta_t,
 *       db (H,) += delta_t (dw / db nullable).
 *     E <= 16, U <= 256, 1 <= H <= 8, temperature > 0.
 * ------------------------------------------------------------------------------------- */
int mm_mmoe_heads_fwd_bwd(const float* x, int64_t B, int E, int U, int64_t x_stride, const float* const* gate_logits_host,
                          const int64_t* gate_strides_host, int H, float temperature, const float* w, const float* bias,
                          const int* loss_kind, const float* loss_weight, const void* const* targets, const int* target_dtypes,
                          const float* const* sample_weights, float* logits, float* loss, float* dx, int64_t dx_stride,
                          int mask_relu, float* const* d_gate_logits_host, const int64_t* d_gate_strides_host, float* dw,
                          float* db, void* stream);
/* The task-tower path: the gates and mixture alone, then H heads with one input per task.
 *   mm_mmoe_mix_fwd  p (B, H E) = the gate weights softmax(L_t / temperature) side by side (saved for the backward);
 *       m (H, B, U) contiguous: m[t] = sum_e p_t,e x_e; m_split (H, B, 2 Kp) nullable: m[t]'s split-bf16 operand
 *       (mm_split_rows layout, Kp = mm_tc_padded_k(U), padding written as zeros).
 *   mm_mmoe_mix_bwd  from dm (H, B, U): dx (B, E U) = sum_t p_t,e dm_t (zeroed where x <= 0 when mask_relu) and
 *       d_gate_logits_host[t] (B, E) = p_t (dg_t - <p_t, dg_t>) / temperature with dg_t,e = <dm_t, x_e>.
 *   mm_mmoe_task_heads_fwd_bwd  head t reads x_host[t] (B, K) (row stride x_strides_host[t]): z_t = x_t . w[:, t] + bias[t],
 *       w (K, H); losses, targets, sample weights, the loss vector, dw / db (accumulated) and the forward-only form as
 *       mm_heads_fwd_bwd; training writes dx_host[t] (B, K) = delta_t w[:, t] (zeroed where x_t <= 0 when mask_relu).
 *     E <= 16, U <= 256, K <= 256, 1 <= H <= 8, temperature > 0. */
int mm_mmoe_mix_fwd(const float* x, int64_t B, int E, int U, int64_t x_stride, const float* const* gate_logits_host,
                    const int64_t* gate_strides_host, int H, float temperature, float* p, float* m, void* m_split, int Kp,
                    void* stream);
int mm_mmoe_mix_bwd(const float* x, int64_t B, int E, int U, int64_t x_stride, const float* p, int H, float temperature,
                    const float* dm, float* dx, int64_t dx_stride, int mask_relu, float* const* d_gate_logits_host,
                    const int64_t* d_gate_strides_host, void* stream);
int mm_mmoe_task_heads_fwd_bwd(const float* const* x_host, const int64_t* x_strides_host, int64_t B, int K, int H, const float* w,
                               const float* bias, const int* loss_kind, const float* loss_weight, const void* const* targets,
                               const int* target_dtypes, const float* const* sample_weights, float* logits, float* loss,
                               float* const* dx_host, const int64_t* dx_strides_host, int mask_relu, float* dw, float* db,
                               void* stream);

/* ---------------------------------------------------------------------------------------
 * K20  Neural collaborative filtering head (NCFModel, models/benchmark.py:32-100): the GMF branch
 *      (MatrixFactorizationBlock with ElementWiseMultiply) next to the MLP branch's output h, concatenated as [mf | mlp]
 *      and read by the output heads.
 *   mm_ncf_head_fwd_bwd  in one pass over the batch: u = table_u[ids_u[b]], i = table_i[ids_i[b]] (D wide; ids of
 *       idx_bytes 1, 2, 3, 4 or 8 as mm_lookup_table's, checked alike; an id outside [0, rows) reads a zero row and bumps
 *       *oob_count, nullable), z_t = [u * i | h] . w[:, t] + bias[t] with w the (D + U, H) Keras kernel and h (B, U) rows
 *       h_stride apart.  Losses, targets, sample weights, loss weights, the loss vector (1 + H) and the forward-only form
 *       (targets null: out (H, B) = the activated predictions) as mm_heads_fwd_bwd; training writes out = the logits,
 *         du (B, D) = r * i + 2 l2 u,  di (B, D) = r * u + 2 l2 i,  r = sum_t delta_t w[:D, t]  (contiguous rows in sample
 *         order: the IndexedSlices values of both tables),
 *         dh (B, U) = sum_t delta_t w[D:, t] (zeroed where h <= 0 when relu_h; rows dh_stride apart)
 *       and ACCUMULATES dw (D + U, H), db (H,) (nullable) and the loss.  reg (1 device float, nullable) ACCUMULATES
 *       l2 sum_b (|u_b|^2 + |i_b|^2 + |x_reg_b|^2), x_reg (B, x_reg_width) rows x_reg_stride apart (nullable: none); in
 *       training the term is also added to loss[0].  1 <= D <= 128, 1 <= U <= 256, 1 <= H <= 8, l2 finite and >= 0. */
int mm_ncf_head_fwd_bwd(const float* table_u, int64_t rows_u, const void* ids_u, int idx_bytes_u, const float* table_i,
                        int64_t rows_i, const void* ids_i, int idx_bytes_i, int D, const float* h, int64_t h_stride, int U,
                        int relu_h, int64_t B, int H, const float* w, const float* bias, const int* loss_kind,
                        const float* loss_weight, const void* const* targets, const int* target_dtypes,
                        const float* const* sample_weights, float l2, const float* x_reg, int64_t x_reg_stride, int x_reg_width,
                        float* out, float* loss, float* reg, float* du, float* di, float* dh, int64_t dh_stride, float* dw,
                        float* db, int32_t* oob_count, void* stream);

/* ---------------------------------------------------------------------------------------
 * K21  In-batch pairwise ranking losses of the retrieval step (losses/pairwise.py: BPR, BPR-max, TOP1, TOP1-v2,
 * TOP1-max, logistic, hinge), forward and backward without the (B, N) scores.  Added with the pairwise retrieval
 * losses; no existing entry point changed.
 *   Scores: sp[b] = pos_logit[b] (mm_positive_scores, already / T); s[b,n] = masked ? false_neg_score / T : q_b.neg_n / T
 *   with masked = downscore && pos_ids[b] == neg_ids[n] (a constant: no gradient).  d = sp - s, w = softmax_n(s[b,:]),
 *   eps0(x) = (x == 0 ? x + 1e-24 : x) decided on float32 values computed without flush-to-zero.  Per element:
 *     MM_PAIRWISE_BPR       -log(eps0(sigmoid(d)))
 *     MM_PAIRWISE_BPR_MAX   -log(eps0(sigmoid(d) w)) + reg_lambda s^2 w
 *     MM_PAIRWISE_TOP1      sigmoid(-d) + sigmoid(s^2)
 *     MM_PAIRWISE_TOP1_V2   as TOP1, plus - sigmoid(sp^2) once per row
 *     MM_PAIRWISE_TOP1_MAX  (sigmoid(-d) + sigmoid(s^2)) w
 *     MM_PAIRWISE_LOGISTIC  relu(-d) + log1p(eps0(exp(-|d|)))
 *     MM_PAIRWISE_HINGE     relu(1 - d)
 *   loss = c sum over the B N elements (+ the TOP1_V2 row terms), c = 1 / (B N): Keras' mean over the (B, N) losses
 *   (TOP1_V2: its mean over N, then over B).  Masked elements take part with their constant score.
 *   mm_inbatch_pairwise_fwd  stats (B, 4) = [row loss, dloss/dsp (without c / T), lse over the row's negatives, A] (lse
 *       and A: the -max kinds' soft-max terms the backward reads); loss (nullable) += c sum_b stats[b, 0] in a fixed
 *       order (zero it first).  One CTA per 128 queries streams the negatives once, the -max kinds twice (the first
 *       pass finds the log-sum-exp the eps0 decision needs).
 *   mm_inbatch_pairwise_bwd  from the forward's stats: g = c / T dloss/ds,
 *         dq[b] = c / T stats[b, 1] pos[b] + sum_n g[b,n] neg[n];  dpos[b] = c / T stats[b, 1] q[b];  dneg[n] = sum_b g[b,n] q[b]
 *       dpos may alias dneg when the negatives are the positives (N == B): the sum is written; dq aliases neither.  Two
 *       wgmma kernels recompute the scores tile by tile (one CTA per 128 queries / per 128 negatives); each output row
 *       is written by one CTA: deterministic.
 *   Both: q_split / neg_split the split-bf16 operands (mm_split_rows, Kp = mm_tc_padded_k(D) <= 128, 16-B aligned),
 *   pos_logit (B,), stats 16-B aligned, q, pos (B, D), dq, dpos (B, D), dneg (N, D) contiguous fp32.  Errors before any
 *   launch: MM_ERR_ARG (null pointer, T <= 0, N <= 0, unknown kind, reg_lambda not finite, ids missing for
 *   down-scoring, dpos == dneg with N != B), MM_ERR_UNSUPPORTED (D > 128, sizes >= 2^31), MM_ERR_ALIGN.  Arguments that
 *   break several rules get the code of one of them, not a fixed one.
 * ------------------------------------------------------------------------------------- */
#define MM_PAIRWISE_BPR 0
#define MM_PAIRWISE_BPR_MAX 1
#define MM_PAIRWISE_TOP1 2
#define MM_PAIRWISE_TOP1_V2 3
#define MM_PAIRWISE_TOP1_MAX 4
#define MM_PAIRWISE_LOGISTIC 5
#define MM_PAIRWISE_HINGE 6
int mm_inbatch_pairwise_fwd(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                            const void* neg_ids, int id_dtype, int downscore, float false_neg_score, float temperature, int kind,
                            float reg_lambda, const float* pos_logit, float* stats, float* loss, void* stream);
int mm_inbatch_pairwise_bwd(const void* q_split, const void* neg_split, int64_t B, int64_t N, int D, const void* pos_ids,
                            const void* neg_ids, int id_dtype, int downscore, float false_neg_score, float temperature, int kind,
                            float reg_lambda, const float* pos_logit, const float* stats, const float* q, const float* pos,
                            float* dq, float* dpos, float* dneg, void* stream);

/* ---------------------------------------------------------------------------------------
 * K22  Backward of the full-catalog soft-max cross-entropy (CategoricalOutput over a weight-tied EmbeddingTable,
 * outputs/classification.py:127-216 and :311-382; CategoricalCrossentropy(from_logits=True)) without the (B, N) logits.
 * Added with catalog training; no existing entry point changed.
 *   mm_catalog_softmax_ce_backward  x_split = mm_split_rows(x / T) (the tempered queries), e_split = mm_split_rows(E)
 *       (N, D), bias (N,) = b / T or null, T = temperature: the operands mm_catalog_score read for stats (B, 3).  With
 *       s[b,j] = (x_b / T).e_j + b_j / T recomputed from them exactly as that call did, p = exp(s - stats[b,1]) and
 *       y = labels (B,) (label_dtype MM_I32 / MM_I64):
 *         G[b,j] = c[b] (p[b,j] - [j == y_b])
 *         dx[b] = 1/T sum_j G[b,j] e_j  (the gradient of x itself);  de[j] = sum_b G[b,j] x_b / T;  db[j] = 1/T sum_b G[b,j]
 *         *loss += sum_b c[b] (stats[b,1] - stats[b,2])   (loss nullable; accumulated: zero it first)
 *       c = row_scale: (B,) device floats, or ONE device float when row_scale_is_scalar.  db nullable (no bias gradient).
 *       A label outside [0, N) is never used as an address: it matches no column, so its row's gradient keeps the
 *       soft-max term only (and mm_catalog_score leaves its target logit NaN), and it adds one to *oob_count (nullable,
 *       int32: the out-of-range counter of the gathers, which the trainers read after the step).  dx (B, D), de (N, D), db (N,): fp32,
 *       contiguous, dx and de distinct.  Two wgmma kernels (inbatch_flash_kernel<CatalogCE, DQ / DN>): one CTA per 128 queries
 *       streaming the catalog and one per 128 catalog rows streaming the queries; each output row is written by one CTA.
 *       When ceil(B / 128) is below the SM count the dq kernel splits the catalog over several CTAs per query tile, which
 *       write partial dx into `workspace` that one more kernel sums in split order: deterministic, no atomics.  Both
 *       kernels add their wgmma accumulator into their own output rows every 256 streamed tiles (long fp32 accumulations
 *       on wgmma lose magnitude), so the workspace stays below 128 * SMs * D floats for any catalog.
 *       workspace: at least mm_catalog_softmax_ce_workspace_bytes(B, N, D) bytes, 16-B aligned (null when that is 0).
 *       Errors before any launch: MM_ERR_ARG (null pointer, T <= 0, N <= 0, bad label dtype, workspace too small),
 *       MM_ERR_UNSUPPORTED (D > 128, sizes >= 2^31), MM_ERR_ALIGN.  Arguments that break several rules get the code of
 *       one of them, not a fixed one.
 *   mm_catalog_softmax_ce_workspace_bytes  the workspace those shapes need (0: no split); depends on the device's SM count.
 * ------------------------------------------------------------------------------------- */
int64_t mm_catalog_softmax_ce_workspace_bytes(int64_t B, int64_t N, int D);
int mm_catalog_softmax_ce_backward(const void* x_split, const void* e_split, int64_t B, int64_t N, int D, const float* bias,
                                   const void* labels, int label_dtype, float temperature, const float* stats,
                                   const float* row_scale, int row_scale_is_scalar, float* dx, float* de, float* db, float* loss,
                                   int* oob_count, void* workspace, int64_t workspace_bytes, void* stream);

/* K22 with label smoothing (Keras CategoricalCrossentropy(from_logits=True, label_smoothing=eps): the target is
 * (1 - eps) onehot(y) + eps / N).  Added with label-smoothed catalog training; no existing entry point changed.
 *   mm_catalog_smoothed_ce_backward  the arguments of mm_catalog_softmax_ce_backward and label_smoothing = eps in [0, 1).
 *       eps == 0 runs exactly mm_catalog_softmax_ce_backward (same kernels, same workspace, bit-identical outputs).  For
 *       eps > 0, with s_E = sum_j e_j (D,), beta = sum_j bias_j (bias already b / T; 0 when null) and u[b] =
 *       (eps / N) ((x_b / T).s_E + beta), the mean logit times eps:
 *         G[b,j] = c[b] (p[b,j] - (1 - eps) [j == y_b] - eps / N)
 *         dx[b] = 1/T sum_j G[b,j] e_j;  de[j] = sum_b G[b,j] x_b / T;  db[j] = 1/T sum_b G[b,j]
 *         *loss += sum_b c[b] (stats[b,1] - (1 - eps) stats[b,2] - u[b])
 *       The wgmma kernels (inbatch_flash_kernel<SmoothedCatalogCE, DQ / DN>) weigh the one-hot by 1 - eps; the uniform
 *       part is rank one and is added where each output row is written, from two fixed-order column reductions per call
 *       (of e_split with the bias, and of x_split weighted by c), so the (N, D) de is not passed over twice.  An
 *       out-of-range label keeps K22's rule (no one-hot term, counted in *oob_count, loss NaN); its uniform term applies.
 *       workspace: at least mm_catalog_smoothed_ce_workspace_bytes(B, N, D) bytes (eps == 0: K22's), 16-B aligned.
 *       Errors before any launch: K22's, and MM_ERR_ARG for eps outside [0, 1).
 *   mm_catalog_mean_logit  out[b] = mean_j ((x_b / T).e_j + bias_j) over the N catalog rows (the uniform target's logit,
 *       for the smoothed loss of an evaluation pass): x_split (B, 2*Kp), e_split (N, 2*Kp), bias (N,) or null, out (B,)
 *       fp32; the same column reduction, then one warp per row.  workspace: mm_catalog_mean_logit_workspace_bytes(N)
 *       bytes (the column reduction's partials and sums), 16-B aligned.  Errors before any launch: MM_ERR_ARG,
 *       MM_ERR_UNSUPPORTED (D > 128), MM_ERR_ALIGN.
 *   mm_catalog_smoothed_ce_workspace_bytes  the backward's workspace for those shapes; depends on the device's SM count.
 * ------------------------------------------------------------------------------------- */
int64_t mm_catalog_smoothed_ce_workspace_bytes(int64_t B, int64_t N, int D);
int mm_catalog_smoothed_ce_backward(const void* x_split, const void* e_split, int64_t B, int64_t N, int D, const float* bias,
                                    const void* labels, int label_dtype, float temperature, float label_smoothing,
                                    const float* stats, const float* row_scale, int row_scale_is_scalar, float* dx, float* de,
                                    float* db, float* loss, int* oob_count, void* workspace, int64_t workspace_bytes,
                                    void* stream);
int64_t mm_catalog_mean_logit_workspace_bytes(int64_t N);
int mm_catalog_mean_logit(const void* x_split, const void* e_split, int64_t B, int64_t N, int D, const float* bias, float* out,
                          void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * K23  IndexedSlices into a dense gradient (the weight-tied catalog step: the tied table's input-side rows added to the
 * output side's dE).  Added with the catalog training step; no existing entry point changed.
 *   mm_slices_add_dense  dense[ids[i]] += rows[i] for i in [0, n): ids (n,) MM_I32 / MM_I64, rows (n, D) fp32 contiguous,
 *       dense (N, D) fp32 contiguous.  An id outside [0, N) (a multi-hot expansion's -1, an out-of-range id the gathers
 *       counted) adds nothing.  Duplicate ids are summed in index order and each dense row has one writer: a stable radix
 *       sort of the ids (8-bit digits, ceil(log2(N + 1) / 8) passes), then each run of equal ids summed in 256-position
 *       pieces whose partials are added in piece order (a run of length r costs one group at most 256 + r / 256 row
 *       additions); no float atomics, so repeats are bit-identical.  4 <= D <= 128, D % 4 == 0; n, N < 2^31.  workspace: at least
 *       mm_slices_add_dense_workspace_bytes(n) bytes, 16-B aligned.  Errors before any launch: MM_ERR_ARG, MM_ERR_UNSUPPORTED,
 *       MM_ERR_ALIGN.
 *   mm_slices_add_dense_workspace_bytes  the workspace of n slices (0 for n <= 0).
 * ------------------------------------------------------------------------------------- */
int64_t mm_slices_add_dense_workspace_bytes(int64_t n);
int mm_slices_add_dense(const void* ids, int idx_dtype, const float* rows, int64_t n, int D, float* dense, int64_t N,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * K24  Pretrained embeddings (PretrainedEmbeddings, inputs/embedding.py:717-800; the dataloader's EmbeddingOperator):
 * rows of a device-resident fp32 matrix P (rows, Dp) at row stride p_stride, looked up by ids (B,) MM_I32 / MM_I64, go
 * straight into their slot of the input block's concat.  ids == NULL reads row b of a dense (B, Dp) input instead
 * (rows >= B).  An id outside [0, rows) reads a zero row and adds 1 to *oob_count (when non-null), once per sample.
 * Added with the pretrained input slots; no existing entry point changed.
 *   mm_pretrained_gather  out[b, 0:Dp] = P[ids[b]]; `out` points at the slot's first column, columns outside [0, Dp) of
 *       each row are not written.  1 <= Dp <= MM_PRETRAINED_MAX_DIM.
 *   mm_pretrained_project  out[b, 0:N] = P[ids[b]] W + bias (W (Dp, N) fp32 contiguous, bias (N,) or NULL), fp32
 *       products in ascending k; the gathered rows are staged in shared memory only.  1 <= N <= MM_PRETRAINED_MAX_OUT.
 *       Grid: min(ceil(B/64) * ceil(N/64), MM_PRETRAINED_CTAS_PER_SM * SMs) CTAs of 256 threads over the 64x64 tiles.
 *   mm_pretrained_project_backward  g = sum of the n_addends (1..4) (B, N) matrices (each at its own row stride; pass
 *       pointers to the slot's first column), through the l2-norm backward at the pre-norm projection ypre when non-null
 *       (mm_l2_normalize_backward's rule), then dW (Dp, N) = P[ids]^T g and db (N,) = sum_b g (db may be NULL), both
 *       overwritten.  Fixed row chunks (a function of B, Dp, N) and a chunk-ordered sum: repeats are bit-identical.
 *       workspace: mm_pretrained_backward_workspace_bytes(B, Dp, N) bytes, 16-B aligned; that size is non-decreasing in B,
 *       so a workspace sized for B serves every batch of at most B samples.
 * Errors before any launch: MM_ERR_ARG, MM_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------- */
#define MM_PRETRAINED_MAX_DIM 1024
#define MM_PRETRAINED_MAX_OUT 256
#define MM_PRETRAINED_CTAS_PER_SM 8
int mm_pretrained_gather(const float* P, int64_t rows, int Dp, int64_t p_stride, const void* ids, int idx_dtype, int64_t B,
                         float* out, int64_t out_stride, int32_t* oob_count, void* stream);
int mm_pretrained_project(const float* P, int64_t rows, int Dp, int64_t p_stride, const void* ids, int idx_dtype, int64_t B,
                          const float* W, const float* bias, int N, float* out, int64_t out_stride, int32_t* oob_count,
                          void* stream);
int64_t mm_pretrained_backward_workspace_bytes(int64_t B, int Dp, int N);
int mm_pretrained_project_backward(const float* P, int64_t rows, int Dp, int64_t p_stride, const void* ids, int idx_dtype,
                                   int64_t B, const float* const* addends, const int64_t* addend_strides, int n_addends,
                                   const float* ypre, int64_t y_stride, int N, float* dW, float* db, void* workspace,
                                   int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * K25  Learning-rate schedules evaluated on the device (tf.keras.optimizers.schedules of TF 2.9-2.12), so a captured CUDA
 * graph follows the schedule without host work.  Added with schedules and per-block optimizers; no existing entry point
 * changed.
 *   mm_opt_tick_schedule  s = hyper[MM_HYPER_STEP] (the optimizer's `iterations` before this step's update);
 *       hyper[MM_HYPER_LR] = lr(s) in fp32; then what mm_opt_tick does: step = s + 1 and
 *       hyper[MM_HYPER_LR_T] = lr(s) sqrt(1 - b2^(s+1)) / (1 - b1^(s+1)).  One thread.
 *   sched: device float[MM_SCHED_COUNT]: [MM_SCHED_KIND] one of MM_SCHED_*, then the schedule's parameters
 *       (init = initial_learning_rate, decay_steps > 0, rate = decay_rate / end_learning_rate / alpha, power,
 *       flag = staircase / cycle as 0 or 1) and, for MM_SCHED_PIECEWISE, nb (1..MM_SCHED_MAX_BOUNDARIES) increasing
 *       boundaries and nb + 1 values.  lr(s), p = s / decay_steps (floored when staircase):
 *         EXPONENTIAL   init * rate^p
 *         PIECEWISE     values[0] if s <= b[0]; values[i] if b[i-1] < s <= b[i]; values[nb] if s > b[nb-1]
 *         POLYNOMIAL    (init - rate) * (1 - s'/D)^power + rate; no cycle: s' = min(s, decay_steps), D = decay_steps;
 *                       cycle: s' = s, D = decay_steps * max(1, ceil(s / decay_steps))
 *         INVERSE_TIME  init / (1 + rate * p)
 *         COSINE        init * ((1 - rate) * 0.5 * (1 + cos(pi * min(s, decay_steps) / decay_steps)) + rate)
 *   The step counter is fp32: it counts exactly up to 2^24 steps (the step after 16 777 216 stays at 16 777 216).
 *   An unknown kind or an out-of-range nb is refused by the host wrapper; the kernel leaves MM_HYPER_LR as it is then.
 * Errors before any launch: MM_ERR_ARG (null pointer).
 * ------------------------------------------------------------------------------------- */
#define MM_SCHED_EXPONENTIAL 1
#define MM_SCHED_PIECEWISE 2
#define MM_SCHED_POLYNOMIAL 3
#define MM_SCHED_INVERSE_TIME 4
#define MM_SCHED_COSINE 5
#define MM_SCHED_KIND 0
#define MM_SCHED_INIT 1
#define MM_SCHED_DECAY_STEPS 2
#define MM_SCHED_RATE 3
#define MM_SCHED_POWER 4
#define MM_SCHED_FLAG 5
#define MM_SCHED_NB 6
#define MM_SCHED_MAX_BOUNDARIES 32
#define MM_SCHED_BOUNDARIES 8
#define MM_SCHED_VALUES (MM_SCHED_BOUNDARIES + MM_SCHED_MAX_BOUNDARIES)
#define MM_SCHED_COUNT (MM_SCHED_VALUES + MM_SCHED_MAX_BOUNDARIES + 1)
int mm_opt_tick_schedule(float* hyper, const float* sched, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MM_B200_H_ */
