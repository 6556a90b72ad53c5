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
 * Tensor-core path (mma.sync bf16, 3-pass split, one warp per sample, cp.async.bulk row staging)
 * when F <= 32, D % 16 == 0, P in {0, D}, no self interaction; CUDA-core path otherwise.
 * ------------------------------------------------------------------------------------- */
int mm_dot_interaction(const float* x, int64_t B, int F, int D, int64_t x_stride,
                       const float* prefix, int P, int64_t prefix_stride, int self_interaction,
                       float* out, int64_t out_stride, void* out_split, int out_Kp, void* stream);

/* Fused K1+K5+K6+K3 for DLRM: gather T rows per sample straight into shared memory, append
 * the bottom-MLP vector at slot `bottom_slot`, write [bottom | interactions]; the (B,F,D)
 * stack never touches HBM.  tables[t].out_col is interpreted as slot(t)*D.  All dims == D. */
int mm_dlrm_gather_interact(const mm_gather_table* tables_host, int n_tables, int idx_dtype,
                            int64_t B, int D, const float* bottom, int64_t bottom_stride,
                            int bottom_slot, float* out, int64_t out_stride, void* out_split,
                            int out_Kp, int32_t* oob_count, void* stream);

/* Second-generation fused lookup + interaction (same result as mm_dlrm_gather_interact), with a richer
 * table descriptor:
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
 * F = n_tables + (bottom ? 1 : 0) <= 32, D in {16, 32, 64, 128}, world <= 8. */
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
 *   out_f32 : (M, N) fp32 (nullable);  out_split : (M, 2*Np_next) bf16 for the next layer
 *             (nullable; its padding columns are written as zeros)
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
 * within 227 KB of shared memory. */
int mm_mlp_tc_supported(int K, int n_layers, const int* widths, int with_head);
int mm_mlp_tc(const void* a_split, int64_t M, int K, int n_layers, const void* const* w_split,
              const int* widths, const float* const* bias, const int* acts, float* out,
              int64_t out_stride, const float* head_w, float head_b, int head_act, float* head_out,
              void* stream);

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

/* Whole-op entry points over fp32 Keras-layout weights (kernel (in, out) row-major, bias (out,) or
 * NULL) and a caller-provided workspace — for callers outside this package's Python host; nothing is
 * allocated, no pre-split weights are needed (the bf16 splits live in the workspace).
 *   mm_mlp_forward: MLPBlock, h_l = act_l(h_{l-1} W_l + b_l), 1..8 layers (blocks/mlp.py:97-139,
 *     :275-280); the whole-tower kernel when mm_mlp_tc_supported, else one wgmma launch per layer.
 *   mm_cross_forward: CrossBlock, x_{l+1} = x0 * (x_l W_l + b_l) + x_l, W_l (d, d)
 *     (blocks/cross.py:29-109, :188-202); depth > 1 needs x_stride == d.
 * workspace: 256-B aligned device memory of at least mm_*_workspace_bytes(...) (-1 on bad arguments). */
int64_t mm_mlp_workspace_bytes(int64_t M, int K, int n_layers, const int* widths);
int mm_mlp_forward(const float* x, int64_t M, int K, int64_t x_stride, int n_layers,
                   const float* const* kernels, const float* const* biases, const int* widths,
                   const int* acts, float* out, int64_t out_stride, void* workspace,
                   int64_t workspace_bytes, void* stream);
int64_t mm_cross_workspace_bytes(int64_t M, int d, int depth);
int mm_cross_forward(const float* x0, int64_t M, int d, int64_t x_stride, int depth,
                     const float* const* kernels, const float* const* biases, float* out,
                     int64_t out_stride, void* workspace, int64_t workspace_bytes, void* stream);

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
 *   mm_bce_head_fwd_bwd       Dense(K -> 1) + sigmoid + binary cross-entropy (Keras evaluates it on the logits),
 *                             forward AND backward in one pass over x (M, K), K <= 256:
 *                               z = x.w + b;  *loss_sum += sum_i sw_i (max(z,0) - z y + log(1 + e^-|z|)) / M;
 *                               dz = sw_i (sigmoid(z) - y) / M;  dx = dz w (zeroed where x <= 0 when mask_relu);
 *                               dw += x^T dz;  *db += sum dz.      loss_sum / dw / db are ACCUMULATED (zero them first).
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
 *   mm_dense_apply            the same update rules over a flat fp32 arena; g is scaled by grad_scale and CLEARED.
 *   mm_opt_tick               step counter += 1 and the Adam bias-corrected rate (once per step, before the applies)
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

int mm_bce_head_fwd_bwd(const float* x, int64_t M, int K, int64_t x_stride, const float* w, const float* bias,
                        const void* targets, int target_dtype, const float* sample_weight, float* logits,
                        float* loss_sum, float* dx, int64_t dx_stride, int mask_relu, float* dw, float* db, void* stream);
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
int mm_dense_apply(int opt, float* w, float* grad, float* state1, float* state2, int64_t n, const float* hyper,
                   float grad_scale, void* stream);
int mm_opt_tick(float* hyper, void* stream);
int mm_fill_i32(int32_t* p, int64_t n, int32_t value, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* MM_B200_H_ */
