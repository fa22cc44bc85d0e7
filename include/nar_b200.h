/*
 * nar_b200.h - C ABI of the H100-native NAR (CHAMELEON next-article recommendation)
 * training hot path.  libnar_b200.so exports exactly these symbols.
 *
 * The reference (gabrielspmoreira/chameleon_recsys @ 2e50af5) has NO native / FFI layer:
 * its boundary is the TF-Estimator Python contract (nar_module/nar/nar_trainer_gcom.py:234-332
 * model_fn, nar_module/nar/datasets.py:166-179 input_fn) and every "kernel" is a TensorFlow
 * 1.12 library op.  Each entry point below therefore cites the reference op group it
 * replaces (file:line of the TF call site) instead of a pre-existing FFI declaration.
 *
 * Conventions: extern "C"; plain pointers and sizes; every pointer is a DEVICE pointer
 * unless it says "host"; the caller owns every buffer; `stream` is a cudaStream_t passed
 * as void*; functions return 0 on success, a negative nar_status, or a positive
 * cudaError_t; nothing throws; no hidden global state beyond the opaque nar_ctx.
 * There is no CPU fallback anywhere: without a CUDA device every call fails.
 */
#ifndef NAR_B200_H
#define NAR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NAR_ABI_VERSION 3

typedef enum {
  NAR_OK = 0,
  NAR_ERR_INVALID = -1,        /* bad argument (null pointer, misaligned ld, size limit) */
  NAR_ERR_UNSUPPORTED = -2,    /* valid request the library does not implement */
  NAR_ERR_NO_DEVICE = -3,      /* no sm_90 device / driver entry point missing */
  NAR_ERR_WORKSPACE = -4       /* workspace too small */
} nar_status;

typedef struct nar_ctx nar_ctx;

/* ---- context ------------------------------------------------------------------------- */
int  nar_abi_version(void);
/* sizeof of an ABI struct as this library was compiled: 0 nar_feature_plan, 1 nar_model_cfg, 2 nar_step_io,
 * 3 nar_row_layout, 4 nar_gemm_epilogue, 5 nar_segment (bindings check their mirrors against it); -1 otherwise */
int  nar_abi_struct_size(int which);
const char* nar_status_string(int status);
int  nar_ctx_create(int device, nar_ctx** out);
int  nar_ctx_destroy(nar_ctx* ctx);

/* ---- feature-row gather  (replaces tf.nn.embedding_lookup nar_model.py:948 (ACR, frozen),
 *      :918 (trainable item embedding), tf.gather :929/:1067/:1095/:1138, tf.one_hot :734,
 *      small embedding_lookup :741, recency/novelty normalisation :996-1193, the concat
 *      :332/:992 and scale_center_features :905).  One output row per (position, item)
 *      pair; written straight into the GEMM A operand.                                     */
typedef enum {
  NAR_SEG_CTX_OHE = 0, NAR_SEG_CTX_EMBED = 1, NAR_SEG_CTX_NUM = 2, NAR_SEG_CTX_ZERO = 3,
  NAR_SEG_META_OHE = 4, NAR_SEG_META_EMBED = 5, NAR_SEG_META_NUM = 6,
  NAR_SEG_ACR = 7, NAR_SEG_ITEM_EMB = 8, NAR_SEG_RECENCY = 9, NAR_SEG_NOVELTY = 10
} nar_seg_kind;

typedef struct {
  int32_t kind;        /* nar_seg_kind */
  int32_t col;         /* first column in the output row */
  int32_t width;       /* columns written */
  int32_t card;        /* categorical cardinality (OHE / EMBED) */
  int32_t src;         /* index into ctx_int / ctx_float / meta pointer arrays */
  int32_t ld;          /* leading dimension of `table` (floats) */
  const float* table;  /* embedding table (EMBED, ACR, ITEM_EMB) */
  float* grad;         /* gradient table for trainable embeddings (backward only) */
} nar_segment;

#define NAR_MAX_SEGMENTS 24
#define NAR_MAX_SRC 16
#define NAR_MAX_COLS 1024

typedef struct {
  int32_t n_segments;
  int32_t row_ld;                       /* floats per output row (Fp) */
  nar_segment seg[NAR_MAX_SEGMENTS];
  const int64_t* ctx_int[NAR_MAX_SRC];  /* [B*T] int64 context ids per feature */
  const float*   ctx_float[NAR_MAX_SRC];/* [B*T] float context values per feature */
  const int64_t* meta[NAR_MAX_SRC];     /* [V] int64 metadata per feature */
  const int64_t* created_at_ts;         /* [V] int64 ms */
  const float*   pop_norm;              /* [V] articles_recent_pop_norm */
  const float*   gamma;                 /* [Fp] scale  (nar_model.py:891) */
  const float*   beta;                  /* [Fp] centre (nar_model.py:895) */
  const float*   stats;                 /* [3][8] normalisation stats (input / positive / negative rows), see nar_feature_stats */
  float log_base_recency;               /* elapsed_days_smooth_log_base */
  float log_base_novelty;               /* popularity_smooth_log_base */
  /* column map: col_seg[c] = index into seg[] of the segment that owns output column c, 255 = padding.
   * narrow_begin/end: the column ranges NOT covered by the wide (ACR / item-embedding) segments. */
  int32_t n_narrow;
  int32_t narrow_begin[4];
  int32_t narrow_end[4];
  uint8_t col_seg[NAR_MAX_COLS];
} nar_feature_plan;

/* Which rows a row list holds.  Rows [0, n_input) are clicked items (reference timestamp = event_timestamp[row_pos],
 * normalisation statistics group 0, nar_model.py:328); the others use max_ts (:343, :356) and are either
 *   n_cand > 0 : groups of n_cand rows per position, the positive first (group 1) then its negatives (group 2), or
 *   n_cand == 0: n_positive positive rows (group 1) followed by negative rows (group 2) - the base rows of the
 *                per-unique-id CAR layer 1 (nar_build_base_rows).
 * Rows >= n_full carry ITEM features only: their context columns (internal column >= ctx_col0) are written as 0 and
 * skipped by the backward pass.  n_full >= n_rows: every row is a full row.                                         */
typedef struct {
  int64_t n_rows, n_input, n_cand, n_positive, n_full, ctx_col0;
} nar_row_layout;

/* rows: row_pos[r] = flat index b*T+t of the position that owns row r (context features,
 * reference timestamp), row_item[r] = article id.                                           */
int nar_gather_features(nar_ctx* ctx, const nar_feature_plan* plan /*host*/,
                        const int32_t* row_pos, const int64_t* row_item, const nar_row_layout* rows /*host*/,
                        const int64_t* event_timestamp /*[B*T]*/, const int64_t* max_ts /*[1]*/,
                        float* out /*[n_rows,row_ld]*/, void* stream);

/* backward of the same: d_gamma += sum_r dX*raw, d_beta += sum_r dX, trainable embedding
 * grads += dX*gamma scattered by id (IndexedSlices scatter-add, nar_model.py:918/:741).     */
int nar_gather_features_bwd(nar_ctx* ctx, const nar_feature_plan* plan /*host*/,
                            const int32_t* row_pos, const int64_t* row_item, const nar_row_layout* rows /*host*/,
                            const int64_t* event_timestamp, const int64_t* max_ts,
                            const float* d_out /*[n_rows,row_ld]*/, float* d_gamma, float* d_beta, void* stream);

/* row lists of one step.  The L valid positions (pos_idx[l] = b*T+t, session-major) produce
 * n_rows = L + L*(1+K) rows: input rows [0,L) = clicked items (nar_model.py:328), then for each
 * position its candidates contiguously: positive label_next_item (:343) followed by its K
 * negatives (:356).                                                                        */
int nar_build_rows(const int32_t* pos_idx, int64_t L, const int64_t* item_clicked, const int64_t* label_next_item,
                   const int64_t* negatives /*[B*T,K]*/, int64_t K, int32_t* row_pos, int64_t* row_item, void* stream);

/* base rows of the per-unique-id CAR layer 1 (csrc/car.cu): n_base = 2L + U rows = the L clicked items, the L positives,
 * then one ITEM-ONLY row per entry of the step's unique-negative table (unique_items / n_unique as returned by
 * nar_sample_negatives_uidx; U = table capacity K*20 plus one trailing slot for the padding negative, id 0).         */
int nar_build_base_rows(const int32_t* pos_idx, int64_t L, const int64_t* item_clicked, const int64_t* label_next_item,
                        const int64_t* unique_items, const int32_t* n_unique /*[1] device*/, int64_t U,
                        const int32_t* neg_uidx, int64_t K, int32_t* base_pos /*[2L+U]*/, int64_t* base_item /*[2L+U]*/,
                        void* stream);

/* normalisation statistics of recency / novelty over the first n_norm nonzero buffer entries
 * (nar_model.py:1062-1089, :1150-1193, :1011-1039).  stats[g][8], g = 0 input / 1 positive /
 * 2 negative rows: {rec_mean, rec_std, rec_zmin, rec_zmax, nov_mean, nov_std, nov_zmin, nov_zmax};
 * all three groups are equal unless the buffer is empty (first batch), where each group
 * uses its own non-padded rows (the tf.cond at nar_model.py:1082 / :1179): pass the rows.    */
int nar_feature_stats(nar_ctx* ctx, const int64_t* buffer, int64_t buf_len, int64_t n_norm,
                      const int64_t* created_at_ts, const float* pop_norm, const int64_t* max_ts,
                      float log_base_recency, float log_base_novelty,
                      const int32_t* row_pos, const int64_t* row_item, int64_t n_rows, int64_t n_input,
                      int64_t n_cand, const int64_t* event_timestamp,
                      float* stats /*[24]*/, void* stream);

/* plain row gather / scatter-add used by the parity tests and the roofline micro-benchmark
 * (tf.nn.embedding_lookup nar_model.py:948 and its IndexedSlices gradient :918).           */
int nar_gather_rows_f32(const float* table, int64_t n_table_rows, int64_t ld, int width,
                        const int64_t* ids, int64_t n, float* out, int64_t ld_out, void* stream);
int nar_scatter_add_rows_f32(float* table, int64_t n_table_rows, int64_t ld, int width,
                             const int64_t* ids, int64_t n, const float* src, int64_t ld_src, void* stream);

/* ---- dense contraction (replaces every tf.layers.Dense nar_model.py:375-473 and the
 *      UGRNN input projection :1317 -> Eigen/MKL or cuBLAS sgemm in the reference).
 *      D[M,N] = epilogue( sum_k A(m,k) * B(n,k) ), TMA-fed wgmma (tf32 or bf16 operands), fp32
 *      accumulation in registers.  a_kmajor: A(m,k) = A[m*lda + k] else A[k*lda + m];
 *      b_kmajor: B(n,k) = B[n*ldb + k] else B[k*ldb + n].                                  */
typedef enum { NAR_ACT_NONE = 0, NAR_ACT_LEAKY_RELU = 1, NAR_ACT_TANH = 2 } nar_act;
/* session cell, nar_model_cfg.rnn_cell */
typedef enum { NAR_CELL_UGRNN = 0, NAR_CELL_GRU = 1, NAR_CELL_LSTM = 2 } nar_rnn_cell;

typedef struct {
  const float* bias;      /* [N] added before the activation, or NULL */
  int32_t act;            /* nar_act applied to acc+bias (any other value is rejected) */
  int32_t dact;           /* nar_act whose DERIVATIVE (evaluated from the forward OUTPUT aux) multiplies the result */
  const float* aux;       /* [M,N] forward output of the layer being differentiated (dact != NONE) */
  int64_t ld_aux;
  int32_t accumulate;     /* 1: D += result with atomics (required when split_k > 1) */
  int32_t split_k;        /* >=1; <= 0 with accumulate: chosen by the library.  Each split runs the epilogue on its own
                             partial sum, so split_k > 1 with bias or act is rejected, and the library's choice is 1 then */
  int32_t precision;      /* 1 = TF32, 3 = 3xTF32 (error-compensated, ~fp32 accuracy) */
  const float* b_lo;      /* precision 3 only, optional: x - tf32_trunc(x) of operand B, same shape / ld as B (see
                             nar_tf32_lo; the weights' lo plane is maintained by nar_adam_tf).  NULL: split B in-kernel */
  const void* b_bf16;     /* precision 4 (bf16x3: bf16 hi + lo pieces on the bf16 tensor path, fp32 accumulate; A fp32 of
                             either major): operand B as the pre-split transposed plane written by nar_pack_bf16x3 - [N, ld_bf16]
                             bf16, row n = per block of 32 k the 32 hi values then the 32 lo values; B / ldb are ignored */
  int64_t ld_bf16;        /* elements per row of b_bf16 (>= ceil(K/32)*64, multiple of 8) */
  const float* a_scale;   /* optional A scale, defined on A's storage: the stored element A[i*lda + j] enters the MMA as
                             A[i*lda + j] * a_scale[(i / a_scale_group)*ld_a_scale + j] (one fp32 multiply, rounded), so
                             a K-major A is scaled per (row group, k) and an MN-major A per (k group, m).  Implemented for
                             precision 4 and for precision 1 with both operands MN-major (the weight gradient); NULL: none */
  int64_t ld_a_scale;     /* multiple of 4, >= A's storage row length */
  int64_t a_scale_group;  /* >= 1 */
  const float* pred;      /* optional scorer-product backward epilogue (precision 1, K-major A and B, no split-K / bias /
                             act / accumulate / a_scale): with g = pred_group (1..128, M a multiple of g), row r of the result
                             v is the gradient of prod[r] = aux[r] * pred[r / g] (aux = the candidate rows, e.g. the CAR
                             output); D[r] = v[r] * pred[r/g] * dact'(aux[r]) and d_pred[l] = sum over the g rows of
                             position l, in row order, of v * aux (fmaf chain).  M tiles hold whole positions.  NULL: none */
  float* d_pred;
  int64_t ld_pred;        /* row stride of pred and d_pred (>= N) */
  int64_t pred_group;
  float* d_bias;          /* optional with pred: d_bias[c] += sum over the M rows of D[r, c] (the gradient of a bias added
                             before dact), float atomics into a buffer the caller owns; rejected without pred.  NULL: none */
  const float* car_pp;    /* optional CAR layer-1 backward epilogue (precision 1, or 3 without b_lo; K-major A and B, no split-K / bias / act /
                             accumulate / aux / a_scale / pred; D must be NULL; N a multiple of 4): row r of the result v is
                             the gradient of H1c[r] = dact(pre) for candidate j = r % (car_k+1) of position l = r / (car_k+1),
                             pre = j == 0 ? car_pp[l] : car_pc[l] + car_pi[u], u = car_neg_uidx[car_pos_idx[l]*car_k + j-1]
                             (the rows nar_car_combine writes).  With g = v * dact'(pre): car_dpp[l] = g of j == 0;
                             car_dpc[l] += sum of g over j >= 1 and car_dpi[u] += g, float atomics into buffers the caller
                             zeroes (car_dpc is bit-reproducible for car_k < 128, car_dpi is not).  All [rows, ld_car], 16-byte
                             aligned.  NULL: none */
  const float* car_pc;
  const float* car_pi;
  const int32_t* car_pos_idx;
  const int32_t* car_neg_uidx;
  float* car_dpp;
  float* car_dpc;
  float* car_dpi;
  int64_t ld_car;         /* row stride of the six car_ tensors (>= N, multiple of 4) */
  int64_t car_k;          /* negatives per position (K) */
} nar_gemm_epilogue;

/* bf16x3 weight planes for n matrices in one launch: W[i] [K[i], N[i]] fp32 (row stride ldw[i], i.e. stored [in, out]) ->
 * out[i] [N[i], ld_out[i]] bf16 as nar_gemm_epilogue.b_bf16 describes (zero padded to whole 32-k blocks).
 * descs_dev: caller-owned device scratch of >= 32*32 bytes the call keeps its table in.                               */
int nar_pack_bf16x3(const float* const* W /*host array*/, void* const* out /*host array*/, const int32_t* K, const int32_t* N,
                    const int32_t* ldw, const int32_t* ld_out, int n, void* descs_dev, void* stream);

int nar_gemm_tf32(nar_ctx* ctx, int64_t M, int64_t N, int64_t K,
                  const float* A, int64_t lda, int a_kmajor,
                  const float* B, int64_t ldb, int b_kmajor,
                  float* D, int64_t ldd, const nar_gemm_epilogue* epi /*host*/, void* stream);
/* the same product with D stored transposed: D[n*ldd + m].  For a weight gradient dW [in, out] += X^T dY computed as
 * dW^T = dY^T X: A = dY MN-major, B = X^T K-major (e.g. nar_car_combine_t's H1cT), so that both operands reach the
 * tensor cores without a transpose in shared memory.  precision 1, or 3 without b_lo; a_kmajor = 0, b_kmajor = 1; no bias /
 * act / dact / a_scale / pred / car_ epilogue; accumulate and split_k as for nar_gemm_tf32.                              */
int nar_gemm_tf32_dt(nar_ctx* ctx, int64_t M, int64_t N, int64_t K,
                     const float* A, int64_t lda, int a_kmajor,
                     const float* B, int64_t ldb, int b_kmajor,
                     float* D, int64_t ldd, const nar_gemm_epilogue* epi /*host*/, void* stream);

/* ---- session RNN (replaces tf.contrib.rnn.UGRNNCell in MultiRNNCell / dynamic_rnn,
 *      nar_model.py:1308-1342).  Rows are the valid positions only, grouped by session:
 *      session b owns rows [sess_off[b], sess_off[b+1]).  gx = x*Wx + b for all rows
 *      (nar_gemm_tf32), gate cols [0,Hp), candidate cols [Hp,2Hp).                          */
int nar_ugrnn_fwd(nar_ctx* ctx, const float* gx /*[L,2Hp]*/, const float* Wh /*[Hp,2Hp]*/,
                  const int32_t* sess_off /*[B+1]*/, int64_t B, int64_t Hp,
                  float* h_out /*[L,Hp]*/, float* gate /*[L,Hp]*/, float* cand /*[L,Hp]*/, void* stream);
int nar_ugrnn_bwd(nar_ctx* ctx, const float* d_hout /*[L,Hp]*/, const float* h_out, const float* gate,
                  const float* cand, const float* WhT /*[2Hp,Hp]*/, const int32_t* sess_off, int64_t B,
                  int64_t Hp, float* d_gx /*[L,2Hp]*/, float* h_prev /*[L,Hp]*/, void* stream);

/* GRU recurrence (tf.nn.rnn_cell.GRUCell; rnn_cell='gru'): gx [L,3Hp] = x*Wx + b with Wx [in,3Hp] (r | u | c pre-activations
 * of the input), Whg [Hp,2Hp], Whc [Hp,Hp]:  [r,u] = sigmoid(gx_ru + h*Whg) ; c = tanh(gx_c + (r*h)*Whc) ;
 * h' = u*h + (1-u)*c.  Outputs per row: state h_out, gates r / u, candidate c, rh = r * (state entering the step).      */
int nar_gru_fwd(nar_ctx* ctx, const float* gx, const float* Whg, const float* Whc, const int32_t* sess_off, int64_t B,
                int64_t Hp, float* h_out, float* r_out, float* u_out, float* c_out, float* rh_out, void* stream);
/* d_gx [L,3Hp] = dL/d(pre-activations); h_prev [L,Hp] = state entering the step (dWhg = h_prev^T d_gx[:, :2Hp],
 * dWhc = rh^T d_gx[:, 2Hp:]); WhgT [2Hp,Hp], WhcT [Hp,Hp] are the transposed recurrent blocks.                        */
int nar_gru_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* r_out, const float* u_out,
                const float* c_out, const float* WhgT, const float* WhcT, const int32_t* sess_off, int64_t B, int64_t Hp,
                float* d_gx, float* h_prev, void* stream);

/* LSTM recurrence (tf.nn.rnn_cell.LSTMCell(H, state_is_tuple=True), nar_model.py:1316; rnn_cell='lstm'; no peepholes, no
 * cell clip, no projection, forget_bias 1.0): gx [L,4Hp] = x*Wx + b (i | j | f | o pre-activations of the input),
 * Wh [Hp,4Hp]:  c' = sigmoid(f + h*Wh_f + 1) * c + sigmoid(i + h*Wh_i) * tanh(j + h*Wh_j) ; h' = sigmoid(o + h*Wh_o) * tanh(c').
 * gx is overwritten in place with the activated gates (sigmoid(i) | tanh(j) | sigmoid(f+1) | sigmoid(o)); per row: output
 * h_out = h', cell state c_out = c'.                                                                                       */
int nar_lstm_fwd(nar_ctx* ctx, float* gx, const float* Wh, const int32_t* sess_off, int64_t B, int64_t Hp, float* h_out,
                 float* c_out, void* stream);
/* act [L,4Hp] = the activated gates nar_lstm_fwd left in gx; d_gx [L,4Hp] = dL/d(pre-activations); h_prev [L,Hp] = h entering
 * the step (dWh = h_prev^T d_gx); WhT [4Hp,Hp] is the transposed recurrent block.                                          */
int nar_lstm_bwd(nar_ctx* ctx, const float* d_hout, const float* h_out, const float* c_out, const float* act, const float* WhT,
                 const int32_t* sess_off, int64_t B, int64_t Hp, float* d_gx, float* h_prev, void* stream);

/* ---- negative sampler (replaces nar_model.py:1220-1304: tf.random_shuffle x(2+clicks),
 *      tf.unique, unsorted_segment_min, tf.setdiff1d inside nested tf.map_fn).  RNG spec:
 *      oracle/sampler_ref.py.  all_items_global [Bg,T1] builds the pool; negatives are
 *      produced for local sessions [sess0, sess0+B).  out [B,T1-1,K] int64, zero padded.
 *      buf_len < 0 or n_from_buffer < 0: NAR_ERR_INVALID; K*20 > 16384: NAR_ERR_UNSUPPORTED. */
int nar_sample_negatives_workspace(int64_t Bg, int64_t T1, int64_t buf_len, int64_t K, int64_t* bytes /*host*/);
int nar_sample_negatives(nar_ctx* ctx, const int64_t* all_items_global, int64_t Bg, int64_t T1,
                         int64_t sess0, int64_t B, const int64_t* buffer, int64_t buf_len,
                         int64_t K, int64_t n_from_buffer, uint64_t seed, uint32_t step,
                         int64_t* out, void* workspace, int64_t workspace_bytes, void* stream);

/* the same, additionally returning for every negative its index in the pool's sorted unique-item table
 * (out_uidx [B,T1-1,K] int32; K*20 = the padding slot for an id-0 negative) and device pointers to that table /
 * its length inside `workspace` (valid until the next call with the same workspace).                              */
int nar_sample_negatives_uidx(nar_ctx* ctx, const int64_t* all_items_global, int64_t Bg, int64_t T1,
                              int64_t sess0, int64_t B, const int64_t* buffer, int64_t buf_len,
                              int64_t K, int64_t n_from_buffer, uint64_t seed, uint32_t step,
                              int64_t* out, int32_t* out_uidx /*or NULL*/, const int64_t** unique_items /*host, out*/,
                              const int32_t** n_unique /*host, out*/, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- per-unique-id CAR layer 1 (nar_model.py:343-405; see csrc/car.cu): pre-activation of candidate (l, j) =
 *      j == 0 ? PP[l] : PC[l] + PI[neg_uidx[pos_idx[l], j-1]]; H1c [L*(1+K), C] = act(pre).                        */
int nar_car_combine(const float* PP /*[L,C]*/, const float* PC /*[L,C]*/, const float* PI /*[U,C]*/,
                    const int32_t* pos_idx, const int32_t* neg_uidx, int64_t L, int64_t K, int64_t C, int act,
                    float* H1c, void* stream);
/* the same rows stored transposed: H1cT [C, ldr] with H1cT[c*ldr + r] = H1c[r*C + c], r < L*(1+K) <= ldr, ldr a multiple
 * of 4 (columns r >= L*(1+K) are not written); bit-identical values                                                      */
int nar_car_combine_t(const float* PP, const float* PC, const float* PI, const int32_t* pos_idx, const int32_t* neg_uidx,
                      int64_t L, int64_t K, int64_t C, int act, float* H1cT, int64_t ldr, void* stream);
/* (its backward is the layer-2 dgrad's epilogue: nar_gemm_epilogue.car_pp)                                          */

/* ---- scorer + loss (replaces tf.multiply + matching_dense_layer_1..4 :478-500, softmax
 *      :515, log :660, masked mean :664).                                                  */
/* prod[r,:] = cand[r,:] * pred[r / n_cand,:]   (tf.multiply nar_model.py:478,:493)          */
int nar_mul_pred(const float* cand, const float* pred, int64_t n_pos, int64_t n_cand, int64_t C,
                 float* prod, void* stream);
/* d_cand = d_prod*pred*act'(cand) ; d_pred[l] = sum_j d_prod[l,j]*cand[l,j].  cand_act (nar_act): the
 * activation that produced cand (the CAR tanh) is differentiated in the same pass; NAR_ACT_NONE = plain product rule */
int nar_mul_pred_bwd(const float* d_prod, const float* cand, const float* pred, int64_t n_pos, int64_t n_cand,
                     int64_t C, int cand_act, float* d_cand, float* d_pred, void* stream);
/* last Dense(32->1) + /temperature + log-softmax over the 1+K candidates + masked mean CE,
 * forward and backward in one pass.  z3 [n_pos*n_cand, ld_z] ; logits [n_pos,n_cand] ;
 * loss_sum += sum_l -(logp[l,0]) * inv_count ; d_z3 = d(loss)/d(z3) (before leaky');
 * d_m4[k] += ..., d_c4 += ...                                                              */
/* optional novelty regulariser (nar_model.py:517, :531-544, :673-683): total_loss -= factor * mean over the valid
 * positions of sum_k q_k * nov_k, q = softmax over the NEGATIVES only of the scaled scores, nov_k =
 * -log_base(pop_norm[id_k]); its value is added to loss_nov[0] and its gradient to the negatives' score gradients */
typedef struct {
  float factor;               /* novelty_reg_factor; <= 0: off */
  float log_base;             /* popularity_smooth_log_base */
  const float* pop_norm;      /* [num_items] articles_recent_pop_norm */
  const int64_t* cand_ids;    /* [n_pos*n_cand] candidate ids, positive first */
  float* loss_nov;            /* [1] */
} nar_novelty_reg;

int nar_score_softmax_ce(const float* z3, int64_t ld_z, int64_t width, const float* m4, int64_t ld_m4,
                         const float* c4, int64_t n_pos, int64_t n_cand, float inv_temperature,
                         float inv_count, float* logits, float* loss_sum, float* d_z3,
                         float* d_m4, float* d_c4, const nar_novelty_reg* nov /*host, or NULL*/, void* stream);
/* cosine mode (north_star wording; nar_model.py:437 commented l2-normalise): logits =
 * <l2n(pred), l2n(cand)>/temperature fused with the same softmax-CE; writes d_cand, d_pred. */
int nar_cosine_softmax_ce(const float* cand, const float* pred, int64_t n_pos, int64_t n_cand, int64_t C,
                          float inv_temperature, float inv_count, float* logits, float* loss_sum,
                          float* d_cand, float* d_pred, const nar_novelty_reg* nov /*host, or NULL*/, void* stream);

/* ---- evaluation ranking (ModeKeys.EVAL: rank_items_by_predicted_prob nar_model.py:777-795 = tf.nn.top_k over all
 *      1+K candidates, sparse_recall_at_top_k :835-840, define_mrr_metric :862-885).  logits [n_pos,n_cand] as written
 *      by the two *_softmax_ce kernels (already / temperature); cand_ids [n_pos*n_cand]: per position the positive
 *      followed by its negatives.  pred_ids / pred_probs [n_pos,n_cand] (either may be NULL): candidates sorted by
 *      softmax probability, descending, ties to the lower candidate index (top_k order).  metrics[0] += number of
 *      positions whose positive is in the top_n, metrics[1] += sum of 1/rank for those, metrics[2] += n_pos.       */
int nar_rank_candidates(const float* logits, const int64_t* cand_ids, int64_t n_pos, int64_t n_cand, int32_t top_n,
                        int64_t* pred_ids, float* pred_probs, double* metrics /*[3] float64*/, void* stream);

/* ---- recommendation (NarEngine.recommend; csrc/recommend.cu).  A candidate is scored for a query position exactly like
 *      a sampled negative of that position (nar_model.py:356-364, :374-405, :444-515).                               */
/* CAR layer 1 of a grid of (query, candidate) pairs: H1 [Q*Nc, C], row q*Nc + j = act(PC[q] + PI[j]) (PC [Q,C] context
 * halves + bias, PI [Nc,C] item halves; all 16-byte aligned).                                                        */
int nar_car_combine_grid(const float* PC, const float* PI, int64_t Q, int64_t Nc, int64_t C, int act, float* H1, void* stream);
/* per query row of logits [Q,N] (already / temperature): the top_n (1..min(N, 4096)) largest, by descending score, ties to
 * the lower candidate index (tf.nn.top_k order).  cand_ids [N] distinct.  item_clicked [*, T] or NULL: when given, query q
 * at flat position q_pos[q] = b*T+t never returns item_clicked[b*T + 0..t] (T <= 1024).  out_ids / out_scores / out_probs
 * [Q,top_n] (scores / probs may be NULL); probs = softmax over the non-excluded candidates.  A query with fewer than top_n
 * non-excluded candidates gets id 0, score -inf, prob 0 in the remaining slots.                                          */
int nar_topn_candidates(const float* logits, const int64_t* cand_ids, int64_t Q, int64_t N, int32_t top_n,
                        const int64_t* item_clicked, const int32_t* q_pos, int64_t T, int64_t* out_ids, float* out_scores,
                        float* out_probs, void* stream);
/* per query row of logits [Q,N] (unsampled evaluation, DESIGN.md section 13): query q at flat position q_pos[q] = b*T+t
 * has the label label_next[b*T+t]; cand_ids [N] strictly ascending (N < 2^31).  Its competitors are the candidates other
 * than the label that are not in the session's row all_items[b*(T+1) + 0..T] (T + 1 <= 1024, else NAR_ERR_UNSUPPORTED).
 * rank[q] = number of competitors whose score orders above the label's (the order of nar_topn_candidates: -0 == +0, NaN
 * above +inf; ties go to the label), or -1 when the label is 0 or not a candidate (such a query is not counted).
 * hist [top_n + 2] int64 (accumulated): [r] += 1 for rank r < top_n, [top_n] += 1 per ranked query, [top_n + 1] += its
 * number of competitors.                                                                                               */
int nar_rank_labels(const float* logits, const int64_t* cand_ids, int64_t Q, int64_t N, const int64_t* label_next,
                    const int64_t* all_items, const int32_t* q_pos, int64_t T, int32_t top_n, int32_t* rank, int64_t* hist,
                    void* stream);

/* ---- host state (CPU, no CUDA): ClickedItemsState.update_items_state (clicked_items_state.py:187-250) in one pass.
 *      buffer [cap,2] int64 {item, timestamp} newest first, zero padded (in/out); batch_items / batch_ts: the step's
 *      non-padded clicks in batch order (nar_model.py:1635-1646); hours_ms = recent_clicks_buffer_hours * 3.6e6;
 *      scratch [cap,2]; recent_pop [V] (out), pop_norm [V] float64 (out) = max(pop / (sum(pop) + 1), min_norm_pop);
 *      articles_pop [V] (in/out, += bincount(batch)).                                                           */
int nar_host_state_update(int64_t* buffer, int64_t cap, const int64_t* batch_items, const int64_t* batch_ts,
                          int64_t n_batch, int64_t hours_ms, int64_t* scratch, int64_t* recent_pop,
                          double* pop_norm, int64_t* articles_pop, int64_t num_items, double min_norm_pop);
/* the same, straight from the padded batch (ItemsStateUpdaterHook.after_run nar_model.py:1635-1646): item_clicked /
 * event_ts [B,T], label_last [B]; batch_scratch [2*B*(T+1)] int64                                                */
int nar_host_state_update_batch(int64_t* buffer, int64_t cap, const int64_t* item_clicked, const int64_t* event_ts,
                                const int64_t* label_last, int64_t B, int64_t T, int64_t hours_ms,
                                int64_t* batch_scratch, int64_t* scratch, int64_t* recent_pop, double* pop_norm,
                                int64_t* articles_pop, int64_t num_items, double min_norm_pop);

/* ---- device-resident ClickedItemsState (same update as above, in HBM; what Estimator.train advances every step).
 *      old_items / old_ts [cap] -> new_items / new_ts [cap] (distinct buffers: ping-pong); all_items [Bg,T+1] =
 *      [item_clicked | label_last_item], event_ts [Bg,T]; recent_pop [V] int64 scratch / output; pop_norm [V] float32
 *      (what the graph reads), pop_norm64 [V] float64 or NULL; articles_pop [V] in/out; err[0] = 1 on an id outside
 *      [0, V).  A batch without clicks leaves new_* untouched: the caller keeps using old_*.                        */
int nar_state_update(const int64_t* old_items, const int64_t* old_ts, int64_t cap, const int64_t* all_items,
                     const int64_t* event_ts, int64_t Bg, int64_t T, int64_t hours_ms, int64_t* new_items,
                     int64_t* new_ts, int64_t* recent_pop, float* pop_norm, double* pop_norm64, int64_t* articles_pop,
                     int64_t num_items, double min_norm_pop, int* err, void* stream);

/* ---- dropout (replaces tf.layers.dropout nar_model.py:338-340 / :351-353 / :367-369 / :417-419 and
 *      DropoutWrapper(output_keep_prob) :1330-1333).  dst[r,c] = src[r,c] * keep(r,c) / keep_prob; the masks come from
 *      the counter-based generator specified in oracle/dropout_ref.py (Philox4x32-10 keyed by seed, counter = column
 *      block, row key, tensor id, step) so that forward, backward and the oracle draw the same bits.
 *      tensor_id > 0: every row belongs to that tensor, row key = row_pos[r] (flat position b*T+t).
 *      tensor_id == 0: feature rows in the n_cand > 0 layout of nar_row_layout: rows [0,n_input) tensor 1 (key =
 *      position), then per position the positive (tensor 2, key = position) and K negatives (tensor 3, key =
 *      position*K + k).  In place (dst == src) is allowed.  cols and ld multiples of 4, src and dst 16-byte aligned
 *      (float4 accesses; checked even when there is nothing to do): NAR_ERR_INVALID otherwise.                      */
int nar_dropout_rows(const float* src, float* dst, int64_t rows, int64_t cols, int64_t ld, const int32_t* row_pos,
                     int64_t n_input, int64_t n_cand, int64_t K, int tensor_id, float keep_prob, uint64_t seed,
                     uint32_t step, void* stream);

/* ---- small helpers ------------------------------------------------------------------ */
/* out[c] += sum_r x[r,c]   (bias gradients)                                                */
int nar_colsum_add(const float* x, int64_t rows, int64_t cols, int64_t ld, float* out, void* stream);
/* y = x * act'(aux) elementwise                                                            */
int nar_act_bwd(const float* dy, const float* y, int64_t n, int act, float* dx, void* stream);
/* out[0] += scale * sum(x^2) / 2  (l2_regularizer, nar_model.py:655)                       */
int nar_l2_loss_add(const float* x, int64_t n, float scale, float* out, void* stream);
int nar_transpose_f32(const float* src, int64_t rows, int64_t cols, int64_t ld_src, float* dst, int64_t ld_dst, void* stream);
/* out[r, c] = h[r, c] + res[r, c] over rows x cols, all three with leading dimension ld (the residual session stack's
 * layer output: the cell's h plus the layer input).  cols and ld multiples of 4, ld >= cols, h, res and out 16-byte
 * aligned (float4 accesses; checked even when rows or cols is 0): NAR_ERR_INVALID otherwise.
 * out may be h or res.                                                                                                */
int nar_residual_add(const float* h, const float* res, int64_t rows, int64_t cols, int64_t ld, float* out, void* stream);

/* ---- optimiser (replaces tf.train.AdamOptimizer(lr,.9,.999,1e-8) nar_model.py:708-722;
 *      TF form: lr_t = lr*sqrt(1-b2^t)/(1-b1^t); w -= lr_t*m/(sqrt(v)+eps); the gradient of
 *      elements [0,reg_end) gets + reg_l2*w (l2_regularizer); grad is scaled by grad_scale
 *      first (1/world after a sum-allreduce is NOT needed: losses are already global means) */
int nar_adam_tf(float* params, const float* grads, float* m, float* v, int64_t n, int64_t reg_end,
                float reg_l2, float lr, float beta1, float beta2, float eps, int64_t step,
                float* params_lo /* optional [n]: receives w - tf32_trunc(w) of the updated weights */, void* stream);
/* lo[i] = x[i] - tf32_trunc(x[i])  (the second operand plane of the 3xTF32 GEMM)          */
int nar_tf32_lo(const float* x, int64_t n, float* lo, void* stream);

/* =====================================================================================================
 * The whole step behind ONE call (replaces the single session.run(train_op) of nar_trainer_gcom.py:515-517 /
 * MonitoredTrainingSession: sampler -> features -> CAR -> RNN -> FC -> scorer -> loss -> backward -> Adam,
 * nar_model.py:102-728).  The engine sequences every kernel of the step from C: the caller stages the batch in
 * HBM, fills a nar_step_io and makes one call per phase; no per-kernel host round trip is left.
 *   nar_engine_prepare  the weight-independent front of a step (negatives, row lists, normalisation statistics,
 *                       base rows): may run one step ahead on a side stream
 *   nar_engine_step     forward (+ backward when io->train): gradients complete in cfg.grads on return-stream order
 *   nar_engine_apply    TF-Adam over the flat parameter buffer (after the data-parallel gradient exchange, if any)
 * Internally the step forks weight / bias gradients onto an engine-owned auxiliary stream (events, no host sync).
 * ===================================================================================================== */
#define NAR_MAX_LAYERS 4

typedef struct {
  /* dimensions */
  int64_t num_items, C /*CAR_embedding_size*/, Hp /*rnn_units padded to 4*/, Fp /*feature row width*/, ctx_col0;
  int32_t layers, rnn_cell /*nar_rnn_cell: UGRNNCell (nar_model.py:1318), GRUCell (:1315), LSTMCell (:1316)*/, ranking /*0 = MLP scorer (:444-500), 1 = cosine*/;
  int32_t fwd_precision, bwd_precision;       /* nar_gemm_epilogue.precision of the forward (3 or 4) / backward (1 or 3) GEMMs */
  int32_t dedup;                              /* 1: per-unique-id CAR layer 1 (csrc/car.cu); 0: every candidate row materialised */
  int32_t use_aux_stream;                     /* 1: weight / bias gradients (and the forward session branch) on the auxiliary stream */
  float keep_prob;                            /* dropout_keep_prob (training steps only; < 1 needs dedup == 0) */
  float novelty_reg_factor;                   /* nar_model.py:673-683; 0 = off */
  uint64_t dropout_seed;
  /* hyper-parameters */
  int64_t K /*negatives per click*/, n_from_buffer, buf_len, n_norm;
  float inv_temperature, reg_l2, lr, beta1, beta2, eps;
  uint64_t sampler_seed;
  int32_t world, rank;                        /* data parallel: rank 0 adds the regulariser term to the loss */
  /* flat parameter buffers: params / params_lo / grads / adam_m / adam_v share offsets (floats) */
  float *params, *params_lo, *grads, *adam_m, *adam_v;
  int64_t n_params, reg_end;
  int64_t off_W1, off_b1, off_W2, off_b2, off_W3, off_b3, off_W4, off_b4, off_gamma, off_beta;
  int64_t off_M[4], off_c[4], ld_M[4];        /* matching_dense_layer_1..4 kernels / biases, leading dimensions */
  /* per layer: Wx [in, G*Hp] and b [G*Hp], G gate blocks: UGRNN (gate | candidate), GRU (r | u | candidate), LSTM (i | j | f | o);
   * Wh [Hp, G*Hp], except the GRU's Wh [Hp, 2Hp] (r | u) and Whc [Hp, Hp] (candidate: a product with r*h) */
  int64_t off_Wx[NAR_MAX_LAYERS], off_Wh[NAR_MAX_LAYERS], off_rb[NAR_MAX_LAYERS], off_Whc[NAR_MAX_LAYERS];
  /* residual session stack (build_rnn(residual_connections=True), nar_model.py:1319-1323): layer 0 reads the projection
   * P = E*Wp + bp (Wp [C, Hp], bp [Hp]) and outputs cell(P) + P, layer i > 0 outputs cell(x) + x; 0 = plain stack */
  int32_t rnn_residual;
  int64_t off_Wp, off_bp;
  /* feature plan: static part (segments, tables, metadata, created_at_ts, gamma / beta, column map) */
  nar_feature_plan plan;
} nar_model_cfg;

typedef struct {
  int64_t B /*local sessions*/, Bg /*global sessions*/, T, sess0 /*first local session*/, L /*local valid positions*/,
          L_global /*sum(mask) over the global batch: the loss normaliser*/;
  int64_t L_cap;                  /* positions the workspace was sized for (>= L) */
  int64_t global_step;            /* optimiser steps applied so far; this step is number global_step + 1 */
  uint32_t sampler_step;          /* counter of the negative sampler (training: global_step + 1) */
  int32_t train;                  /* 1: forward + backward, 0: forward + loss only */
  /* staged inputs (device) */
  const int64_t *all_items /*[Bg,T+1] item_clicked | label_last_item*/, *event_ts /*[Bg,T]*/, *item_clicked /*[Bg,T]*/,
                *label_next /*[Bg,T]*/, *buffer /*[buf_len]*/, *max_ts /*[1]*/;
  const float* pop_norm;          /* [num_items] */
  const int64_t* ctx_int[NAR_MAX_SRC];
  const float* ctx_float[NAR_MAX_SRC];
  const int32_t *pos_idx /*[L] flat b*T+t of the valid positions, session-major*/, *sess_off /*[B+1]*/;
  /* buffers */
  void* prep_ws;  int64_t prep_ws_bytes;      /* results of nar_engine_prepare (one slot per step in flight) */
  void* ws;       int64_t ws_bytes;           /* activations / activation gradients of the step */
  float* loss;                                /* [4] device: {cross-entropy (mean over L_global), l2 regulariser, -, -} */
  /* optional [24] device, read by nar_engine_recommend / nar_engine_rank_labels (steps ignore it): the call's
   * feature-normalisation statistics, computed by the caller; NULL: computed from the call's rows.  With an empty
   * recent-clicks buffer the statistics of the clicked rows are taken over those rows, so a data-parallel rank passes
   * the statistics of the global batch's rows here */
  const float* stats;
} nar_step_io;

typedef struct nar_engine nar_engine;

int nar_engine_create(nar_ctx* ctx, const nar_model_cfg* cfg /*host*/, nar_engine** out);
int nar_engine_destroy(nar_engine* eng);
/* cfg fields that may change between steps without re-creating the engine (lr, precisions, stream use, world / rank) */
int nar_engine_update_cfg(nar_engine* eng, const nar_model_cfg* cfg /*host*/);
/* bytes of nar_step_io.prep_ws / .ws for a global batch of Bg x T, B local sessions, room for L_cap valid positions */
int nar_engine_workspace_bytes(const nar_engine* eng, int64_t Bg, int64_t B, int64_t T, int64_t L_cap, int32_t train,
                               int64_t* prep_bytes /*host*/, int64_t* ws_bytes /*host*/);
int nar_engine_prepare(nar_engine* eng, const nar_step_io* io /*host*/, void* stream);
int nar_engine_step(nar_engine* eng, const nar_step_io* io /*host*/, void* stream);
int nar_engine_apply(nar_engine* eng, const nar_step_io* io /*host*/, void* stream);
/* after the caller wrote the weights itself (initialisation, checkpoint restore): rebuild what the engine derives from
 * them (the bf16x3 planes of the forward weights, fwd_precision 4)                                                      */
int nar_engine_refresh(nar_engine* eng, void* stream);
/* device address / shape of a named intermediate of the LAST nar_engine_prepare / nar_engine_step with this io
 * (parity tests, evaluation ranking): "neg", "neg_uidx", "row_pos", "row_item", "stats", "X", "H1", "E", "HO<i>", "F1",
 * "PR", "logits", "base_pos", "base_item", ...  Returns NAR_ERR_INVALID for an unknown name.                       */
int nar_engine_buffer(const nar_engine* eng, const nar_step_io* io /*host*/, const char* name, void** ptr /*host*/,
                      int64_t* rows /*host*/, int64_t* ld /*host*/);
/* Recommendation (forward only; reads the weights, writes nothing but the workspace and the outputs).  io: a staged batch
 * as for a step with train = 0 (labels unused), L valid positions, io->ws / ws_bytes = the workspace; prep_ws unused.
 * Q queries: q_rows [Q] int64 = the local row l (index into pos_idx) of each query, or NULL for every row (Q = L);
 * q_pos [Q] int32 = its flat position b*T+t.  cand_ids [N] distinct ids in [1, V).  Per query block of q_block queries:
 * every candidate chunk of n_block candidates through CAR layer 1 (PC + PI, nar_car_combine_grid), layer 2, the scorer
 * into logits [q_block, N], then nar_topn_candidates (exclusion of the session's own clicks when exclude_session_clicks).
 * Forward GEMMs follow cfg.fwd_precision without split-K: the outputs do not depend on the block sizes.
 * nar_engine_recommend_workspace_bytes picks the largest blocks whose workspace fits budget_bytes (gather_q: q_rows != NULL). */
int nar_engine_recommend_workspace_bytes(const nar_engine* eng, int64_t L, int64_t Q, int64_t N, int32_t gather_q,
                                         int64_t budget_bytes, int64_t* ws_bytes /*host*/, int64_t* q_block /*host*/,
                                         int64_t* n_block /*host*/);
int nar_engine_recommend(nar_engine* eng, const nar_step_io* io /*host*/, const int64_t* q_rows, const int32_t* q_pos, int64_t Q,
                         const int64_t* cand_ids, int64_t N, int32_t top_n, int32_t exclude_session_clicks, int64_t q_block,
                         int64_t n_block, int64_t* out_ids, float* out_scores, float* out_probs, void* stream);
/* Unsampled evaluation of a staged EVAL batch (same io and workspace as nar_engine_recommend with Q = L, q_rows = NULL):
 * every valid position is a query, scored against cand_ids [N] (strictly ascending ids in [1, V)) block by block as
 * nar_engine_recommend scores it, each logits block finished by nar_rank_labels with the batch's label_next, all_items
 * and pos_idx.  rank [L] int32, hist [top_n + 2] int64 as there.  NAR_ERR_UNSUPPORTED for T + 1 > 1024.              */
int nar_engine_rank_labels(nar_engine* eng, const nar_step_io* io /*host*/, const int64_t* cand_ids, int64_t N, int32_t top_n,
                           int64_t q_block, int64_t n_block, int32_t* rank, int64_t* hist, void* stream);
/* kernels launched by this engine so far */
int64_t nar_engine_launch_count(const nar_engine* eng);

/* ---- baseline recommenders of the evaluation hook (csrc/baselines.cu, spec oracle/baselines_ref.py) ----------------
 * Pair table: cap (a power of two) slots of keys [cap] ((a << 32) | c, -1 empty), cooc [cap] (sessions with a and c at
 * two different positions), sr_w [cap] (sequential-rules weight in units of 1 / lcm(1..max_clicks_dist)), sr_first [cap]
 * (min (batch_seq << 32) | ordinal of the rule's occurrences, INT64_MAX when none); count [1] = occupied slots.
 * nar_baselines_clear empties a table; nar_baselines_rehash clears the new table and moves every entry into it.
 * nar_baselines_update folds one batch: all_items [Bg, T1] = item_clicked | label_last_item (0 = padding); *err = 1 for
 * an id outside [0, num_items), 2 when the table is full (the caller sizes it: at most sum len*(len-1) new entries).  */
int nar_baselines_clear(int64_t* keys, int64_t* cooc, int64_t* sr_w, int64_t* sr_first, int64_t cap, void* stream);
int nar_baselines_rehash(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w, const int64_t* sr_first, int64_t cap,
                         int64_t* new_keys, int64_t* new_cooc, int64_t* new_sr_w, int64_t* new_sr_first, int64_t new_cap,
                         int* err, void* stream);
int nar_baselines_update(int64_t* keys, int64_t* cooc, int64_t* sr_w, int64_t* sr_first, int64_t cap, int64_t* count,
                         const int64_t* all_items, int64_t Bg, int64_t T1, int64_t num_items, int32_t max_clicks_dist,
                         int64_t batch_seq, int* err, void* stream);
/* count [num_items] / first [num_items] int32: occurrences and first index of every nonzero id of buffer [n] */
int nar_baselines_buffer_hist(const int64_t* buffer, int64_t n, int64_t num_items, int32_t* count, int32_t* first, int* err,
                              void* stream);
/* norms [V] fp64: Euclidean norm of every row of acr [V, ld] (first dim columns) */
int nar_baselines_row_norms(const float* acr, int64_t V, int64_t dim, int64_t ld, double* norms, void* stream);
/* Scores, ranks and measures the enabled baselines (bit b of enabled: 0 pop_recent, 1 coocurrent, 2 item_knn, 3 cb, 4 sr)
 * for every query (b, t) with label_next != 0, over the candidates label + negatives [B, T, K] (first occurrence of an id
 * only).  metrics [5, 3] fp64 += {hits, sum of reciprocal ranks, queries} per baseline (rank_hist [5, top_n + 1] int64 is
 * scratch); out_ids [5, B*T, top_n] (optional) = each query's top-n ids, 0-padded.                                    */
int nar_baselines_score(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w, const int64_t* sr_first, int64_t cap,
                        const int64_t* item_clicked, const int64_t* label_next, const int64_t* negatives, int64_t B,
                        int64_t T, int64_t K, const int32_t* buf_count, const int32_t* buf_first,
                        const int64_t* articles_pop, const float* acr, int64_t acr_dim, int64_t acr_ld,
                        const double* acr_norm, int64_t num_items, double knn_lambda, double knn_alpha, int32_t enabled,
                        int32_t top_n, int64_t* rank_hist, double* metrics, int64_t* out_ids, int* err, void* stream);
/* Unsampled ranking (DESIGN.md section 14) of the enabled baselines of nar_baselines_score (same tables, buffer
 * histogram, popularity and ACR inputs): every query (b, t) with label_next != 0 ranks its label against the pool [N]
 * (distinct ids in [1, num_items)) minus the label and the ids of its session row all_items[b*(T+1) + 0..T]
 * (T + 1 <= 1024, else NAR_ERR_UNSUPPORTED), each id scored as nar_baselines_score scores a candidate.  rank = the
 * admissible competitors before the label in the baseline's order, 0x7fffffff when the baseline does not admit the label.
 * hist [5, top_n + 2] int64 (accumulated): per baseline [r] += 1 for rank r < top_n, [top_n] += 1 per query,
 * [top_n + 1] += its competitor count.  rank [5, B*T] int32 (optional; -1 where no query).  max_blocks > 0 caps the
 * grid (one CTA per query otherwise).  One launch.                                                                   */
int nar_baselines_rank_unsampled(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w, const int64_t* sr_first,
                                 int64_t cap, const int64_t* item_clicked, const int64_t* label_next,
                                 const int64_t* all_items, int64_t B, int64_t T, const int64_t* pool, int64_t N,
                                 const int32_t* buf_count, const int32_t* buf_first, const int64_t* articles_pop,
                                 const float* acr, int64_t acr_dim, int64_t acr_ld, const double* acr_norm,
                                 int64_t num_items, double knn_lambda, double knn_alpha, int32_t enabled, int32_t top_n,
                                 int64_t max_blocks, int32_t* rank, int64_t* hist, int* err, void* stream);
/* Recommendations of one table baseline (DESIGN.md section 16): for every query q < Q at flat position q_pos[q] = b*T + t
 * of item_clicked [B, T] (T <= 1024), the first top_n ids of cand [N] (distinct ids in [1, num_items)) in the order of
 * baseline (0 pop_recent, 1 coocurrent, 2 item_knn, 3 cb, 4 sr; inputs as in nar_baselines_score) among the admissible
 * ones, without item_clicked[b*T + 0..t] when exclude != 0.  out_ids [Q, top_n] int64 and out_scores [Q, top_n] float64
 * (the baseline's own score), then id 0 and NaN when fewer ids are admissible.  1 <= top_n <= 1024, else
 * NAR_ERR_UNSUPPORTED above.  max_blocks > 0 caps the grid (one CTA per query otherwise).  Any grid gives the same
 * bits.  *err = 1 for an id outside [1, num_items), 3 when cand is not strictly ascending.  One launch.          */
int nar_baselines_recommend(const int64_t* keys, const int64_t* cooc, const int64_t* sr_w, const int64_t* sr_first,
                            int64_t cap, const int64_t* item_clicked, int64_t B, int64_t T, const int32_t* q_pos, int64_t Q,
                            const int64_t* cand, int64_t N, int32_t exclude, const int32_t* buf_count,
                            const int32_t* buf_first, const int64_t* articles_pop, const float* acr, int64_t acr_dim,
                            int64_t acr_ld, const double* acr_norm, int64_t num_items, double knn_lambda, double knn_alpha,
                            int32_t baseline, int32_t top_n, int64_t max_blocks, int64_t* out_ids, double* out_scores,
                            int* err, void* stream);

/* ---- session-based kNN baseline, V-SkNN / SkNN (csrc/sknn.cu, spec oracle/sknn_ref.py) -------------------------------
 * Ring of S slots (logical index i at slot (head + i) % S, count entries, oldest first; head and count are the caller's):
 * ids [S] session id, lens [S], items [S, W] int32 sorted item set, +x while (x, id) is in the item -> sessions map and
 * -x once an eviction discarded it.  nar_sknn_update appends one batch (all_items [B, T1], 0 = padding; session_ids [B]),
 * then evicts the max(0, count + B - S) oldest entries; st_* [S] / [S, W] are staging scratch.  Requires B <= S,
 * T1 <= W <= 128.  Afterwards head += evicted (mod S), count += B - evicted.  *err = 1 for an id outside [0, num_items). */
int nar_sknn_update(int64_t* ids, int32_t* lens, int32_t* items, int64_t S, int64_t W, int64_t head, int64_t count,
                    int64_t* st_ids, int32_t* st_lens, int32_t* st_items, const int64_t* all_items,
                    const int64_t* session_ids, int64_t B, int64_t T1, int64_t num_items, int* err, void* stream);
/* Ranks label + negatives [B, T, K] of every query (b, t) with label_next != 0 by the kNN item scores of the active
 * session item_clicked[b, :t+1] (sample_size 0 = no 'recent' cut; decay_div 1 = 'div', 0 = 'same'; jaccard 1 = jaccard,
 * 0 = cosine).  metrics [3] fp64 += {hits, sum of reciprocal ranks, queries} (rank_hist [top_n + 1] int64 is scratch);
 * out_ids [B*T, top_n] (optional) = the top-n ids of each query, 0-padded.  NAR_ERR_UNSUPPORTED for S > 4096, T > 64
 * or K + 1 > 1024.                                                                                                     */
int nar_sknn_score(const int64_t* ids, const int32_t* lens, const int32_t* items, int64_t S, int64_t W, int64_t head,
                   int64_t count, const int64_t* item_clicked, const int64_t* label_next, const int64_t* negatives,
                   int64_t B, int64_t T, int64_t K, int64_t num_items, int64_t sample_size, int64_t nn, int32_t decay_div,
                   int32_t jaccard, int32_t top_n, int64_t* rank_hist, double* metrics, int64_t* out_ids, int* err,
                   void* stream);
/* Unsampled ranking (DESIGN.md section 14) with the neighbours of nar_sknn_score: every query (b, t) with label_next != 0
 * ranks its label against the pool [N] (ascending distinct ids in [1, num_items)) minus the label and the ids of its
 * session row all_items[b*(T+1) + 0..T], by (item score desc, first neighbour asc, id asc) over the ids some kept
 * neighbour holds.  rank [B*T] int32 (optional): the competitors before the label, 0x7fffffff when no kept neighbour
 * holds it, -1 where no query.  hist [top_n + 2] int64 accumulated as in nar_baselines_rank_unsampled.  max_blocks > 0
 * caps the grid.  NAR_ERR_UNSUPPORTED for S > 4096 or T > 64.                                                        */
int nar_sknn_rank_unsampled(const int64_t* ids, const int32_t* lens, const int32_t* items, int64_t S, int64_t W, int64_t head,
                            int64_t count, const int64_t* item_clicked, const int64_t* label_next, const int64_t* all_items,
                            int64_t B, int64_t T, const int64_t* pool, int64_t N, int64_t num_items, int64_t sample_size,
                            int64_t nn, int32_t decay_div, int32_t jaccard, int32_t top_n, int64_t max_blocks,
                            int32_t* rank, int64_t* hist, int* err, void* stream);
/* Recommendations of the kNN baseline (DESIGN.md section 16) with the neighbours of nar_sknn_score: queries, exclusion,
 * top_n and outputs as in nar_baselines_recommend, over cand [N] (ascending distinct ids in [1, num_items)), in the
 * order (item score desc, first neighbour asc, id asc) of the ids some kept neighbour holds.  NAR_ERR_UNSUPPORTED for
 * S > 4096, T > 64 or top_n > 1024.  *err as in nar_baselines_recommend.  One launch.                           */
int nar_sknn_recommend(const int64_t* ids, const int32_t* lens, const int32_t* items, int64_t S, int64_t W, int64_t head,
                       int64_t count, const int64_t* item_clicked, int64_t B, int64_t T, const int32_t* q_pos, int64_t Q,
                       const int64_t* cand, int64_t N, int32_t exclude, int64_t num_items, int64_t sample_size, int64_t nn,
                       int32_t decay_div, int32_t jaccard, int32_t top_n, int64_t max_blocks, int64_t* out_ids,
                       double* out_scores, int* err, void* stream);

/* ---- NDCG, item coverage, ESI-R / ESI-RR and EILD-R / EILD-RR of top-n lists (csrc/eval_metrics.cu, spec
 *      oracle/eval_metrics_ref.py; the reference's metrics.py).  Coverage sets are bitmaps of (num_items + 31) / 32
 *      uint32 words.  *err = 1 for an id outside [0, num_items).                                                     */
/* sets the bit of every id of ids [n] (zeros skipped when skip_zero) */
int nar_eval_metrics_mark(const int64_t* ids, int64_t n, int64_t num_items, int32_t skip_zero, uint32_t* bitmap, int* err,
                          void* stream);
/* For every recommender row r < rows with bit r of row_mask set and every query q < nq whose label
 * labels[q * label_stride] is nonzero: the list ids[r * row_stride + q * q_stride + j], j < len, scored over its first
 * m = min(top_n, len) ids (2 <= m <= 64); NDCG counts the label's occurrences over all len.  pop [num_items] float32
 * normalised recent popularity; acr [num_items, acr_ld] float32 (first acr_dim columns) with fp64 row norms acr_norm.
 * per_query [rows, nq, 6] fp64 = {ndcg, esi-r, esi-rr, eild-r, eild-rr, 1} (zeros for label 0); the ids go into the
 * row's bitmap rec_bitmaps[r].                                                                                        */
int nar_eval_metrics_lists(const int64_t* ids, int64_t row_stride, int64_t q_stride, int64_t rows, int64_t row_mask,
                           int64_t nq, int64_t len, int32_t top_n, const int64_t* labels, int64_t label_stride,
                           const float* pop, const float* acr, int64_t acr_dim, int64_t acr_ld, const double* acr_norm,
                           int64_t num_items, double neg_relevance, double* per_query, uint32_t* rec_bitmaps, int* err,
                           void* stream);
/* acc [rows, 6] fp64 += the sum over q of per_query [rows, nq, 6], for the rows of row_mask, in a fixed order */
int nar_eval_metrics_reduce(const double* per_query, int64_t rows, int64_t row_mask, int64_t nq, double* acc, void* stream);
/* counts [n_maps] int64 = set bits of each of the bitmaps [n_maps, words] */
int nar_eval_metrics_popcount(const uint32_t* bitmaps, int64_t n_maps, int64_t words, int64_t* counts, void* stream);
/* Hit rate by session position: replaces the reference hook's HitRateBySessionPosition.add (metrics.py:136-168, fed by
 * evaluation.py update_metrics from nar_model.py:1595-1603 and benchmarks.py:35-55; spec oracle/by_position_ref.py).
 * For every recommender row r < rows with bit r of row_mask set and every query q < nq whose label
 * labels[q * label_stride] is nonzero, at position t = pos_idx[q] % T (pos_idx null: q % T, nq a multiple of T):
 * total[r * ld + t] += 1, and hits[r * ld + t] += 1 when the label is among the first min(top_n, len) ids of
 * ids[r * row_stride + q * q_stride + j].  hits / total int64 [rows, ld], ld >= T, T <= 1024.  With pop (float32 [V],
 * needs pos_idx and sess_off [n_sess + 1]: query rows of session b are sess_off[b] + t, t < sess_off[b+1] - sess_off[b]):
 * norm_pop[t] (float32 [T]) += pop[label] of each such row with a nonzero label, sessions b in order, one float32
 * round per add.  *err = 1 for an id outside [0, num_items) (the query is not counted).                             */
int nar_eval_by_position(const int64_t* ids, int64_t row_stride, int64_t q_stride, int64_t rows, int64_t row_mask,
                         int64_t nq, int64_t len, int32_t top_n, const int64_t* labels, int64_t label_stride,
                         const int32_t* pos_idx, int64_t T, const int32_t* sess_off, int64_t n_sess, const float* pop,
                         int64_t num_items, int64_t* hits, int64_t* total, int64_t ld, float* norm_pop, int* err,
                         void* stream);

/* ---- per-session evaluation logs (csrc/session_logs.cu, spec oracle/session_logs_ref.py; the reference hook's
 *      sessions_negative_items_log and sessions_chameleon_recommendations_log, nar_model.py:1529-1581).
 * flags bit 0: the negatives log, bit 1: the recommendations log.  A query is a compact row r < L whose label
 * label_next[pos_idx[r]] is nonzero; queries are numbered in row order (session-major), Q of them.  The packed buffer:
 *   int32 {Q, err, 0, 0}, int32 counts [B] (queries of each session), then from 16-byte aligned offsets and with
 *   Kp = K rounded up to 2, Wp = 1 + K rounded up to 4 (padding columns are 0):
 *   bit 0: neg [rows, Kp] int64 = negatives[pos_idx[r], :] of each query;
 *   bit 1: labels [rows] int64 = cand[r * cand_stride]; ids [rows, Wp] int64 = pred_ids[r, :]; probs [rows, Wp] float32 =
 *          pred_probs[r, :] rounded to 7 decimals as ndarray.round does in float32 (rint(x * 1e7) / 1e7); pops
 *          [rows, Wp] float32 = pop[ids] rounded the same way.
 * Only the first Q rows of a section are written.  nar_eval_session_logs_layout: offsets [9] = byte offsets of {counts,
 * neg, labels, ids, probs, pops}, the total bytes, Kp, Wp, for sections of `rows` rows.  nar_eval_session_logs_pack writes
 * the buffer `out` (16-byte aligned, laid out for rows = L) in one launch; err is set to 1 (never cleared) when an id of
 * pred_ids lies outside [0, num_items) (its popularity is written as 0).                                             */
int nar_eval_session_logs_layout(int64_t B, int64_t rows, int64_t K, int32_t flags, int64_t* offsets);
int nar_eval_session_logs_pack(const int64_t* pred_ids, const float* pred_probs, const int64_t* cand, int64_t cand_stride,
                               const int32_t* pos_idx, const int32_t* sess_off, const float* pop, const int64_t* negatives,
                               const int64_t* label_next, int64_t B, int64_t K, int64_t L, int64_t num_items, int32_t flags,
                               void* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NAR_B200_H */
