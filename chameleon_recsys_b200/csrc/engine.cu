// The NAR training / evaluation step sequenced in C: one call per phase instead of ~50 host round trips.
//
// Replaces the single session.run(train_op) of the reference trainer (nar_trainer_gcom.py:515-517) over the graph of
// nar_model.py:102-728: sampler (:265-276) -> features (:314-370) -> CAR (:374-405) -> RNN (:408, :1308-1342) ->
// FC1/FC2 (:410-438) -> scorer (:444-517) -> loss (:639-704) -> gradients -> TF-Adam (:706-722).  Only the valid
// positions (mask == 1) are materialised: padded positions never reach the loss (:660-664).
//
// Row layouts (L = valid local positions, n_cand = 1+K, R = L + L*n_cand):
//   H1 / E [R, C]  rows [0,L) = clicked items, then per position its positive followed by its K negatives
//   full mode      X [R, Fp] feature rows in the same order (every candidate row gathered and multiplied by W1)
//   dedup mode     XB [2L+U, Fp] base rows: L clicked, L positives, U unique-negative ITEM rows (csrc/car.cu):
//                  PP = XB[L:2L] W1 + b1 ; PI = XB[2L:, item cols] W1[item rows] ; PC = XB[:L, ctx cols] W1[ctx rows] + b1
//                  H1[L + l*n_cand + j] = leaky(j == 0 ? PP[l] : PC[l] + PI[u(l, j-1)]), stored transposed:
//                  H1cT [C, ldr] behind the L_cap clicked rows of H1, so that layer 2's weight gradient reads both
//                  operands in the major the tensor cores take (the forward reads it MN-major)
//                  backward: DB = [dH1(in) | dPP | dPI | dPC], the last three formed in the candidate rows' layer-2
//                  dgrad epilogue (no dH1 of the candidate rows), then ONE wgrad / dgrad over the 2L+U base rows (+ the
//                  context block), instead of two GEMMs over all R rows.
// Streams: the caller's stream carries the critical path (forward, dgrad chain); everything only Adam needs (weight /
// bias gradients) and the forward session branch run on an engine-owned auxiliary stream behind events.
#include "common.cuh"
#include <string.h>
#include <stdio.h>
#include <stdlib.h>

extern "C" int nar_sample_negatives_uidx(nar_ctx*, const int64_t*, int64_t, int64_t, int64_t, int64_t, const int64_t*, int64_t,
                                         int64_t, int64_t, uint64_t, uint32_t, int64_t*, int32_t*, const int64_t**,
                                         const int32_t**, void*, int64_t, void*);
namespace nar {
int recommend_rows(const int32_t* pos_idx, int64_t L, const int64_t* item_clicked, const int64_t* cand_ids, int64_t N,
                   int32_t* row_pos, int64_t* row_item, cudaStream_t st);        // csrc/recommend.cu
}

namespace {

constexpr int N_EVENTS = 64;

inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

struct Carver {
  char* base; int64_t off;
  explicit Carver(void* b) : base(static_cast<char*>(b)), off(0) {}
  template <typename T> T* take(int64_t n) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off = align_up(off + (n > 0 ? n : 1) * (int64_t)sizeof(T), 256);
    return p;
  }
};

struct PrepBufs {
  void* sampler_ws; int64_t sampler_bytes;
  int64_t* neg; int32_t* neg_uidx; float* stats; int32_t* row_pos; int64_t* row_item;
  int32_t* base_pos; int64_t* base_item; int64_t U;
};

struct StepBufs {
  float *X, *dX, *H1, *E, *dE, *dH1, *F1, *PR, *logits, *PD, *dPD, *Z1, *Z2, *Z3, *dZ1, *dZ2, *dZ3, *dPR, *dF1, *dHO;
  float *GX[NAR_MAX_LAYERS], *HO[NAR_MAX_LAYERS], *GT[NAR_MAX_LAYERS], *CD[NAR_MAX_LAYERS], *dGX[NAR_MAX_LAYERS],
        *HPV[NAR_MAX_LAYERS], *dHOb[NAR_MAX_LAYERS], *HOd[NAR_MAX_LAYERS],   // HOd: RNN outputs after DropoutWrapper
        *UO[NAR_MAX_LAYERS], *RH[NAR_MAX_LAYERS];
  // per cell: GT = UGRNN gate / GRU r (LSTM: none); CD = UGRNN and GRU candidate / LSTM cell state; UO = GRU u;
  // RH = GRU r * previous state.  The LSTM's activated gates replace its pre-activations in GX.
  float *P, *HR[NAR_MAX_LAYERS];   // residual stack: layer 0's input projection, each layer's output HO + its input
  float *PP, *PI, *PC, *DB;        // dedup: layer-1 pre-activations and their gradients
  float* H1cT; int64_t ldr;        // dedup: the candidate rows of H1 transposed, [C, ldr], ldr >= L_cap * n_cand
};

}  // namespace

// bf16x3 planes of the forward weights (fwd_precision 4; see gemm_wgmma.cu MODE 4): one entry per (weight block, K) a
// forward GEMM uses; refreshed by one nar_pack_bf16x3 launch after every optimiser step / weight load
constexpr int MAX_PLANES = 32;
struct PlaneSet {
  int n;
  int64_t off_W[MAX_PLANES]; int32_t K[MAX_PLANES], N[MAX_PLANES], ldw[MAX_PLANES], ld_out[MAX_PLANES];
  int64_t dst[MAX_PLANES];                 // element offset of the plane in `buf`
  const float* W[MAX_PLANES]; void* out[MAX_PLANES];
  uint16_t* buf; void* descs;
};

struct nar_engine {
  nar_ctx* ctx;
  nar_model_cfg cfg;
  PlaneSet planes;
  cudaStream_t aux;
  cudaEvent_t ev[N_EVENTS];
  int ev_i;
  float* WhT[NAR_MAX_LAYERS];       // transposed recurrent blocks [gate_blocks * Hp, Hp] (GRU: Whg, then Whc)
  int64_t launches;
  int fused_product;               // NAR_FUSED_SCORER_PRODUCT (default 1), read when the engine is created
};

namespace {

// The MLP scorer's product PD = Ec * PR[position] (nar_model.py:478, :493) folded into its first Dense layer's GEMMs: the
// forward and the weight gradient scale Ec by PR as they load it (nar_gemm_epilogue.a_scale, the same rounded product), the
// dgrad's epilogue forms dEc and dPR from whole positions (nar_gemm_epilogue.pred).  PD and dPD are never stored.  Needs
// the bf16x3 forward and single-pass TF32 backward, and positions that fit an M tile (1 + K <= 128); otherwise, or with
// NAR_FUSED_SCORER_PRODUCT=0, nar_mul_pred / nar_mul_pred_bwd run around the plain GEMMs.  A recommend call folds the
// product whenever the forward is bf16x3: the two other conditions belong to the training step's dgrad epilogue and
// backward precision, and a recommend call runs neither.
bool fused_product(const nar_engine* e) {
  const nar_model_cfg& c = e->cfg;
  return e->fused_product && c.ranking == 0 && c.K + 1 <= 128 && c.fwd_precision == 4 && c.bwd_precision == 1;
}

// gate blocks per unit (the width of GX, Wx and the bias): UGRNN (gate | candidate), GRU (r | u | candidate), LSTM (i | j | f | o)
int64_t gate_blocks(const nar_model_cfg& c) { return c.rnn_cell == NAR_CELL_LSTM ? 4 : c.rnn_cell == NAR_CELL_GRU ? 3 : 2; }

// the feature plan of one call: the static part + the call's staged context and popularity inputs + its row statistics
nar_feature_plan call_plan(const nar_model_cfg& c, const nar_step_io* io, const float* stats) {
  nar_feature_plan plan = c.plan;
  for (int i = 0; i < NAR_MAX_SRC; ++i) { plan.ctx_int[i] = io->ctx_int[i]; plan.ctx_float[i] = io->ctx_float[i]; }
  plan.pop_norm = io->pop_norm;
  plan.stats = stats;
  return plan;
}

int64_t prep_carve(const nar_engine* e, int64_t Bg, int64_t B, int64_t T, int64_t L_cap, void* base, PrepBufs* pb) {
  const nar_model_cfg& c = e->cfg;
  const int64_t K = c.K, n_cand = K + 1, Rcap = L_cap * (n_cand + 1);
  Carver cv(base);
  int64_t sb = 0;
  nar_sample_negatives_workspace(Bg, T + 1, c.buf_len, K, &sb);
  pb->sampler_bytes = sb;
  pb->sampler_ws = cv.take<char>(sb);
  pb->neg = cv.take<int64_t>(Bg * T * K);
  pb->neg_uidx = cv.take<int32_t>(c.dedup ? Bg * T * K : 1);
  pb->stats = cv.take<float>(24);
  pb->row_pos = cv.take<int32_t>(Rcap);
  pb->row_item = cv.take<int64_t>(Rcap);
  pb->U = K * 20 + 1;
  pb->base_pos = cv.take<int32_t>(c.dedup ? 2 * L_cap + pb->U : 1);
  pb->base_item = cv.take<int64_t>(c.dedup ? 2 * L_cap + pb->U : 1);
  (void)B;
  return cv.off;
}

// the session branch's buffers for L rows (what clicked_rows_forward writes), in the same order for a step and a recommend call
void session_carve(const nar_model_cfg& c, int64_t L, Carver& cv, StepBufs* sb) {
  const int64_t Hp = c.Hp;
  for (int i = 0; i < c.layers; ++i) {
    sb->GX[i] = cv.take<float>(L * gate_blocks(c) * Hp); sb->HO[i] = cv.take<float>(L * Hp);
    if (c.rnn_cell != NAR_CELL_LSTM) sb->GT[i] = cv.take<float>(L * Hp);
    sb->CD[i] = cv.take<float>(L * Hp);
    if (c.rnn_cell == NAR_CELL_GRU) { sb->UO[i] = cv.take<float>(L * Hp); sb->RH[i] = cv.take<float>(L * Hp); }
  }
  sb->F1 = cv.take<float>(L * 512);
  sb->PR = cv.take<float>(L * c.C);
  if (c.rnn_residual) {
    sb->P = cv.take<float>(L * Hp);
    for (int i = 0; i < c.layers; ++i) sb->HR[i] = cv.take<float>(L * Hp);
  }
}

int64_t step_carve(const nar_engine* e, int64_t L_cap, int train, void* base, StepBufs* sb) {
  const nar_model_cfg& c = e->cfg;
  const int64_t K = c.K, n_cand = K + 1, Rc = L_cap * n_cand, R = L_cap + Rc, C = c.C, Hp = c.Hp, Fp = c.Fp;
  const int64_t U = K * 20 + 1, NB = 2 * L_cap + U;
  memset(sb, 0, sizeof(*sb));
  Carver cv(base);
  if (c.dedup) { sb->X = cv.take<float>(NB * Fp); } else { sb->X = cv.take<float>(R * Fp); }
  if (c.dedup) {
    // column segments of 32 rows start 128-byte aligned; H1 keeps >= R * C floats
    sb->ldr = align_up(Rc, 32);
    sb->H1 = cv.take<float>(L_cap * C + C * sb->ldr);
    sb->H1cT = sb->H1 + L_cap * C;
  } else {
    sb->H1 = cv.take<float>(R * C);
  }
  sb->E = cv.take<float>(R * C);
  session_carve(c, L_cap, cv, sb);
  sb->logits = cv.take<float>(L_cap * n_cand);
  if (c.dedup) { sb->PP = cv.take<float>(L_cap * C); sb->PI = cv.take<float>(U * C); sb->PC = cv.take<float>(L_cap * C); }
  const bool fused = fused_product(e);
  if (c.ranking == 0) {
    if (!fused) sb->PD = cv.take<float>(Rc * C);
    sb->Z1 = cv.take<float>(Rc * 128); sb->Z2 = cv.take<float>(Rc * 64); sb->Z3 = cv.take<float>(Rc * 32);
  }
  if (train) {
    sb->dE = cv.take<float>(R * C);
    sb->dPR = cv.take<float>(L_cap * C); sb->dF1 = cv.take<float>(L_cap * 512); sb->dHO = cv.take<float>(L_cap * Hp);
    for (int i = 0; i < c.layers; ++i) {
      sb->dGX[i] = cv.take<float>(L_cap * gate_blocks(c) * Hp); sb->HPV[i] = cv.take<float>(L_cap * Hp); sb->dHOb[i] = cv.take<float>(L_cap * Hp);
    }
    if (c.ranking == 0) {
      sb->dZ3 = cv.take<float>(Rc * 32); sb->dZ2 = cv.take<float>(Rc * 64); sb->dZ1 = cv.take<float>(Rc * 128);
      if (!fused) sb->dPD = cv.take<float>(Rc * C);
    }
    if (c.keep_prob < 1.f)
      for (int i = 0; i < c.layers; ++i) sb->HOd[i] = cv.take<float>(L_cap * Hp);
    if (c.dedup) {
      sb->DB = cv.take<float>((3 * L_cap + U) * C);
      sb->dX = cv.take<float>(NB * Fp);
    } else {
      sb->dH1 = cv.take<float>(R * C);
      sb->dX = cv.take<float>(R * Fp);
    }
  }
  return cv.off;
}

// ---------------------------------------------------------------------------------------------- one step
struct Seq {
  nar_engine* e; const nar_step_io* io; cudaStream_t main, aux;
  bool use_aux, aux_dirty = false;
  int rc = 0;
  const nar_model_cfg& c;
  Seq(nar_engine* e_, const nar_step_io* io_, cudaStream_t s)
      : e(e_), io(io_), main(s), aux(e_->aux), use_aux(e_->cfg.use_aux_stream != 0), c(e_->cfg) {}

  cudaEvent_t next_event() { cudaEvent_t v = e->ev[e->ev_i]; e->ev_i = (e->ev_i + 1) % N_EVENTS; return v; }
  // stream that deferred work (weight / bias gradients, forward session branch) runs on, after everything queued on main so far
  cudaStream_t fork() {
    if (!use_aux) return main;
    cudaEvent_t v = next_event();
    if (cudaEventRecord(v, main) != cudaSuccess || cudaStreamWaitEvent(aux, v, 0) != cudaSuccess) rc = rc ? rc : (int)cudaGetLastError();
    aux_dirty = true;
    return aux;
  }
  void join() {
    if (!use_aux || !aux_dirty) return;
    cudaEvent_t v = next_event();
    if (cudaEventRecord(v, aux) != cudaSuccess || cudaStreamWaitEvent(main, v, 0) != cudaSuccess) rc = rc ? rc : (int)cudaGetLastError();
    aux_dirty = false;
  }
  void chk(int r) { if (r && !rc) rc = r; ++e->launches; }

  const float* W(int64_t off) const { return c.params + off; }
  float* G(int64_t off) const { return c.grads + off; }

  // Y[M,N] = act(X[M,Kd] * W[Kd,N] + b)      (W stored [in,out]: MN-major B operand, or its bf16x3 plane)
  // (a_scale: X's row i scaled by a_scale[i / group] as it is loaded, see fused_product; x_kmajor = 0: X is stored
  // transposed, [Kd, ldx])
  void fwd(const float* X, int64_t ldx, int64_t off_W, int64_t ldw, int64_t off_b, float* Y, int64_t ldy, int64_t M, int64_t N,
           int64_t Kd, int act, cudaStream_t st, const float* a_scale = nullptr, int64_t ld_scale = 0, int64_t group = 0,
           int x_kmajor = 1) {
    nar_gemm_epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.a_scale = a_scale; ep.ld_a_scale = ld_scale; ep.a_scale_group = group;
    ep.bias = off_b >= 0 ? W(off_b) : nullptr; ep.act = act; ep.split_k = 1; ep.precision = c.fwd_precision;
    ep.b_lo = c.fwd_precision == 3 ? c.params_lo + off_W : nullptr;
    if (c.fwd_precision == 4) {
      const PlaneSet& ps = e->planes;
      int i = 0;
      for (; i < ps.n; ++i) if (ps.off_W[i] == off_W && ps.K[i] == Kd && ps.N[i] == N) break;
      if (i == ps.n) { if (!rc) rc = NAR_ERR_INVALID; return; }   // planes_build registers every forward block: a miss is a bug
      ep.b_bf16 = ps.buf + ps.dst[i]; ep.ld_bf16 = ps.ld_out[i];
    }
    chk(nar_gemm_tf32(e->ctx, M, N, Kd, X, ldx, x_kmajor, W(off_W), ldw, 0, Y, ldy, &ep, st));
  }
  // dX[M,n_in] (+)= dY[M,n_out] * W^T, optionally times act'(aux)
  void dgrad(const float* dY, int64_t lddy, int64_t off_W, int64_t ldw, float* dX, int64_t lddx, int64_t M, int64_t n_in,
             int64_t n_out, int dact, const float* auxp, int64_t ld_aux, int accumulate, cudaStream_t st) {
    nar_gemm_epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.dact = dact; ep.aux = auxp; ep.ld_aux = ld_aux; ep.accumulate = accumulate; ep.split_k = accumulate ? 0 : 1;
    ep.precision = c.bwd_precision;
    chk(nar_gemm_tf32(e->ctx, M, n_in, n_out, dY, lddy, 1, W(off_W), ldw, 1, dX, lddx, &ep, st));
  }
  // dW[n_in,n_out] += X[rows,n_in]^T * dY[rows,n_out]   (split-K, red.add into the gradient buffer)
  // (a_scale: as in fwd)
  void wgrad(const float* X, int64_t ldx, const float* dY, int64_t lddy, int64_t off_W, int64_t ldw, int64_t n_in, int64_t n_out,
             int64_t rows, cudaStream_t st, const float* a_scale = nullptr, int64_t ld_scale = 0, int64_t group = 0) {
    nar_gemm_epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.a_scale = a_scale; ep.ld_a_scale = ld_scale; ep.a_scale_group = group;
    ep.accumulate = 1; ep.split_k = 0; ep.precision = c.bwd_precision;
    chk(nar_gemm_tf32(e->ctx, n_in, n_out, rows, X, ldx, 0, dY, lddy, 0, G(off_W), ldw, &ep, st));
  }
  // the same from X stored transposed (XT [n_in, ldxt]), as dW^T = dY^T * X: A = dY MN-major, B = XT K-major, so that
  // neither operand is transposed in shared memory; the epilogue adds the tile transposed into dW [in, out]
  void wgrad_xt(const float* XT, int64_t ldxt, const float* dY, int64_t lddy, int64_t off_W, int64_t ldw, int64_t n_in,
                int64_t n_out, int64_t rows, cudaStream_t st) {
    nar_gemm_epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.accumulate = 1; ep.split_k = 0; ep.precision = c.bwd_precision;
    chk(nar_gemm_tf32_dt(e->ctx, n_out, n_in, rows, dY, lddy, 0, XT, ldxt, 1, G(off_W), ldw, &ep, st));
  }
  // through the scorer product and the CAR tanh: v = dY W^T; dX[r] = v[r] * pred[r / group] * tanh'(cand[r]) and
  // dpred[l] = sum over position l's rows of v * cand (nar_mul_pred_bwd's arithmetic); the column sums of dX are added
  // to the gradient of the bias at off_b (the bias of the layer that produced cand)
  void dgrad_prod(const float* dY, int64_t lddy, int64_t off_W, int64_t ldw, const float* cand, const float* pred, int64_t group,
                  float* dX, float* dpred, int64_t off_b, int64_t M, int64_t n_in, int64_t n_out, cudaStream_t st) {
    nar_gemm_epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.dact = NAR_ACT_TANH; ep.aux = cand; ep.ld_aux = n_in; ep.split_k = 1; ep.precision = c.bwd_precision;
    ep.pred = pred; ep.d_pred = dpred; ep.ld_pred = n_in; ep.pred_group = group; ep.d_bias = G(off_b);
    chk(nar_gemm_tf32(e->ctx, M, n_in, n_out, dY, lddy, 1, W(off_W), ldw, 1, dX, n_in, &ep, st));
  }
  // through CAR layer 1 of the candidate rows (dedup): v = dY W^T is the gradient of H1c = leaky(pre) (nar_car_combine);
  // dPP = v * leaky'(pre) of the positives, dPC / dPI += the sums over the negatives (zeroed by the caller)
  void dgrad_car(const float* dY, int64_t lddy, int64_t off_W, int64_t ldw, const float* PP, const float* PC, const float* PI,
                 const int32_t* pos_idx, const int32_t* neg_uidx, float* dPP, float* dPC, float* dPI, int64_t M, int64_t n_in,
                 int64_t n_out, cudaStream_t st) {
    nar_gemm_epilogue ep; memset(&ep, 0, sizeof(ep));
    ep.dact = NAR_ACT_LEAKY_RELU; ep.split_k = 1; ep.precision = c.bwd_precision;
    ep.car_pp = PP; ep.car_pc = PC; ep.car_pi = PI; ep.car_pos_idx = pos_idx; ep.car_neg_uidx = neg_uidx;
    ep.car_dpp = dPP; ep.car_dpc = dPC; ep.car_dpi = dPI; ep.ld_car = n_in; ep.car_k = c.K;
    chk(nar_gemm_tf32(e->ctx, M, n_in, n_out, dY, lddy, 1, W(off_W), ldw, 1, nullptr, 0, &ep, st));
  }
  void bgrad(const float* dY, int64_t ld, int64_t rows, int64_t cols, int64_t off_b, cudaStream_t st) {
    chk(nar_colsum_add(dY, rows, cols, ld, G(off_b), st));
  }
  // training-step dropout at site tensor_id (masks of oracle/dropout_ref.py, keyed by each row's position); dst may be src
  void dropout(const float* src, float* dst, int64_t rows, int64_t cols, const int32_t* row_pos, int tensor_id, cudaStream_t st) {
    chk(nar_dropout_rows(src, dst, rows, cols, cols, row_pos, io->L, c.K + 1, c.K, tensor_id, c.keep_prob, c.dropout_seed,
                         (uint32_t)(io->global_step + 1), st));
  }
  // the scorer (nar_model.py:444-517) of n_pos positions x n_cand candidate rows Ec against their positions' PR, on main:
  // logits, and the softmax cross-entropy times inv_count added to loss[0] (:639-667; nov: the novelty regulariser).
  // MLP: `fused` folds the product Ec * PR into the M1 GEMM (fused_product), else nar_mul_pred writes it to PD first;
  // dZ3 given (training): also dZ3 and the last layer's gradients.  Cosine: dE / dPR given (training): their gradients.
  void scorer(const float* Ec, const float* PR, int64_t n_pos, int64_t n_cand, bool fused, float* PD, float* Z1, float* Z2,
              float* Z3, float* logits, float* loss, float inv_count, float* dZ3, float* dE, float* dPR,
              const nar_novelty_reg* nov) {
    const int64_t R = n_pos * n_cand, C = c.C;
    if (c.ranking == 0) {
      if (fused) {
        fwd(Ec, C, c.off_M[0], c.ld_M[0], c.off_c[0], Z1, 128, R, 128, C, NAR_ACT_LEAKY_RELU, main, PR, C, n_cand);
      } else {
        chk(nar_mul_pred(Ec, PR, n_pos, n_cand, C, PD, main));
        fwd(PD, C, c.off_M[0], c.ld_M[0], c.off_c[0], Z1, 128, R, 128, C, NAR_ACT_LEAKY_RELU, main);
      }
      fwd(Z1, 128, c.off_M[1], c.ld_M[1], c.off_c[1], Z2, 64, R, 64, 128, NAR_ACT_LEAKY_RELU, main);
      fwd(Z2, 64, c.off_M[2], c.ld_M[2], c.off_c[2], Z3, 32, R, 32, 64, NAR_ACT_LEAKY_RELU, main);
      chk(nar_score_softmax_ce(Z3, 32, 32, W(c.off_M[3]), c.ld_M[3], W(c.off_c[3]), n_pos, n_cand, c.inv_temperature, inv_count,
                               logits, loss, dZ3, dZ3 ? G(c.off_M[3]) : nullptr, dZ3 ? G(c.off_c[3]) : nullptr, nov, main));
    } else {
      chk(nar_cosine_softmax_ce(Ec, PR, n_pos, n_cand, C, c.inv_temperature, inv_count, logits, loss, dE, dPR, nov, main));
    }
  }
};

// CAR (nar_model.py:374-405) of the L clicked rows sb.X[0:L] on the main stream, then the session branch - RNN (:408,
// :1308-1342) + FC1 / FC2 (:410-438) -> sb.PR - forked onto the auxiliary stream, so that it runs under whatever the
// caller queues next on main (the candidate rows); the caller joins before reading sb.PR.  (Moving the two CAR GEMMs
// into the session branch as well was measured neutral and is not used: DESIGN.md section 6.)  `drop`: training-step
// dropout on the RNN outputs and FC1.  Residual stack (c.rnn_residual, DESIGN.md section 15): layer 0 reads P = E Wp + bp,
// and each layer's output HR = HO + its input feeds dropout, the next layer and FC1; HO stays the cell's own state.
void clicked_rows_forward(Seq& s, const StepBufs& sb, int64_t L, bool drop) {
  const nar_model_cfg& c = s.c;
  const nar_step_io* io = s.io;
  const int64_t B = io->B, C = c.C, Hp = c.Hp, Fp = c.Fp;
  s.fwd(sb.X, Fp, c.off_W1, C, c.off_b1, sb.H1, C, L, C, Fp, NAR_ACT_LEAKY_RELU, s.main);
  s.fwd(sb.H1, C, c.off_W2, C, c.off_b2, sb.E, C, L, C, C, NAR_ACT_TANH, s.main);
  cudaStream_t st = s.fork();
  const float* rnn_in = sb.E; int64_t n_in = C;
  if (c.rnn_residual) {            // InputProjectionWrapper: no activation
    s.fwd(sb.E, C, c.off_Wp, Hp, c.off_bp, sb.P, Hp, L, Hp, C, NAR_ACT_NONE, st);
    rnn_in = sb.P; n_in = Hp;
  }
  const int64_t gw = gate_blocks(c) * Hp;
  for (int i = 0; i < c.layers; ++i) {
    // input projection gx = x Wx + b, then the recurrence (csrc/rnn.cu)
    s.fwd(rnn_in, n_in, c.off_Wx[i], gw, c.off_rb[i], sb.GX[i], gw, L, gw, n_in, NAR_ACT_NONE, st);
    if (c.rnn_cell == NAR_CELL_GRU) {
      s.chk(nar_gru_fwd(s.e->ctx, sb.GX[i], s.W(c.off_Wh[i]), s.W(c.off_Whc[i]), io->sess_off, B, Hp, sb.HO[i], sb.GT[i], sb.UO[i],
                        sb.CD[i], sb.RH[i], st));
    } else if (c.rnn_cell == NAR_CELL_LSTM) {
      // LSTMCell (i | j | f | o): the recurrence leaves the activated gates in gx and the cell state in CD
      s.chk(nar_lstm_fwd(s.e->ctx, sb.GX[i], s.W(c.off_Wh[i]), io->sess_off, B, Hp, sb.HO[i], sb.CD[i], st));
    } else {
      s.chk(nar_ugrnn_fwd(s.e->ctx, sb.GX[i], s.W(c.off_Wh[i]), io->sess_off, B, Hp, sb.HO[i], sb.GT[i], sb.CD[i], st));
    }
    // ResidualWrapper: the output is cell(x) + x, the state the cell carries is its own
    const float* out = sb.HO[i];
    if (c.rnn_residual) { s.chk(nar_residual_add(sb.HO[i], rnn_in, L, Hp, Hp, sb.HR[i], st)); out = sb.HR[i]; }
    // DropoutWrapper(output_keep_prob) (nar_model.py:1330-1333): the cell's OUTPUT is dropped, its state is not
    if (drop) s.dropout(out, sb.HOd[i], L, Hp, io->pos_idx, 8 + i, st);
    rnn_in = drop ? sb.HOd[i] : out; n_in = Hp;
  }
  s.fwd(rnn_in, Hp, c.off_W3, 512, c.off_b3, sb.F1, 512, L, 512, Hp, NAR_ACT_LEAKY_RELU, st);
  if (drop) s.dropout(sb.F1, sb.F1, L, 512, io->pos_idx, 4, st);                                // nar_model.py:417-419
  s.fwd(sb.F1, 512, c.off_W4, C, c.off_b4, sb.PR, C, L, C, 512, NAR_ACT_TANH, st);
}

int run_step(nar_engine* e, const nar_step_io* io, cudaStream_t main) {
  const nar_model_cfg& c = e->cfg;
  const int64_t B = io->B, T = io->T, L = io->L, K = c.K, n_cand = K + 1, Rc = L * n_cand, R = L + Rc;
  const int64_t C = c.C, Hp = c.Hp, Fp = c.Fp, c0 = c.ctx_col0;
  const int train = io->train;
  if (L > io->L_cap || L < 0 || B <= 0) return NAR_ERR_INVALID;
  PrepBufs pb; StepBufs sb;
  if (prep_carve(e, io->Bg, B, T, io->L_cap, io->prep_ws, &pb) > io->prep_ws_bytes) return NAR_ERR_WORKSPACE;
  if (step_carve(e, io->L_cap, train, io->ws, &sb) > io->ws_bytes) return NAR_ERR_WORKSPACE;
  NAR_CHECK_CUDA(cudaMemsetAsync(io->loss, 0, 4 * sizeof(float), main));
  if (train) NAR_CHECK_CUDA(cudaMemsetAsync(c.grads, 0, (size_t)c.n_params * sizeof(float), main));
  if (L == 0) return NAR_OK;
  // dropout (training steps only): masks are per candidate row, so every row must be materialised
  const bool drop = train && c.keep_prob < 1.f;
  if (drop && c.dedup) return NAR_ERR_INVALID;
  Seq s(e, io, main);
  const float inv_count = 1.0f / (float)(io->L_global > 0 ? io->L_global : 1);
  const int64_t U = pb.U, NB = 2 * L + U;

  const nar_feature_plan plan = call_plan(c, io, pb.stats);
  nar_row_layout rl;
  if (c.dedup) { rl.n_rows = NB; rl.n_input = L; rl.n_cand = 0; rl.n_positive = L; rl.n_full = 2 * L; rl.ctx_col0 = c0; }
  else { rl.n_rows = R; rl.n_input = L; rl.n_cand = n_cand; rl.n_positive = 0; rl.n_full = R; rl.ctx_col0 = c0; }
  const int32_t* g_pos = c.dedup ? pb.base_pos : pb.row_pos;
  const int64_t* g_item = c.dedup ? pb.base_item : pb.row_item;
  s.chk(nar_gather_features(e->ctx, &plan, g_pos, g_item, &rl, io->event_ts, io->max_ts, sb.X, main));
  if (drop) s.dropout(sb.X, sb.X, R, Fp, pb.row_pos, 0, main);        // nar_model.py:338-340, :351-353, :367-369

  float* H1c = sb.H1 + L * C; float* Ec = sb.E + L * C;
  clicked_rows_forward(s, sb, L, drop);
  if (c.dedup) {
    s.fwd(sb.X + L * Fp, Fp, c.off_W1, C, c.off_b1, sb.PP, C, L, C, Fp, NAR_ACT_NONE, main);                       // positives: full rows
    s.fwd(sb.X + 2 * L * Fp, Fp, c.off_W1, C, -1, sb.PI, C, U, C, c0, NAR_ACT_NONE, main);                          // item half, once per unique id
    s.fwd(sb.X + c0, Fp, c.off_W1 + c0 * C, C, c.off_b1, sb.PC, C, L, C, Fp - c0, NAR_ACT_NONE, main);             // context half, once per position
    s.chk(nar_car_combine_t(sb.PP, sb.PC, sb.PI, io->pos_idx, pb.neg_uidx, L, K, C, NAR_ACT_LEAKY_RELU, sb.H1cT, sb.ldr, main));
    s.fwd(sb.H1cT, sb.ldr, c.off_W2, C, c.off_b2, Ec, C, Rc, C, C, NAR_ACT_TANH, main, nullptr, 0, 0, 0);
  } else {
    s.fwd(sb.X + L * Fp, Fp, c.off_W1, C, c.off_b1, H1c, C, Rc, C, Fp, NAR_ACT_LEAKY_RELU, main);
    s.fwd(H1c, C, c.off_W2, C, c.off_b2, Ec, C, Rc, C, C, NAR_ACT_TANH, main);
  }
  s.join();

  // ---- scorer + loss (nar_model.py:444-517, :639-667), optional novelty regulariser (:673-683)
  nar_novelty_reg nov; memset(&nov, 0, sizeof(nov));
  nov.factor = c.novelty_reg_factor; nov.log_base = c.plan.log_base_novelty; nov.pop_norm = io->pop_norm;
  nov.cand_ids = pb.row_item + L; nov.loss_nov = io->loss + 2;
  const nar_novelty_reg* novp = c.novelty_reg_factor > 0.f ? &nov : nullptr;
  const bool fused = fused_product(e);
  s.scorer(Ec, sb.PR, L, n_cand, fused, sb.PD, sb.Z1, sb.Z2, sb.Z3, sb.logits, io->loss, inv_count, train ? sb.dZ3 : nullptr,
           train ? sb.dE + L * C : nullptr, train ? sb.dPR : nullptr, novp);
  // every rank holds the same weights: the regulariser is added once (rank 0) so that a sum over ranks is exact
  // (off the critical path: it only feeds the reported loss)
  if (c.reg_l2 > 0.f && c.rank == 0) { cudaStream_t st = s.fork(); s.chk(nar_l2_loss_add(c.params, c.reg_end, c.reg_l2, io->loss + 1, st)); }
  if (!train || s.rc) { s.join(); return s.rc; }

  // =============================================================================================== backward
  float* dEc = sb.dE + L * C;
  if (c.ranking == 0) {
    { cudaStream_t st = s.fork(); s.wgrad(sb.Z2, 64, sb.dZ3, 32, c.off_M[2], c.ld_M[2], 64, 32, Rc, st); s.bgrad(sb.dZ3, 32, Rc, 32, c.off_c[2], st); }
    s.dgrad(sb.dZ3, 32, c.off_M[2], c.ld_M[2], sb.dZ2, 64, Rc, 64, 32, NAR_ACT_LEAKY_RELU, sb.Z2, 64, 0, main);
    { cudaStream_t st = s.fork(); s.wgrad(sb.Z1, 128, sb.dZ2, 64, c.off_M[1], c.ld_M[1], 128, 64, Rc, st); s.bgrad(sb.dZ2, 64, Rc, 64, c.off_c[1], st); }
    s.dgrad(sb.dZ2, 64, c.off_M[1], c.ld_M[1], sb.dZ1, 128, Rc, 128, 64, NAR_ACT_LEAKY_RELU, sb.Z1, 128, 0, main);
    {
      cudaStream_t st = s.fork();
      if (fused) s.wgrad(Ec, C, sb.dZ1, 128, c.off_M[0], c.ld_M[0], C, 128, Rc, st, sb.PR, C, n_cand);
      else s.wgrad(sb.PD, C, sb.dZ1, 128, c.off_M[0], c.ld_M[0], C, 128, Rc, st);
      s.bgrad(sb.dZ1, 128, Rc, 128, c.off_c[0], st);
    }
    // candidate rows: through the product and the CAR tanh in one pass; d(pred) reduced over the candidates, and the
    // candidate rows' share of the layer-2 bias gradient summed from the dEc the epilogue writes (red.add into the
    // gradient buffer, which the memset at the top of the step zeroed earlier on this stream)
    if (fused) {
      s.dgrad_prod(sb.dZ1, 128, c.off_M[0], c.ld_M[0], Ec, sb.PR, n_cand, dEc, sb.dPR, c.off_b2, Rc, C, 128, main);
    } else {
      s.dgrad(sb.dZ1, 128, c.off_M[0], c.ld_M[0], sb.dPD, C, Rc, C, 128, NAR_ACT_NONE, nullptr, 0, 0, main);
      s.chk(nar_mul_pred_bwd(sb.dPD, Ec, sb.PR, L, n_cand, C, NAR_ACT_TANH, dEc, sb.dPR, main));
    }
  } else {
    s.chk(nar_act_bwd(dEc, Ec, Rc * C, NAR_ACT_TANH, dEc, main));
  }
  // ---- the two branches that share CAR layer 2's weights, one after the other on the main stream:
  //   S  session branch: FC2 / FC1 (nar_model.py:410-426) -> BPTT -> d(E) of the L clicked rows - a dozen small kernels
  //   C  candidates: CAR layer-2 dgrad over the L*(1+K) candidate rows - the big GEMM (+ the CAR layer-1 sums)
  // then the clicked rows' CAR backward, which needs S's dE.  The candidate rows' layer-2 weight gradient needs only dEc:
  // queued on the auxiliary stream before S, the longest kernel of that stream starts as soon as dEc exists.
  {
    cudaStream_t st = s.fork();
    if (c.dedup) s.wgrad_xt(sb.H1cT, sb.ldr, dEc, C, c.off_W2, C, C, C, Rc, st);
    else s.wgrad(H1c, C, dEc, C, c.off_W2, C, C, C, Rc, st);
    if (!fused) s.bgrad(dEc, C, Rc, C, c.off_b2, st);            // fused: summed in dgrad_prod's epilogue
  }
  // ---- S
  {
    s.chk(nar_act_bwd(sb.dPR, sb.PR, L * C, NAR_ACT_TANH, sb.dPR, main));
    { cudaStream_t st = s.fork(); s.wgrad(sb.F1, 512, sb.dPR, C, c.off_W4, C, 512, C, L, st); s.bgrad(sb.dPR, C, L, C, c.off_b4, st); }
    s.dgrad(sb.dPR, C, c.off_W4, C, sb.dF1, 512, L, 512, C, NAR_ACT_LEAKY_RELU, sb.F1, 512, 0, main);
    if (drop) s.dropout(sb.dF1, sb.dF1, L, 512, io->pos_idx, 4, main); // F1 holds the dropped activations: re-apply the mask to the gradient
    const float* rnn_out = drop ? sb.HOd[c.layers - 1] : (c.rnn_residual ? sb.HR[c.layers - 1] : sb.HO[c.layers - 1]);
    { cudaStream_t st = s.fork(); s.wgrad(rnn_out, Hp, sb.dF1, 512, c.off_W3, 512, Hp, 512, L, st); s.bgrad(sb.dF1, 512, L, 512, c.off_b3, st); }
    s.dgrad(sb.dF1, 512, c.off_W3, 512, sb.dHO, Hp, L, Hp, 512, NAR_ACT_NONE, nullptr, 0, 0, main);
    float* dho = sb.dHO;
    for (int i = c.layers - 1; i >= 0; --i) {
      if (drop) s.dropout(dho, dho, L, Hp, io->pos_idx, 8 + i, main);   // gradient of the dropped cell output
      // dho now holds the gradient of the layer's output before dropout: the cell's d_hout and, with residual
      // connections, also the gradient of the layer's input through the skip path
      const float* x_in = i == 0 ? (c.rnn_residual ? sb.P : sb.E) : (drop ? sb.HOd[i - 1] : (c.rnn_residual ? sb.HR[i - 1] : sb.HO[i - 1]));
      const int64_t n_in = (i == 0 && !c.rnn_residual) ? C : Hp;
      // gx, Wx and the bias are gw wide; the recurrent blocks differ per cell
      const int64_t gw = gate_blocks(c) * Hp;
      if (c.rnn_cell == NAR_CELL_GRU) {
        float* cand_T = e->WhT[i] + 2 * Hp * Hp;     // Whc transposed, after Whg transposed
        s.chk(nar_transpose_f32(s.W(c.off_Wh[i]), Hp, 2 * Hp, 2 * Hp, e->WhT[i], Hp, main));
        s.chk(nar_transpose_f32(s.W(c.off_Whc[i]), Hp, Hp, Hp, cand_T, Hp, main));
        s.chk(nar_gru_bwd(e->ctx, dho, sb.HO[i], sb.GT[i], sb.UO[i], sb.CD[i], e->WhT[i], cand_T, io->sess_off, B, Hp, sb.dGX[i],
                          sb.HPV[i], main));
      } else {
        s.chk(nar_transpose_f32(s.W(c.off_Wh[i]), Hp, gw, gw, e->WhT[i], Hp, main));
        if (c.rnn_cell == NAR_CELL_LSTM)
          s.chk(nar_lstm_bwd(e->ctx, dho, sb.HO[i], sb.CD[i], sb.GX[i], e->WhT[i], io->sess_off, B, Hp, sb.dGX[i], sb.HPV[i], main));
        else
          s.chk(nar_ugrnn_bwd(e->ctx, dho, sb.HO[i], sb.GT[i], sb.CD[i], e->WhT[i], io->sess_off, B, Hp, sb.dGX[i], sb.HPV[i], main));
      }
      {
        cudaStream_t st = s.fork();
        s.wgrad(x_in, n_in, sb.dGX[i], gw, c.off_Wx[i], gw, n_in, gw, L, st);
        if (c.rnn_cell == NAR_CELL_GRU) {     // dWhg = h_prev^T d_gx[:, :2Hp], dWhc = (r * h_prev)^T d_gx[:, 2Hp:]
          s.wgrad(sb.HPV[i], Hp, sb.dGX[i], gw, c.off_Wh[i], 2 * Hp, Hp, 2 * Hp, L, st);
          s.wgrad(sb.RH[i], Hp, sb.dGX[i] + 2 * Hp, gw, c.off_Whc[i], Hp, Hp, Hp, L, st);
        } else {
          s.wgrad(sb.HPV[i], Hp, sb.dGX[i], gw, c.off_Wh[i], gw, Hp, gw, L, st);
        }
        s.bgrad(sb.dGX[i], gw, L, gw, c.off_rb[i], st);
      }
      if (c.rnn_residual) {
        // d(input) = dGX Wx^T + dho: accumulated onto dho once the cell's backward has read it (layer 0: dP)
        s.dgrad(sb.dGX[i], gw, c.off_Wx[i], gw, dho, Hp, L, Hp, gw, NAR_ACT_NONE, nullptr, 0, 1, main);
        if (i == 0) {
          { cudaStream_t st = s.fork(); s.wgrad(sb.E, C, dho, Hp, c.off_Wp, Hp, C, Hp, L, st); s.bgrad(dho, Hp, L, Hp, c.off_bp, st); }
          s.dgrad(dho, Hp, c.off_Wp, Hp, sb.dE, C, L, C, Hp, NAR_ACT_TANH, sb.E, C, 0, main);      // clicked rows of dE (pre-tanh)
        }
      } else if (i == 0) {
        s.dgrad(sb.dGX[0], gw, c.off_Wx[0], gw, sb.dE, C, L, C, gw, NAR_ACT_TANH, sb.E, C, 0, main);   // clicked rows of dE (pre-tanh)
      } else {
        s.dgrad(sb.dGX[i], gw, c.off_Wx[i], gw, sb.dHOb[i], Hp, L, Hp, gw, NAR_ACT_NONE, nullptr, 0, 0, main);
        dho = sb.dHOb[i];
      }
    }
  }
  // ---- C: CAR layer 2 of the candidate rows (shared weights: the clicked rows follow once S has produced their dE)
  float* DBin = sb.DB; float* DBpp = sb.DB + L * C; float* DBpi = sb.DB + 2 * L * C; float* DBpc = sb.DB + NB * C;
  if (c.dedup) {
    s.chk((int)cudaMemsetAsync(DBpi, 0, (size_t)(U + L) * C * sizeof(float), main));       // dPI | dPC: red.add targets
    s.dgrad_car(dEc, C, c.off_W2, C, sb.PP, sb.PC, sb.PI, io->pos_idx, pb.neg_uidx, DBpp, DBpc, DBpi, Rc, C, C, main);
  } else {
    s.dgrad(dEc, C, c.off_W2, C, sb.dH1 + L * C, C, Rc, C, C, NAR_ACT_LEAKY_RELU, H1c, C, 0, main);
  }
  { cudaStream_t st = s.fork(); s.wgrad(sb.H1, C, sb.dE, C, c.off_W2, C, C, C, L, st); s.bgrad(sb.dE, C, L, C, c.off_b2, st); }
  if (c.dedup) {
    s.dgrad(sb.dE, C, c.off_W2, C, DBin, C, L, C, C, NAR_ACT_LEAKY_RELU, sb.H1, C, 0, main);
    {
      cudaStream_t st = s.fork();
      s.wgrad(sb.X, Fp, sb.DB, C, c.off_W1, C, Fp, C, NB, st);                                    // clicked + positive + unique item rows
      s.wgrad(sb.X + c0, Fp, DBpc, C, c.off_W1 + c0 * C, C, Fp - c0, C, L, st);                    // context block of the negatives
      s.bgrad(sb.DB, C, NB, C, c.off_b1, st);
    }
    s.dgrad(sb.DB, C, c.off_W1, C, sb.dX, Fp, NB, Fp, C, NAR_ACT_NONE, nullptr, 0, 0, main);
    // the negatives' context gradient lands on the clicked row of the same position (identical raw context features)
    s.dgrad(DBpc, C, c.off_W1 + c0 * C, C, sb.dX + c0, Fp, L, Fp - c0, C, NAR_ACT_NONE, nullptr, 0, 1, main);
  } else {
    s.dgrad(sb.dE, C, c.off_W2, C, sb.dH1, C, L, C, C, NAR_ACT_LEAKY_RELU, sb.H1, C, 0, main);
    { cudaStream_t st = s.fork(); s.wgrad(sb.X, Fp, sb.dH1, C, c.off_W1, C, Fp, C, R, st); s.bgrad(sb.dH1, C, R, C, c.off_b1, st); }
    s.dgrad(sb.dH1, C, c.off_W1, C, sb.dX, Fp, R, Fp, C, NAR_ACT_NONE, nullptr, 0, 0, main);
    if (drop) s.dropout(sb.dX, sb.dX, R, Fp, pb.row_pos, 0, main);
  }
  s.chk(nar_gather_features_bwd(e->ctx, &plan, g_pos, g_item, &rl, io->event_ts, io->max_ts, sb.dX, s.G(c.off_gamma),
                                s.G(c.off_beta), main));
  s.join();
  return s.rc;
}

// ---------------------------------------------------------------------------------------------- recommend
// Workspace of one recommend call: L clicked rows, Q queries, N candidates, processed in blocks of qb queries x nb
// candidates.  The session part reuses the StepBufs fields clicked_rows_forward reads and writes.
struct RecBufs {
  StepBufs sb;
  int32_t* row_pos; int64_t* row_item;
  float *stats, *PC, *PCq, *PRq, *logits, *lg_chunk, *PI, *H1g, *Eg, *Z1, *Z2, *Z3, *loss;
};

int64_t rec_carve(const nar_engine* e, int64_t L, int64_t Q, int64_t N, int64_t qb, int64_t nb, int gather_q, void* base,
                  RecBufs* rb) {
  const nar_model_cfg& c = e->cfg;
  const int64_t C = c.C, Fp = c.Fp, P = qb * nb;
  memset(rb, 0, sizeof(*rb));
  StepBufs& sb = rb->sb;
  Carver cv(base);
  rb->row_pos = cv.take<int32_t>(L + N);
  rb->row_item = cv.take<int64_t>(L + N);
  rb->stats = cv.take<float>(24);
  rb->loss = cv.take<float>(4);
  sb.X = cv.take<float>((L + N) * Fp);
  sb.H1 = cv.take<float>(L * C);
  sb.E = cv.take<float>(L * C);
  session_carve(c, L, cv, &sb);
  rb->PC = cv.take<float>(L * C);
  rb->PCq = gather_q ? cv.take<float>(Q * C) : rb->PC;
  rb->PRq = gather_q ? cv.take<float>(Q * C) : sb.PR;
  rb->logits = cv.take<float>(qb * N);
  rb->lg_chunk = nb < N ? cv.take<float>(P) : rb->logits;
  rb->PI = cv.take<float>(nb * C);
  rb->H1g = cv.take<float>(P * C);                 // layer-1 activations, then the product with PR (MLP scorer)
  rb->Eg = cv.take<float>(P * C);
  if (c.ranking == 0) { rb->Z1 = cv.take<float>(P * 128); rb->Z2 = cv.take<float>(P * 64); rb->Z3 = cv.take<float>(P * 32); }
  return cv.off;
}

// largest candidate chunk the cosine scorer takes (its shared memory holds the prediction row + 3 floats per candidate)
int64_t cosine_chunk_cap(const nar_model_cfg& c) { return (48 * 1024 / 4 - c.C) / 3; }

// Blocks within `budget` bytes: as many queries as fit with at most half the budget in the [qb, N] logits, then as many
// candidates per chunk as the rest allows.  Returns the workspace size, or -1 when not even one query x one candidate fits.
int64_t rec_plan(const nar_engine* e, int64_t L, int64_t Q, int64_t N, int gather_q, int64_t budget, int64_t* qb_out,
                 int64_t* nb_out) {
  const nar_model_cfg& c = e->cfg;
  RecBufs rb;
  const int64_t fixed = rec_carve(e, L, Q, N, 0, 0, gather_q, nullptr, &rb);
  if (fixed >= budget) return -1;
  int64_t qb = (budget - fixed) / 2 / (N * 4);
  qb = qb > Q ? Q : (qb < 1 ? 1 : qb);
  const int64_t nb_cap = (c.ranking == 1 && cosine_chunk_cap(c) < N) ? cosine_chunk_cap(c) : N;
  for (;;) {
    // bytes per candidate of a chunk: its PI row, qb pairs of activations, qb chunk logits
    const int64_t per = 4 * (c.C + qb * (2 * c.C + (c.ranking == 0 ? 128 + 64 + 32 : 0) + 1));
    const int64_t avail = budget - rec_carve(e, L, Q, N, qb, 0, gather_q, nullptr, &rb) - 8 * 256;   // carve alignment
    int64_t nb = avail > 0 ? avail / per : 0;
    nb = nb > nb_cap ? nb_cap : nb;
    while (nb >= 1 && rec_carve(e, L, Q, N, qb, nb, gather_q, nullptr, &rb) > budget) nb -= nb / 64 + 1;
    if (nb >= 1) { *qb_out = qb; *nb_out = nb; return rec_carve(e, L, Q, N, qb, nb, gather_q, nullptr, &rb); }
    if (qb == 1) return -1;
    qb = (qb + 1) / 2;
  }
}

// Scores every (query, candidate) pair of a recommend call block by block: each finished [Qb, N] logits block of the
// queries q0 .. q0+Qb-1 goes to finish(logits, q0, Qb) (the top n, or the label ranks of an unsampled evaluation).
template <class Finish>
int run_candidate_blocks(nar_engine* e, const nar_step_io* io, const int64_t* q_rows, int64_t Q, const int64_t* cand_ids,
                         int64_t N, int64_t qb, int64_t nb, cudaStream_t main, Finish finish) {
  const nar_model_cfg& c = e->cfg;
  const int64_t L = io->L, C = c.C, Fp = c.Fp, c0 = c.ctx_col0;
  if (L <= 0 || Q <= 0 || Q > L || N <= 0 || qb < 1 || nb < 1 || (c.ranking == 1 && nb > cosine_chunk_cap(c))) return NAR_ERR_INVALID;
  if (qb > Q) qb = Q;
  if (nb > N) nb = N;
  const int gather_q = q_rows != nullptr;
  RecBufs rb;
  if (rec_carve(e, L, Q, N, qb, nb, gather_q, io->ws, &rb) > io->ws_bytes) return NAR_ERR_WORKSPACE;
  StepBufs& sb = rb.sb;
  Seq s(e, io, main);

  // ---- rows, statistics (empty buffer: the candidate rows are group 2, like the negatives), one gather.  io->stats:
  // statistics the caller computed instead (a data-parallel rank's, over the global batch's rows)
  s.chk(nar::recommend_rows(io->pos_idx, L, io->item_clicked, cand_ids, N, rb.row_pos, rb.row_item, main));
  if (!io->stats)
    s.chk(nar_feature_stats(e->ctx, io->buffer, c.buf_len, c.n_norm, c.plan.created_at_ts, io->pop_norm, io->max_ts,
                            c.plan.log_base_recency, c.plan.log_base_novelty, rb.row_pos, rb.row_item, L + N, L, 0, io->event_ts,
                            rb.stats, main));
  const nar_feature_plan plan = call_plan(c, io, io->stats ? io->stats : rb.stats);
  nar_row_layout rl;
  rl.n_rows = L + N; rl.n_input = L; rl.n_cand = 0; rl.n_positive = 0; rl.n_full = L; rl.ctx_col0 = c0;
  s.chk(nar_gather_features(e->ctx, &plan, rb.row_pos, rb.row_item, &rl, io->event_ts, io->max_ts, sb.X, main));
  if (s.rc) return s.rc;

  // ---- clicked rows + session branch (aux), the context half of layer 1 per position (main)
  clicked_rows_forward(s, sb, L, false);
  s.fwd(sb.X + c0, Fp, c.off_W1 + c0 * C, C, c.off_b1, rb.PC, C, L, C, Fp - c0, NAR_ACT_NONE, main);
  s.join();
  if (gather_q) {
    s.chk(nar_gather_rows_f32(rb.PC, L, C, (int)C, q_rows, Q, rb.PCq, C, main));
    s.chk(nar_gather_rows_f32(sb.PR, L, C, (int)C, q_rows, Q, rb.PRq, C, main));
  }

  // ---- per block of queries: every candidate chunk into logits [qb, N], then the top n of each query
  const bool fused = e->fused_product && c.fwd_precision == 4;
  for (int64_t q0 = 0; q0 < Q && !s.rc; q0 += qb) {
    const int64_t Qb = Q - q0 < qb ? Q - q0 : qb;
    const float* pcq = rb.PCq + q0 * C; const float* prq = rb.PRq + q0 * C;
    for (int64_t j0 = 0; j0 < N && !s.rc; j0 += nb) {
      const int64_t Nc = N - j0 < nb ? N - j0 : nb, P = Qb * Nc;
      s.fwd(sb.X + (L + j0) * Fp, Fp, c.off_W1, C, -1, rb.PI, C, Nc, C, c0, NAR_ACT_NONE, main);     // item half, per candidate
      s.chk(nar_car_combine_grid(pcq, rb.PI, Qb, Nc, C, NAR_ACT_LEAKY_RELU, rb.H1g, main));
      s.fwd(rb.H1g, C, c.off_W2, C, c.off_b2, rb.Eg, C, P, C, C, NAR_ACT_TANH, main);
      float* lg = Nc == N ? rb.logits : rb.lg_chunk;
      s.scorer(rb.Eg, prq, Qb, Nc, fused, rb.H1g, rb.Z1, rb.Z2, rb.Z3, lg, rb.loss, 0.f, nullptr, nullptr, nullptr, nullptr);
      if (Nc != N)
        s.chk((int)cudaMemcpy2DAsync(rb.logits + j0, (size_t)N * sizeof(float), lg, (size_t)Nc * sizeof(float),
                                     (size_t)Nc * sizeof(float), (size_t)Qb, cudaMemcpyDeviceToDevice, main));
    }
    s.chk(finish(rb.logits, q0, Qb));
  }
  return s.rc;
}

int run_recommend(nar_engine* e, const nar_step_io* io, const int64_t* q_rows, const int32_t* q_pos, int64_t Q,
                  const int64_t* cand_ids, int64_t N, int32_t top_n, int32_t exclude, int64_t qb, int64_t nb, int64_t* out_ids,
                  float* out_scores, float* out_probs, cudaStream_t main) {
  if (top_n < 1 || top_n > N || top_n > 4096) return NAR_ERR_INVALID;
  const int64_t T = io->T;
  return run_candidate_blocks(e, io, q_rows, Q, cand_ids, N, qb, nb, main, [&](const float* logits, int64_t q0, int64_t Qb) {
    return nar_topn_candidates(logits, cand_ids, Qb, N, top_n, exclude ? io->item_clicked : nullptr, q_pos + q0, T,
                               out_ids + q0 * top_n, out_scores ? out_scores + q0 * top_n : nullptr,
                               out_probs ? out_probs + q0 * top_n : nullptr, main);
  });
}

// every valid position of the batch is a query (Q = L, q_pos = pos_idx); see nar_engine_rank_labels
int run_rank_labels(nar_engine* e, const nar_step_io* io, const int64_t* cand_ids, int64_t N, int32_t top_n, int64_t qb,
                    int64_t nb, int32_t* rank, int64_t* hist, cudaStream_t main) {
  if (top_n < 1) return NAR_ERR_INVALID;
  const int64_t T = io->T;
  const int32_t* q_pos = io->pos_idx;
  return run_candidate_blocks(e, io, nullptr, io->L, cand_ids, N, qb, nb, main, [&](const float* logits, int64_t q0, int64_t Qb) {
    return nar_rank_labels(logits, cand_ids, Qb, N, io->label_next, io->all_items, q_pos + q0, T, top_n, rank + q0, hist, main);
  });
}

}  // namespace

// NAR_ERR_INVALID when the forward blocks do not fit MAX_PLANES
int planes_build(nar_engine* e) {
  const nar_model_cfg& c = e->cfg;
  PlaneSet& ps = e->planes;
  ps.n = 0;
  int64_t total = 0;
  bool overflow = false;
  auto add = [&](int64_t off, int64_t K, int64_t N, int64_t ldw) {
    if (ps.n >= MAX_PLANES) { overflow = true; return; }
    const int i = ps.n++;
    ps.off_W[i] = off; ps.K[i] = (int32_t)K; ps.N[i] = (int32_t)N; ps.ldw[i] = (int32_t)ldw;
    ps.ld_out[i] = (int32_t)((K + 31) / 32 * 64);
    ps.dst[i] = total;
    total += align_up((int64_t)N * ps.ld_out[i], 128);
  };
  const int64_t C = c.C, Hp = c.Hp, Fp = c.Fp, c0 = c.ctx_col0;
  add(c.off_W1, Fp, C, C); add(c.off_W1, c0, C, C); add(c.off_W1 + c0 * C, Fp - c0, C, C);
  add(c.off_W2, C, C, C); add(c.off_W3, Hp, 512, 512); add(c.off_W4, 512, C, C);
  add(c.off_M[0], C, 128, c.ld_M[0]); add(c.off_M[1], 128, 64, c.ld_M[1]); add(c.off_M[2], 64, 32, c.ld_M[2]);
  for (int i = 0; i < c.layers; ++i) {
    const int64_t gw = gate_blocks(c) * Hp;
    add(c.off_Wx[i], (i == 0 && !c.rnn_residual) ? C : Hp, gw, gw);
  }
  if (c.rnn_residual) add(c.off_Wp, C, Hp, Hp);
  if (overflow) return NAR_ERR_INVALID;
  if (!ps.buf) {
    cudaMalloc(&ps.buf, (size_t)total * sizeof(uint16_t));
    cudaMemset(ps.buf, 0, (size_t)total * sizeof(uint16_t));
    cudaMalloc(&ps.descs, MAX_PLANES * 32);
  }
  for (int i = 0; i < ps.n; ++i) { ps.W[i] = c.params + ps.off_W[i]; ps.out[i] = ps.buf + ps.dst[i]; }
  return NAR_OK;
}

int planes_refresh(nar_engine* e, cudaStream_t st) {
  PlaneSet& ps = e->planes;
  if (!ps.buf || ps.n == 0) return NAR_ERR_INVALID;
  ++e->launches;
  return nar_pack_bf16x3(ps.W, ps.out, ps.K, ps.N, ps.ldw, ps.ld_out, ps.n, ps.descs, st);
}

// ================================================================================================ C ABI
extern "C" int nar_engine_create(nar_ctx* ctx, const nar_model_cfg* cfg, nar_engine** out) {
  if (!ctx || !cfg || !out) return NAR_ERR_INVALID;
  *out = nullptr;
  if (cfg->layers < 1 || cfg->layers > NAR_MAX_LAYERS || cfg->rnn_cell < NAR_CELL_UGRNN || cfg->rnn_cell > NAR_CELL_LSTM ||
      cfg->ranking < 0 || cfg->ranking > 1)
    return NAR_ERR_UNSUPPORTED;
  if ((cfg->C & 3) || (cfg->Hp & 3) || (cfg->Fp & 3) || (cfg->ctx_col0 & 3) || cfg->ctx_col0 <= 0 || cfg->ctx_col0 >= cfg->Fp)
    return NAR_ERR_INVALID;
  if (!cfg->params || !cfg->grads || !cfg->adam_m || !cfg->adam_v || !cfg->params_lo) return NAR_ERR_INVALID;
  nar_engine* e = new nar_engine();
  memset(e, 0, sizeof(*e));
  e->ctx = ctx; e->cfg = *cfg;
  { const char* v = getenv("NAR_FUSED_SCORER_PRODUCT"); e->fused_product = !(v && atoi(v) == 0); }
  NAR_CHECK_CUDA(cudaSetDevice(ctx->device));
  if (cudaStreamCreateWithFlags(&e->aux, cudaStreamNonBlocking) != cudaSuccess) { delete e; return NAR_ERR_NO_DEVICE; }
  for (int i = 0; i < N_EVENTS; ++i)
    if (cudaEventCreateWithFlags(&e->ev[i], cudaEventDisableTiming) != cudaSuccess) { delete e; return NAR_ERR_NO_DEVICE; }
  for (int i = 0; i < cfg->layers; ++i) {
    const size_t wht = (size_t)gate_blocks(*cfg) * cfg->Hp * cfg->Hp;
    if (cudaMalloc(&e->WhT[i], wht * sizeof(float)) != cudaSuccess) { delete e; return NAR_ERR_NO_DEVICE; }
  }
  if (planes_build(e) != NAR_OK) { delete e; return NAR_ERR_INVALID; }
  if (!e->planes.buf || !e->planes.descs) { delete e; return NAR_ERR_NO_DEVICE; }
  *out = e;
  return NAR_OK;
}

extern "C" int nar_engine_refresh(nar_engine* e, void* stream) {
  if (!e) return NAR_ERR_INVALID;
  return planes_refresh(e, as_stream(stream));
}

extern "C" int nar_engine_destroy(nar_engine* e) {
  if (!e) return NAR_OK;
  cudaStreamSynchronize(e->aux);
  for (int i = 0; i < NAR_MAX_LAYERS; ++i) if (e->WhT[i]) cudaFree(e->WhT[i]);
  for (int i = 0; i < N_EVENTS; ++i) if (e->ev[i]) cudaEventDestroy(e->ev[i]);
  if (e->aux) cudaStreamDestroy(e->aux);
  if (e->planes.buf) cudaFree(e->planes.buf);
  if (e->planes.descs) cudaFree(e->planes.descs);
  delete e;
  return NAR_OK;
}

extern "C" int nar_engine_update_cfg(nar_engine* e, const nar_model_cfg* cfg) {
  if (!e || !cfg) return NAR_ERR_INVALID;
  if (cfg->layers != e->cfg.layers || cfg->Hp != e->cfg.Hp || cfg->C != e->cfg.C || cfg->Fp != e->cfg.Fp ||
      cfg->rnn_cell != e->cfg.rnn_cell || cfg->rnn_residual != e->cfg.rnn_residual)
    return NAR_ERR_INVALID;        // structural changes need a new engine
  e->cfg = *cfg;
  return planes_build(e);               // the parameter buffer may have changed (share_params)
}

extern "C" int nar_engine_workspace_bytes(const nar_engine* e, int64_t Bg, int64_t B, int64_t T, int64_t L_cap, int32_t train,
                                          int64_t* prep_bytes, int64_t* ws_bytes) {
  if (!e || Bg <= 0 || B <= 0 || T <= 0 || L_cap < 0) return NAR_ERR_INVALID;
  PrepBufs pb; StepBufs sb;
  if (prep_bytes) *prep_bytes = prep_carve(e, Bg, B, T, L_cap, nullptr, &pb);
  if (ws_bytes) *ws_bytes = step_carve(e, L_cap, train, nullptr, &sb);
  return NAR_OK;
}

extern "C" int nar_engine_prepare(nar_engine* e, const nar_step_io* io, void* stream) {
  if (!e || !io || !io->prep_ws || !io->all_items || !io->buffer) return NAR_ERR_INVALID;
  const nar_model_cfg& c = e->cfg;
  const int64_t B = io->B, Bg = io->Bg, T = io->T, L = io->L, K = c.K, n_cand = K + 1, R = L + L * n_cand;
  if (L > io->L_cap || io->sess0 < 0 || io->sess0 + B > Bg) return NAR_ERR_INVALID;
  PrepBufs pb;
  if (prep_carve(e, Bg, B, T, io->L_cap, io->prep_ws, &pb) > io->prep_ws_bytes) return NAR_ERR_WORKSPACE;
  cudaStream_t st = as_stream(stream);
  int64_t* neg_local = pb.neg + io->sess0 * T * K;
  int32_t* uidx_local = c.dedup ? pb.neg_uidx + io->sess0 * T * K : nullptr;
  const int64_t* uitems = nullptr; const int32_t* n_unique = nullptr;
  int rc = nar_sample_negatives_uidx(e->ctx, io->all_items, Bg, T + 1, io->sess0, B, io->buffer, c.buf_len, K, c.n_from_buffer,
                                     c.sampler_seed, io->sampler_step, neg_local, uidx_local, &uitems, &n_unique, pb.sampler_ws,
                                     pb.sampler_bytes, st);
  e->launches += 2;
  if (rc) return rc;
  if (L <= 0) return NAR_OK;
  rc = nar_build_rows(io->pos_idx, L, io->item_clicked, io->label_next, pb.neg, K, pb.row_pos, pb.row_item, st);
  ++e->launches;
  if (rc) return rc;
  rc = nar_feature_stats(e->ctx, io->buffer, c.buf_len, c.n_norm, c.plan.created_at_ts, io->pop_norm, io->max_ts,
                         c.plan.log_base_recency, c.plan.log_base_novelty, pb.row_pos, pb.row_item, R, L, n_cand, io->event_ts,
                         pb.stats, st);
  ++e->launches;
  if (rc) return rc;
  if (c.dedup) {
    rc = nar_build_base_rows(io->pos_idx, L, io->item_clicked, io->label_next, uitems, n_unique, pb.U, pb.neg_uidx, K, pb.base_pos,
                             pb.base_item, st);
    ++e->launches;
  }
  return rc;
}

extern "C" int nar_engine_step(nar_engine* e, const nar_step_io* io, void* stream) {
  if (!e || !io || !io->prep_ws || !io->ws || !io->loss) return NAR_ERR_INVALID;
  return run_step(e, io, as_stream(stream));
}

extern "C" int nar_engine_apply(nar_engine* e, const nar_step_io* io, void* stream) {
  if (!e || !io) return NAR_ERR_INVALID;
  const nar_model_cfg& c = e->cfg;
  ++e->launches;
  int rc = nar_adam_tf(c.params, c.grads, c.adam_m, c.adam_v, c.n_params, c.reg_end, c.reg_l2, c.lr, c.beta1, c.beta2, c.eps,
                       io->global_step + 1, c.params_lo, stream);
  if (rc == NAR_OK && c.fwd_precision == 4) rc = planes_refresh(e, as_stream(stream));
  return rc;
}

extern "C" int nar_engine_recommend_workspace_bytes(const nar_engine* e, int64_t L, int64_t Q, int64_t N, int32_t gather_q,
                                                    int64_t budget_bytes, int64_t* ws_bytes, int64_t* q_block, int64_t* n_block) {
  if (!e || !ws_bytes || !q_block || !n_block || L <= 0 || Q <= 0 || Q > L || N <= 0) return NAR_ERR_INVALID;
  const int64_t b = rec_plan(e, L, Q, N, gather_q != 0, budget_bytes, q_block, n_block);
  if (b < 0) return NAR_ERR_WORKSPACE;
  *ws_bytes = b;
  return NAR_OK;
}

extern "C" int nar_engine_recommend(nar_engine* e, const nar_step_io* io, const int64_t* q_rows, const int32_t* q_pos, int64_t Q,
                                    const int64_t* cand_ids, int64_t N, int32_t top_n, int32_t exclude_session_clicks,
                                    int64_t q_block, int64_t n_block, int64_t* out_ids, float* out_scores, float* out_probs,
                                    void* stream) {
  if (!e || !io || !io->ws || !q_pos || !cand_ids || !out_ids || !io->buffer || !io->pop_norm || !io->item_clicked) return NAR_ERR_INVALID;
  if (io->train) return NAR_ERR_INVALID;
  return run_recommend(e, io, q_rows, q_pos, Q, cand_ids, N, top_n, exclude_session_clicks, q_block, n_block, out_ids, out_scores,
                       out_probs, as_stream(stream));
}

extern "C" int nar_engine_rank_labels(nar_engine* e, const nar_step_io* io, const int64_t* cand_ids, int64_t N, int32_t top_n,
                                      int64_t q_block, int64_t n_block, int32_t* rank, int64_t* hist, void* stream) {
  if (!e || !io || !io->ws || !io->pos_idx || !cand_ids || !rank || !hist || !io->buffer || !io->pop_norm || !io->item_clicked ||
      !io->label_next || !io->all_items)
    return NAR_ERR_INVALID;
  if (io->train) return NAR_ERR_INVALID;
  if (io->T + 1 > 1024) return NAR_ERR_UNSUPPORTED;          // the exclusion row of nar_rank_labels
  return run_rank_labels(e, io, cand_ids, N, top_n, q_block, n_block, rank, hist, as_stream(stream));
}

extern "C" int64_t nar_engine_launch_count(const nar_engine* e) { return e ? e->launches : 0; }

extern "C" int nar_engine_buffer(const nar_engine* e, const nar_step_io* io, const char* name, void** ptr, int64_t* rows, int64_t* ld) {
  if (!e || !io || !name || !ptr) return NAR_ERR_INVALID;
  const nar_model_cfg& c = e->cfg;
  const int64_t L = io->L, K = c.K, n_cand = K + 1, Rc = L * n_cand, R = L + Rc;
  PrepBufs pb; StepBufs sb;
  prep_carve(e, io->Bg, io->B, io->T, io->L_cap, io->prep_ws, &pb);
  step_carve(e, io->L_cap, io->train, io->ws, &sb);
  const int64_t NB = 2 * L + pb.U;
  struct Ent { const char* n; void* p; int64_t r, l; };
  const Ent tab[] = {
      {"neg", pb.neg, io->Bg * io->T, K}, {"neg_uidx", pb.neg_uidx, io->Bg * io->T, K}, {"stats", pb.stats, 1, 24},
      {"row_pos", pb.row_pos, R, 1}, {"row_item", pb.row_item, R, 1}, {"base_pos", pb.base_pos, NB, 1},
      {"base_item", pb.base_item, NB, 1},
      {"X", sb.X, c.dedup ? NB : R, c.Fp}, {"dX", sb.dX, c.dedup ? NB : R, c.Fp}, {"H1", sb.H1, R, c.C}, {"H1cT", sb.H1cT, c.C, sb.ldr}, {"E", sb.E, R, c.C},
      {"dE", sb.dE, R, c.C}, {"dPR", sb.dPR, L, c.C}, {"dH1", sb.dH1, R, c.C}, {"F1", sb.F1, L, 512}, {"PR", sb.PR, L, c.C},
      {"logits", sb.logits, L, n_cand}, {"PD", sb.PD, Rc, c.C}, {"Z1", sb.Z1, Rc, 128}, {"Z2", sb.Z2, Rc, 64}, {"Z3", sb.Z3, Rc, 32}, {"PP", sb.PP, L, c.C},
      {"PI", sb.PI, pb.U, c.C}, {"PC", sb.PC, L, c.C}, {"DB", sb.DB, 3 * L + pb.U, c.C},
      {"HO0", sb.HO[0], L, c.Hp}, {"HO1", sb.HO[1], L, c.Hp}, {"HO2", sb.HO[2], L, c.Hp}, {"HO3", sb.HO[3], L, c.Hp},
      {"HOd0", sb.HOd[0], L, c.Hp}, {"HOd1", sb.HOd[1], L, c.Hp}, {"HOd2", sb.HOd[2], L, c.Hp}, {"HOd3", sb.HOd[3], L, c.Hp},
      {"P", sb.P, L, c.Hp}, {"HR0", sb.HR[0], L, c.Hp}, {"HR1", sb.HR[1], L, c.Hp}, {"HR2", sb.HR[2], L, c.Hp},
      {"HR3", sb.HR[3], L, c.Hp}};
  for (const Ent& t : tab)
    if (strcmp(t.n, name) == 0) {
      *ptr = t.p;
      if (rows) *rows = t.r;
      if (ld) *ld = t.l;
      return t.p ? NAR_OK : NAR_ERR_INVALID;
    }
  return NAR_ERR_INVALID;
}
