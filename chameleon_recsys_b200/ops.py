"""torch-tensor wrappers over the C ABI (include/nar_b200.h).  torch is only the container:
allocation, streams, pointers.  Every function launches on torch's current CUDA stream."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import ACT_LEAKY, ACT_NONE, ACT_TANH, Context, FeaturePlanC, GemmEpilogue, NarError, check

_ctx: dict = {}
LAUNCHES = 0          # kernels launched through this module (gpu_launches in bench.py)


def context(device: Optional[int] = None) -> Context:
    if device is None:
        device = torch.cuda.current_device()
    if device not in _ctx:
        _ctx[device] = Context(device)
    return _ctx[device]


_STREAM_OVERRIDE: Optional[int] = None      # raw cudaStream_t the wrappers launch on instead of torch's current stream


class on_stream:
    """``with ops.on_stream(s):`` - every wrapper launches on ``s`` (a torch.cuda.Stream) without touching torch's
    current-stream state (entering ``torch.cuda.stream`` costs ~10 us of host time; the engine switches streams a
    dozen times per step).  Only libnar_b200 launches are redirected - torch ops keep using the current stream."""

    def __init__(self, stream: torch.cuda.Stream):
        self.h = stream.cuda_stream

    def __enter__(self):
        global _STREAM_OVERRIDE
        self.prev = _STREAM_OVERRIDE
        _STREAM_OVERRIDE = self.h
        return self

    def __exit__(self, *exc):
        global _STREAM_OVERRIDE
        _STREAM_OVERRIDE = self.prev
        return False


def _stream() -> C.c_void_p:
    if _STREAM_OVERRIDE is not None:
        return C.c_void_p(_STREAM_OVERRIDE)
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _chk_f32(*ts):
    for t in ts:
        if t is not None:
            assert t.is_cuda and t.dtype == torch.float32, (t.device, t.dtype)


def gemm(A: torch.Tensor, B: torch.Tensor, D: torch.Tensor, M: int, N: int, K: int, *, a_kmajor=True, b_kmajor=True,
         lda=None, ldb=None, ldd=None, bias=None, act=ACT_NONE, dact=ACT_NONE, aux=None, ld_aux=None,
         accumulate=False, split_k=1, precision=3, b_lo=None, b_bf16=None, ld_bf16=0, a_scale=None, a_scale_group=0,
         pred=None, d_pred=None, pred_group=0, d_bias=None, car=None, trans_d=False):
    global LAUNCHES
    LAUNCHES += 1
    """D[M,N] = epilogue(sum_k A(m,k) B(n,k)); see nar_gemm_tf32.  a_scale / pred / d_pred: row strides from the tensors.
    d_bias: += the column sums of D (with pred only).
    car: dict(pp, pc, pi, pos_idx, neg_uidx, dpp, dpc, dpi, k) for the CAR layer-1 backward epilogue (D = None; ld_car from
    pp).  trans_d: D stored transposed, D[n*ldd + m] (nar_gemm_tf32_dt)."""
    _chk_f32(A, B, D, bias, aux, a_scale, pred, d_pred, d_bias)
    lda = A.stride(0) if lda is None else lda
    ldb = (B.stride(0) if B is not None else 0) if ldb is None else ldb
    ldd = (D.stride(0) if D is not None else 0) if ldd is None else ldd
    epi = GemmEpilogue(_p(bias), act, dact, _p(aux), (aux.stride(0) if (aux is not None and ld_aux is None) else (ld_aux or 0)),
                       1 if accumulate else 0, int(split_k), int(precision), _p(b_lo), _p(b_bf16), int(ld_bf16),
                       _p(a_scale), a_scale.stride(0) if a_scale is not None else 0, int(a_scale_group),
                       _p(pred), _p(d_pred), pred.stride(0) if pred is not None else 0, int(pred_group), _p(d_bias))
    if car is not None:
        _chk_f32(car['pp'], car['pc'], car['pi'], car['dpp'], car['dpc'], car['dpi'])
        assert car['pos_idx'].dtype == torch.int32 and car['neg_uidx'].dtype == torch.int32
        for f in ('pp', 'pc', 'pi', 'pos_idx', 'neg_uidx', 'dpp', 'dpc', 'dpi'):
            setattr(epi, 'car_' + f, _p(car[f]))
        epi.ld_car, epi.car_k = car['pp'].stride(0), int(car['k'])
    ctx = context()
    fn = 'nar_gemm_tf32_dt' if trans_d else 'nar_gemm_tf32'
    check(getattr(ctx.lib, fn)(ctx.handle, M, N, K, _p(A), lda, 1 if a_kmajor else 0, _p(B), ldb, 1 if b_kmajor else 0,
                               _p(D), ldd, C.byref(epi), _stream()), fn)


_PACK_SCRATCH: dict = {}


def pack_bf16x3(W: torch.Tensor, K: int, N: int) -> torch.Tensor:
    """bf16x3 plane of W [K, N] (stored [in, out], row stride W.stride(0)) for gemm(precision=4): [N, ceil(K/32)*64] bf16."""
    global LAUNCHES
    LAUNCHES += 1
    ld_out = (K + 31) // 32 * 64
    out = torch.zeros(N, ld_out, dtype=torch.bfloat16, device=W.device)
    dev = W.device.index
    if dev not in _PACK_SCRATCH:
        _PACK_SCRATCH[dev] = torch.zeros(32 * 32, dtype=torch.uint8, device=W.device)
    i32 = lambda v: (C.c_int32 * 1)(v)      # noqa: E731
    check(_lib.load().nar_pack_bf16x3((C.c_void_p * 1)(W.data_ptr()), (C.c_void_p * 1)(out.data_ptr()), i32(K), i32(N),
                                      i32(W.stride(0)), i32(ld_out), 1, _p(_PACK_SCRATCH[dev]), _stream()), 'nar_pack_bf16x3')
    return out


def gather_rows(table: torch.Tensor, ids: torch.Tensor, out: torch.Tensor, width: int):
    global LAUNCHES
    LAUNCHES += 1
    _chk_f32(table, out)
    assert ids.dtype == torch.int64
    lib = _lib.load()
    check(lib.nar_gather_rows_f32(_p(table), table.shape[0], table.stride(0), width, _p(ids), ids.numel(), _p(out),
                                  out.stride(0), _stream()), 'nar_gather_rows_f32')


def scatter_add_rows(table: torch.Tensor, ids: torch.Tensor, src: torch.Tensor, width: int):
    global LAUNCHES
    LAUNCHES += 1
    _chk_f32(table, src)
    lib = _lib.load()
    check(lib.nar_scatter_add_rows_f32(_p(table), table.shape[0], table.stride(0), width, _p(ids), ids.numel(), _p(src),
                                       src.stride(0), _stream()), 'nar_scatter_add_rows_f32')


def row_layout(n_rows, n_input, n_cand, n_positive=0, n_full=None, ctx_col0=0) -> _lib.RowLayout:
    return _lib.RowLayout(n_rows, n_input, n_cand, n_positive, n_rows if n_full is None else n_full, ctx_col0)


def gather_features(plan: FeaturePlanC, row_pos, row_item, rows: _lib.RowLayout, event_ts, max_ts, out):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_gather_features(ctx.handle, C.byref(plan), _p(row_pos), _p(row_item), C.byref(rows),
                                      _p(event_ts), _p(max_ts), _p(out), _stream()), 'nar_gather_features')


def gather_features_bwd(plan: FeaturePlanC, row_pos, row_item, rows: _lib.RowLayout, event_ts, max_ts, d_out, d_gamma, d_beta):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_gather_features_bwd(ctx.handle, C.byref(plan), _p(row_pos), _p(row_item), C.byref(rows),
                                          _p(event_ts), _p(max_ts), _p(d_out), _p(d_gamma), _p(d_beta), _stream()),
          'nar_gather_features_bwd')


def build_rows(pos_idx, L, item_clicked, label_next, negatives, K, row_pos, row_item):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_build_rows(_p(pos_idx), L, _p(item_clicked), _p(label_next), _p(negatives), K, _p(row_pos),
                                     _p(row_item), _stream()), 'nar_build_rows')


def build_base_rows(pos_idx, L, item_clicked, label_next, unique_items, n_unique, U, neg_uidx, K, base_pos, base_item):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_build_base_rows(_p(pos_idx), L, _p(item_clicked), _p(label_next), _p(unique_items), _p(n_unique), U,
                                          _p(neg_uidx), K, _p(base_pos), _p(base_item), _stream()), 'nar_build_base_rows')


def feature_stats(buffer, n_norm, created_at_ts, pop_norm, max_ts, log_base_rec, log_base_nov, row_pos, row_item,
                  n_rows, n_input, n_cand, event_ts, stats):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_feature_stats(ctx.handle, _p(buffer), buffer.numel(), n_norm, _p(created_at_ts), _p(pop_norm),
                                    _p(max_ts), log_base_rec, log_base_nov, _p(row_pos), _p(row_item), n_rows, n_input,
                                    n_cand, _p(event_ts), _p(stats), _stream()), 'nar_feature_stats')


def ugrnn_fwd(gx, Wh, sess_off, B, Hp, h_out, gate, cand):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_ugrnn_fwd(ctx.handle, _p(gx), _p(Wh), _p(sess_off), B, Hp, _p(h_out), _p(gate), _p(cand), _stream()),
          'nar_ugrnn_fwd')


def ugrnn_bwd(d_hout, h_out, gate, cand, WhT, sess_off, B, Hp, d_gx, h_prev):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_ugrnn_bwd(ctx.handle, _p(d_hout), _p(h_out), _p(gate), _p(cand), _p(WhT), _p(sess_off), B, Hp,
                                _p(d_gx), _p(h_prev), _stream()), 'nar_ugrnn_bwd')


def gru_fwd(gx, Whg, Whc, sess_off, B, Hp, h_out, r_out, u_out, c_out, rh_out):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_gru_fwd(ctx.handle, _p(gx), _p(Whg), _p(Whc), _p(sess_off), B, Hp, _p(h_out), _p(r_out), _p(u_out),
                              _p(c_out), _p(rh_out), _stream()), 'nar_gru_fwd')


def gru_bwd(d_hout, h_out, r_out, u_out, c_out, WhgT, WhcT, sess_off, B, Hp, d_gx, h_prev):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_gru_bwd(ctx.handle, _p(d_hout), _p(h_out), _p(r_out), _p(u_out), _p(c_out), _p(WhgT), _p(WhcT),
                              _p(sess_off), B, Hp, _p(d_gx), _p(h_prev), _stream()), 'nar_gru_bwd')


def lstm_fwd(gx, Wh, sess_off, B, Hp, h_out, c_out):
    """gx [L,4Hp] (pre-activations i | j | f | o of the input) is overwritten with the activated gates."""
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_lstm_fwd(ctx.handle, _p(gx), _p(Wh), _p(sess_off), B, Hp, _p(h_out), _p(c_out), _stream()), 'nar_lstm_fwd')


def lstm_bwd(d_hout, h_out, c_out, act, WhT, sess_off, B, Hp, d_gx, h_prev):
    global LAUNCHES
    LAUNCHES += 1
    ctx = context()
    check(ctx.lib.nar_lstm_bwd(ctx.handle, _p(d_hout), _p(h_out), _p(c_out), _p(act), _p(WhT), _p(sess_off), B, Hp, _p(d_gx),
                               _p(h_prev), _stream()), 'nar_lstm_bwd')


def sample_negatives_workspace(Bg, T1, buf_len, K) -> int:
    lib = _lib.load()
    n = C.c_int64(0)
    check(lib.nar_sample_negatives_workspace(Bg, T1, buf_len, K, C.byref(n)), 'nar_sample_negatives_workspace')
    return int(n.value)


def sample_negatives(all_items_global, sess0, B, buffer, K, n_from_buffer, seed, step, out, workspace):
    global LAUNCHES
    LAUNCHES += 2 if B > 0 else 1
    ctx = context()
    Bg, T1 = all_items_global.shape
    check(ctx.lib.nar_sample_negatives(ctx.handle, _p(all_items_global), Bg, T1, sess0, B, _p(buffer), buffer.numel(), K,
                                       n_from_buffer, C.c_uint64(seed & 0xFFFFFFFFFFFFFFFF), C.c_uint32(step & 0xFFFFFFFF),
                                       _p(out), _p(workspace), workspace.numel() * workspace.element_size(), _stream()),
          'nar_sample_negatives')


def mul_pred(cand, pred, n_pos, n_cand, Cdim, prod):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_mul_pred(_p(cand), _p(pred), n_pos, n_cand, Cdim, _p(prod), _stream()), 'nar_mul_pred')


def mul_pred_bwd(d_prod, cand, pred, n_pos, n_cand, Cdim, d_cand, d_pred, cand_act=ACT_NONE):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_mul_pred_bwd(_p(d_prod), _p(cand), _p(pred), n_pos, n_cand, Cdim, cand_act, _p(d_cand), _p(d_pred), _stream()),
          'nar_mul_pred_bwd')


def novelty_reg(factor, log_base, pop_norm, cand_ids, loss_nov) -> _lib.NoveltyReg:
    return _lib.NoveltyReg(factor, log_base, pop_norm.data_ptr(), cand_ids.data_ptr(), loss_nov.data_ptr())


def score_softmax_ce(z3, ld_z, width, m4, ld_m4, c4, n_pos, n_cand, inv_temp, inv_count, logits, loss_sum, d_z3, d_m4, d_c4, nov=None):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_score_softmax_ce(_p(z3), ld_z, width, _p(m4), ld_m4, _p(c4), n_pos, n_cand, inv_temp, inv_count,
                                           _p(logits), _p(loss_sum), _p(d_z3), _p(d_m4), _p(d_c4),
                                           C.byref(nov) if nov is not None else None, _stream()),
          'nar_score_softmax_ce')


def cosine_softmax_ce(cand, pred, n_pos, n_cand, Cdim, inv_temp, inv_count, logits, loss_sum, d_cand, d_pred, nov=None):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_cosine_softmax_ce(_p(cand), _p(pred), n_pos, n_cand, Cdim, inv_temp, inv_count, _p(logits),
                                            _p(loss_sum), _p(d_cand), _p(d_pred), C.byref(nov) if nov is not None else None,
                                            _stream()), 'nar_cosine_softmax_ce')


def rank_candidates(logits, cand_ids, n_pos, n_cand, top_n, pred_ids, pred_probs, metrics):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_rank_candidates(_p(logits), _p(cand_ids), n_pos, n_cand, top_n, _p(pred_ids), _p(pred_probs),
                                          _p(metrics), _stream()), 'nar_rank_candidates')


def car_combine_grid(PC, PI, Q, Nc, Cdim, H1, act=ACT_LEAKY):
    """H1[q*Nc + j] = act(PC[q] + PI[j])  (nar_car_combine_grid)."""
    global LAUNCHES
    LAUNCHES += 1
    _chk_f32(PC, PI, H1)
    check(_lib.load().nar_car_combine_grid(_p(PC), _p(PI), Q, Nc, Cdim, act, _p(H1), _stream()), 'nar_car_combine_grid')


def topn_candidates(logits, cand_ids, Q, N, top_n, out_ids, out_scores=None, out_probs=None, item_clicked=None, q_pos=None, T=0):
    """Per query row of logits [Q, N]: the top_n candidates (score desc, index asc), their scores and softmax probabilities
    over the non-excluded candidates; ``item_clicked`` [*, T] + ``q_pos`` [Q] (flat b*T+t) exclude each query's own
    clicks item_clicked[b, 0..t]  (nar_topn_candidates)."""
    global LAUNCHES
    LAUNCHES += 1
    _chk_f32(logits, out_scores, out_probs)
    check(_lib.load().nar_topn_candidates(_p(logits), _p(cand_ids), Q, N, int(top_n), _p(item_clicked), _p(q_pos), int(T),
                                          _p(out_ids), _p(out_scores), _p(out_probs), _stream()), 'nar_topn_candidates')


def dropout_rows(src, dst, rows, cols, ld, row_pos, n_input, n_cand, K, tensor_id, keep_prob, seed, step):
    """dst = src * mask / keep_prob with the counter-based masks of oracle/dropout_ref.py (tensor_id 0: feature rows)."""
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_dropout_rows(_p(src), _p(dst), rows, cols, ld, _p(row_pos), n_input, n_cand, K, tensor_id, keep_prob,
                                       C.c_uint64(seed & 0xFFFFFFFFFFFFFFFF), C.c_uint32(step & 0xFFFFFFFF), _stream()),
          'nar_dropout_rows')


def colsum_add(x, rows, cols, ld, out):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_colsum_add(_p(x), rows, cols, ld, _p(out), _stream()), 'nar_colsum_add')


def act_bwd(dy, y, n, act, dx):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_act_bwd(_p(dy), _p(y), n, act, _p(dx), _stream()), 'nar_act_bwd')


def l2_loss_add(x, n, scale, out):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_l2_loss_add(_p(x), n, scale, _p(out), _stream()), 'nar_l2_loss_add')


def transpose(src, rows, cols, ld_src, dst, ld_dst):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_transpose_f32(_p(src), rows, cols, ld_src, _p(dst), ld_dst, _stream()), 'nar_transpose_f32')


def adam_tf(params, grads, m, v, n, reg_end, reg_l2, lr, step, beta1=0.9, beta2=0.999, eps=1e-8, params_lo=None):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_adam_tf(_p(params), _p(grads), _p(m), _p(v), n, reg_end, reg_l2, lr, beta1, beta2, eps, step,
                                  _p(params_lo), _stream()), 'nar_adam_tf')


def tf32_lo(x, n, lo):
    global LAUNCHES
    LAUNCHES += 1
    check(_lib.load().nar_tf32_lo(_p(x), n, _p(lo), _stream()), 'nar_tf32_lo')
