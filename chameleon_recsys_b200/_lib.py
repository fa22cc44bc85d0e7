"""ctypes binding of libnar_b200.so (include/nar_b200.h).  There is no fallback: if the
library is missing or no sm_90 device is present, loading / ctx creation raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libnar_b200.so')

NAR_MAX_SEGMENTS = 24
NAR_MAX_SRC = 16
NAR_MAX_COLS = 1024

ACT_NONE, ACT_LEAKY, ACT_TANH = 0, 1, 2


class NarError(RuntimeError):
    pass


class Segment(C.Structure):
    _fields_ = [('kind', C.c_int32), ('col', C.c_int32), ('width', C.c_int32), ('card', C.c_int32),
                ('src', C.c_int32), ('ld', C.c_int32), ('table', C.c_void_p), ('grad', C.c_void_p)]


class FeaturePlanC(C.Structure):
    _fields_ = [('n_segments', C.c_int32), ('row_ld', C.c_int32),
                ('seg', Segment * NAR_MAX_SEGMENTS),
                ('ctx_int', C.c_void_p * NAR_MAX_SRC),
                ('ctx_float', C.c_void_p * NAR_MAX_SRC),
                ('meta', C.c_void_p * NAR_MAX_SRC),
                ('created_at_ts', C.c_void_p), ('pop_norm', C.c_void_p),
                ('gamma', C.c_void_p), ('beta', C.c_void_p), ('stats', C.c_void_p),
                ('log_base_recency', C.c_float), ('log_base_novelty', C.c_float),
                ('n_narrow', C.c_int32), ('narrow_begin', C.c_int32 * 4), ('narrow_end', C.c_int32 * 4),
                ('col_seg', C.c_uint8 * NAR_MAX_COLS)]


class RowLayout(C.Structure):
    _fields_ = [('n_rows', C.c_int64), ('n_input', C.c_int64), ('n_cand', C.c_int64), ('n_positive', C.c_int64),
                ('n_full', C.c_int64), ('ctx_col0', C.c_int64)]


NAR_MAX_LAYERS = 4


class ModelCfg(C.Structure):
    _fields_ = [('num_items', C.c_int64), ('C', C.c_int64), ('Hp', C.c_int64), ('Fp', C.c_int64), ('ctx_col0', C.c_int64),
                ('layers', C.c_int32), ('rnn_cell', C.c_int32), ('ranking', C.c_int32),
                ('fwd_precision', C.c_int32), ('bwd_precision', C.c_int32), ('dedup', C.c_int32), ('use_aux_stream', C.c_int32),
                ('keep_prob', C.c_float), ('novelty_reg_factor', C.c_float), ('dropout_seed', C.c_uint64),
                ('K', C.c_int64), ('n_from_buffer', C.c_int64), ('buf_len', C.c_int64), ('n_norm', C.c_int64),
                ('inv_temperature', C.c_float), ('reg_l2', C.c_float), ('lr', C.c_float), ('beta1', C.c_float),
                ('beta2', C.c_float), ('eps', C.c_float),
                ('sampler_seed', C.c_uint64), ('world', C.c_int32), ('rank', C.c_int32),
                ('params', C.c_void_p), ('params_lo', C.c_void_p), ('grads', C.c_void_p), ('adam_m', C.c_void_p),
                ('adam_v', C.c_void_p), ('n_params', C.c_int64), ('reg_end', C.c_int64),
                ('off_W1', C.c_int64), ('off_b1', C.c_int64), ('off_W2', C.c_int64), ('off_b2', C.c_int64),
                ('off_W3', C.c_int64), ('off_b3', C.c_int64), ('off_W4', C.c_int64), ('off_b4', C.c_int64),
                ('off_gamma', C.c_int64), ('off_beta', C.c_int64),
                ('off_M', C.c_int64 * 4), ('off_c', C.c_int64 * 4), ('ld_M', C.c_int64 * 4),
                ('off_Wx', C.c_int64 * NAR_MAX_LAYERS), ('off_Wh', C.c_int64 * NAR_MAX_LAYERS), ('off_rb', C.c_int64 * NAR_MAX_LAYERS),
                ('off_Whc', C.c_int64 * NAR_MAX_LAYERS),
                ('plan', FeaturePlanC)]


class StepIO(C.Structure):
    _fields_ = [('B', C.c_int64), ('Bg', C.c_int64), ('T', C.c_int64), ('sess0', C.c_int64), ('L', C.c_int64),
                ('L_global', C.c_int64), ('L_cap', C.c_int64), ('global_step', C.c_int64),
                ('sampler_step', C.c_uint32), ('train', C.c_int32),
                ('all_items', C.c_void_p), ('event_ts', C.c_void_p), ('item_clicked', C.c_void_p), ('label_next', C.c_void_p),
                ('buffer', C.c_void_p), ('max_ts', C.c_void_p), ('pop_norm', C.c_void_p),
                ('ctx_int', C.c_void_p * NAR_MAX_SRC), ('ctx_float', C.c_void_p * NAR_MAX_SRC),
                ('pos_idx', C.c_void_p), ('sess_off', C.c_void_p),
                ('prep_ws', C.c_void_p), ('prep_ws_bytes', C.c_int64), ('ws', C.c_void_p), ('ws_bytes', C.c_int64),
                ('loss', C.c_void_p)]


class NoveltyReg(C.Structure):
    _fields_ = [('factor', C.c_float), ('log_base', C.c_float), ('pop_norm', C.c_void_p), ('cand_ids', C.c_void_p),
                ('loss_nov', C.c_void_p)]


class GemmEpilogue(C.Structure):
    _fields_ = [('bias', C.c_void_p), ('act', C.c_int32), ('dact', C.c_int32), ('aux', C.c_void_p),
                ('ld_aux', C.c_int64), ('accumulate', C.c_int32), ('split_k', C.c_int32),
                ('precision', C.c_int32), ('b_lo', C.c_void_p), ('b_bf16', C.c_void_p), ('ld_bf16', C.c_int64),
                ('a_scale', C.c_void_p), ('ld_a_scale', C.c_int64), ('a_scale_group', C.c_int64),
                ('pred', C.c_void_p), ('d_pred', C.c_void_p), ('ld_pred', C.c_int64), ('pred_group', C.c_int64),
                ('d_bias', C.c_void_p), ('car_pp', C.c_void_p), ('car_pc', C.c_void_p), ('car_pi', C.c_void_p), ('car_pos_idx', C.c_void_p),
                ('car_neg_uidx', C.c_void_p), ('car_dpp', C.c_void_p), ('car_dpc', C.c_void_p), ('car_dpi', C.c_void_p),
                ('ld_car', C.c_int64), ('car_k', C.c_int64)]


_lib: Optional[C.CDLL] = None

i64, i32, f32, vp, u64, u32 = C.c_int64, C.c_int32, C.c_float, C.c_void_p, C.c_uint64, C.c_uint32

_SIGNATURES = {
    'nar_abi_version': (C.c_int, []),
    'nar_abi_struct_size': (C.c_int, [C.c_int]),
    'nar_status_string': (C.c_char_p, [C.c_int]),
    'nar_ctx_create': (C.c_int, [C.c_int, C.POINTER(vp)]),
    'nar_ctx_destroy': (C.c_int, [vp]),
    'nar_gather_features': (C.c_int, [vp, C.POINTER(FeaturePlanC), vp, vp, C.POINTER(RowLayout), vp, vp, vp, vp]),
    'nar_gather_features_bwd': (C.c_int, [vp, C.POINTER(FeaturePlanC), vp, vp, C.POINTER(RowLayout), vp, vp, vp, vp, vp, vp]),
    'nar_build_base_rows': (C.c_int, [vp, i64, vp, vp, vp, vp, i64, vp, i64, vp, vp, vp]),
    'nar_sample_negatives_uidx': (C.c_int, [vp, vp, i64, i64, i64, i64, vp, i64, i64, i64, u64, u32, vp, vp,
                                            C.POINTER(vp), C.POINTER(vp), vp, i64, vp]),
    'nar_car_combine': (C.c_int, [vp, vp, vp, vp, vp, i64, i64, i64, C.c_int, vp, vp]),
    'nar_car_combine_t': (C.c_int, [vp, vp, vp, vp, vp, i64, i64, i64, C.c_int, vp, i64, vp]),
    'nar_engine_create': (C.c_int, [vp, C.POINTER(ModelCfg), C.POINTER(vp)]),
    'nar_engine_destroy': (C.c_int, [vp]),
    'nar_engine_update_cfg': (C.c_int, [vp, C.POINTER(ModelCfg)]),
    'nar_engine_workspace_bytes': (C.c_int, [vp, i64, i64, i64, i64, i32, C.POINTER(i64), C.POINTER(i64)]),
    'nar_engine_prepare': (C.c_int, [vp, C.POINTER(StepIO), vp]),
    'nar_engine_step': (C.c_int, [vp, C.POINTER(StepIO), vp]),
    'nar_engine_apply': (C.c_int, [vp, C.POINTER(StepIO), vp]),
    'nar_engine_refresh': (C.c_int, [vp, vp]),
    'nar_engine_buffer': (C.c_int, [vp, C.POINTER(StepIO), C.c_char_p, C.POINTER(vp), C.POINTER(i64), C.POINTER(i64)]),
    'nar_engine_launch_count': (i64, [vp]),
    'nar_build_rows': (C.c_int, [vp, i64, vp, vp, vp, i64, vp, vp, vp]),
    'nar_feature_stats': (C.c_int, [vp, vp, i64, i64, vp, vp, vp, f32, f32, vp, vp, i64, i64, i64, vp, vp, vp]),
    'nar_gather_rows_f32': (C.c_int, [vp, i64, i64, C.c_int, vp, i64, vp, i64, vp]),
    'nar_scatter_add_rows_f32': (C.c_int, [vp, i64, i64, C.c_int, vp, i64, vp, i64, vp]),
    'nar_gemm_tf32': (C.c_int, [vp, i64, i64, i64, vp, i64, C.c_int, vp, i64, C.c_int, vp, i64,
                                C.POINTER(GemmEpilogue), vp]),
    'nar_gemm_tf32_dt': (C.c_int, [vp, i64, i64, i64, vp, i64, C.c_int, vp, i64, C.c_int, vp, i64,
                                   C.POINTER(GemmEpilogue), vp]),
    'nar_pack_bf16x3': (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int, vp, vp]),
    'nar_ugrnn_fwd': (C.c_int, [vp, vp, vp, vp, i64, i64, vp, vp, vp, vp]),
    'nar_ugrnn_bwd': (C.c_int, [vp, vp, vp, vp, vp, vp, vp, i64, i64, vp, vp, vp]),
    'nar_gru_fwd': (C.c_int, [vp, vp, vp, vp, vp, i64, i64, vp, vp, vp, vp, vp, vp]),
    'nar_gru_bwd': (C.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, i64, vp, vp, vp]),
    'nar_lstm_fwd': (C.c_int, [vp, vp, vp, vp, i64, i64, vp, vp, vp]),
    'nar_lstm_bwd': (C.c_int, [vp, vp, vp, vp, vp, vp, vp, i64, i64, vp, vp, vp]),
    'nar_sample_negatives_workspace': (C.c_int, [i64, i64, i64, i64, C.POINTER(i64)]),
    'nar_sample_negatives': (C.c_int, [vp, vp, i64, i64, i64, i64, vp, i64, i64, i64, u64, u32, vp, vp, i64, vp]),
    'nar_mul_pred': (C.c_int, [vp, vp, i64, i64, i64, vp, vp]),
    'nar_mul_pred_bwd': (C.c_int, [vp, vp, vp, i64, i64, i64, C.c_int, vp, vp, vp]),
    'nar_score_softmax_ce': (C.c_int, [vp, i64, i64, vp, i64, vp, i64, i64, f32, f32, vp, vp, vp, vp, vp, C.POINTER(NoveltyReg), vp]),
    'nar_cosine_softmax_ce': (C.c_int, [vp, vp, i64, i64, i64, f32, f32, vp, vp, vp, vp, C.POINTER(NoveltyReg), vp]),
    'nar_dropout_rows': (C.c_int, [vp, vp, i64, i64, i64, vp, i64, i64, i64, C.c_int, f32, u64, u32, vp]),
    'nar_rank_candidates': (C.c_int, [vp, vp, i64, i64, i32, vp, vp, vp, vp]),
    'nar_car_combine_grid': (C.c_int, [vp, vp, i64, i64, i64, C.c_int, vp, vp]),
    'nar_topn_candidates': (C.c_int, [vp, vp, i64, i64, i32, vp, vp, i64, vp, vp, vp, vp]),
    'nar_engine_recommend_workspace_bytes': (C.c_int, [vp, i64, i64, i64, i32, i64, C.POINTER(i64), C.POINTER(i64),
                                                       C.POINTER(i64)]),
    'nar_engine_recommend': (C.c_int, [vp, C.POINTER(StepIO), vp, vp, i64, vp, i64, i32, i32, i64, i64, vp, vp, vp, vp]),
    'nar_rank_labels': (C.c_int, [vp, vp, i64, i64, vp, vp, vp, i64, i32, vp, vp, vp]),
    'nar_engine_rank_labels': (C.c_int, [vp, C.POINTER(StepIO), vp, i64, i32, i64, i64, vp, vp, vp]),
    'nar_host_state_update': (C.c_int, [vp, i64, vp, vp, i64, i64, vp, vp, vp, vp, i64, C.c_double]),
    'nar_host_state_update_batch': (C.c_int, [vp, i64, vp, vp, vp, i64, i64, i64, vp, vp, vp, vp, vp, i64, C.c_double]),
    'nar_state_update': (C.c_int, [vp, vp, i64, vp, vp, i64, i64, i64, vp, vp, vp, vp, vp, vp, i64, C.c_double, vp, vp]),
    'nar_colsum_add': (C.c_int, [vp, i64, i64, i64, vp, vp]),
    'nar_act_bwd': (C.c_int, [vp, vp, i64, C.c_int, vp, vp]),
    'nar_l2_loss_add': (C.c_int, [vp, i64, f32, vp, vp]),
    'nar_transpose_f32': (C.c_int, [vp, i64, i64, i64, vp, i64, vp]),
    'nar_adam_tf': (C.c_int, [vp, vp, vp, vp, i64, i64, f32, f32, f32, f32, f32, i64, vp, vp]),
    'nar_tf32_lo': (C.c_int, [vp, i64, vp, vp]),
    'nar_baselines_clear': (C.c_int, [vp, vp, vp, vp, i64, vp]),
    'nar_baselines_rehash': (C.c_int, [vp, vp, vp, vp, i64, vp, vp, vp, vp, i64, vp, vp]),
    'nar_baselines_update': (C.c_int, [vp, vp, vp, vp, i64, vp, vp, i64, i64, i64, i32, i64, vp, vp]),
    'nar_baselines_buffer_hist': (C.c_int, [vp, i64, i64, vp, vp, vp, vp]),
    'nar_baselines_row_norms': (C.c_int, [vp, i64, i64, i64, vp, vp]),
    'nar_baselines_score': (C.c_int, [vp, vp, vp, vp, i64, vp, vp, vp, i64, i64, i64, vp, vp, vp, vp, i64, i64, vp, i64,
                                      C.c_double, C.c_double, i32, i32, vp, vp, vp, vp, vp]),
    'nar_sknn_update': (C.c_int, [vp, vp, vp, i64, i64, i64, i64, vp, vp, vp, vp, vp, i64, i64, i64, vp, vp]),
    'nar_sknn_score': (C.c_int, [vp, vp, vp, i64, i64, i64, i64, vp, vp, vp, i64, i64, i64, i64, i64, i64, i32, i32, i32,
                                 vp, vp, vp, vp, vp]),
    'nar_eval_metrics_mark': (C.c_int, [vp, i64, i64, i32, vp, vp, vp]),
    'nar_eval_metrics_lists': (C.c_int, [vp, i64, i64, i64, i64, i64, i64, i32, vp, i64, vp, vp, i64, i64, vp, i64,
                                         C.c_double, vp, vp, vp, vp]),
    'nar_eval_metrics_reduce': (C.c_int, [vp, i64, i64, i64, vp, vp]),
    'nar_eval_metrics_popcount': (C.c_int, [vp, i64, i64, vp, vp]),
    'nar_eval_by_position': (C.c_int, [vp, i64, i64, i64, i64, i64, i64, i32, vp, i64, vp, i64, vp, i64, vp, i64, vp, vp,
                                       i64, vp, vp, vp]),
    'nar_eval_session_logs_layout': (C.c_int, [i64, i64, i64, i32, vp]),
    'nar_eval_session_logs_pack': (C.c_int, [vp, vp, vp, i64, vp, vp, vp, vp, vp, i64, i64, i64, i64, i32, vp, vp]),
}

EXPORTED_SYMBOLS = sorted(_SIGNATURES.keys())


def load() -> C.CDLL:
    """Load the shared library (no GPU needed for this step); raises if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NarError('libnar_b200.so is not built (%s). Run __graft_entry__.build() / '
                       'python -m chameleon_recsys_b200.build ; there is no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.nar_abi_version() != 3:
        raise NarError('ABI version mismatch')
    _lib = lib
    return lib


def check(rc: int, what: str = ''):
    if rc != 0:
        msg = load().nar_status_string(rc)
        raise NarError('%s failed: %d (%s)' % (what or 'libnar_b200 call', rc, msg.decode() if msg else '?'))


class Context:
    """Owns a nar_ctx for one device.  Raises when no sm_90 device is available."""

    def __init__(self, device: int = 0):
        lib = load()
        h = vp()
        check(lib.nar_ctx_create(int(device), C.byref(h)), 'nar_ctx_create')
        self.lib = lib
        self.handle = h
        self.device = device

    def close(self):
        if self.handle:
            self.lib.nar_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
