"""Feature plan + parameter layout of the NAR hot path (host side, numpy only).

Two jobs:

1. ``FeaturePlan`` - which columns make up one "user-item feature" row and where each
   segment lives in the *logical* (reference) column order and in the *internal*
   (HBM) column order.  Reference order: nar_model.py:332 (ctx ++ item features),
   nar_model.py:921-994 (metadata ++ ACR ++ item embedding ++ recency ++ novelty),
   nar_model.py:730-773 (one-hot if cardinality <= max_cardinality_for_ohe else embedding).
   Internal order puts the two wide segments (ACR rows, item-embedding rows) first at
   16-byte aligned column offsets so the gather kernel can move them with 128-bit
   loads/stores; the permutation is invisible outside (checkpoints keep logical shapes).

2. ``ParamLayout`` - every trainable variable of SURVEY.md Appendix B with its TF
   variable name, logical shape, initialiser, L2 flag, and its slot in ONE flat fp32
   buffer (params / grads / adam_m / adam_v share offsets).  L2-regularised tensors come
   first so the optimiser kernel can apply ``reg_l2 * w`` by index range.  Padded
   rows/cols (H -> the next of 32, 64, ..., 1024, e.g. 255 -> 256 and 300 -> 512; F -> multiple of 4) hold zeros and
   provably stay zero.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from .hparams import (ARTICLE_REQ_FEATURES, SESSION_REQ_SEQ_FEATURES, get_embedding_size)

# segment kinds (shared with csrc/nar_b200.h : nar_seg_kind)
SEG_CTX_OHE = 0
SEG_CTX_EMBED = 1
SEG_CTX_NUM = 2
SEG_CTX_ZERO = 3
SEG_META_OHE = 4
SEG_META_EMBED = 5
SEG_META_NUM = 6
SEG_ACR = 7
SEG_ITEM_EMB = 8
SEG_RECENCY = 9
SEG_NOVELTY = 10


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


@dataclass
class Segment:
    kind: int
    name: str            # feature name (ctx / metadata) or internal feature name
    width: int           # logical width
    log_col: int         # first column in the reference's concat order
    int_col: int = -1    # first column in the HBM row layout
    card: int = 0        # categorical cardinality
    src: int = -1        # index into ctx-int / ctx-float / metadata arrays
    param: Optional[str] = None   # key of the embedding table in ParamLayout


class FeaturePlan:
    def __init__(self, session_features_config: dict, articles_features_config: dict,
                 internal_features_config: Dict[str, bool], max_cardinality_for_ohe: int,
                 acr_dim: int, num_items: int):
        self.num_items = int(num_items)
        self.acr_dim = int(acr_dim)
        self.item_emb_dim = get_embedding_size(self.num_items)
        self.ctx_int_names: List[str] = []     # int64 [B,T] inputs consumed by the plan
        self.ctx_float_names: List[str] = []   # float32 [B,T] inputs
        self.meta_names: List[str] = []        # int64 [V] metadata arrays (besides created_at_ts)
        segs: List[Segment] = []
        col = 0
        seq_cfg = session_features_config['sequence_features']
        for fname, fc in seq_cfg.items():
            if fname in SESSION_REQ_SEQ_FEATURES:
                continue
            if fc['type'] == 'categorical':
                card = int(fc['cardinality'])
                src = len(self.ctx_int_names)
                self.ctx_int_names.append(fname)
                if card <= max_cardinality_for_ohe:
                    segs.append(Segment(SEG_CTX_OHE, fname, card, col, card=card, src=src))
                    col += card
                else:
                    dim = get_embedding_size(card)
                    segs.append(Segment(SEG_CTX_EMBED, fname, dim, col, card=card, src=src,
                                        param='ctx_emb/' + fname))
                    col += dim
            elif fc['type'] == 'numerical':
                src = len(self.ctx_float_names)
                self.ctx_float_names.append(fname)
                segs.append(Segment(SEG_CTX_NUM, fname, 1, col, src=src))
                col += 1
            else:
                raise Exception('Invalid feature type: {}'.format(fname))
        if col == 0:
            # nar_model.py:323-325: dummy zero tensor so the concat does not break
            segs.append(Segment(SEG_CTX_ZERO, '_dummy_ctx', 1, col))
            col += 1
        self.ctx_width = col
        for fname, fc in articles_features_config.items():
            if fname in ARTICLE_REQ_FEATURES:
                continue
            if fc['type'] == 'categorical':
                card = int(fc['cardinality'])
                src = len(self.meta_names)
                self.meta_names.append(fname)
                if card <= max_cardinality_for_ohe:
                    segs.append(Segment(SEG_META_OHE, fname, card, col, card=card, src=src))
                    col += card
                else:
                    dim = get_embedding_size(card)
                    segs.append(Segment(SEG_META_EMBED, fname, dim, col, card=card, src=src,
                                        param='meta_emb/' + fname))
                    col += dim
            elif fc['type'] == 'numerical':
                src = len(self.meta_names)
                self.meta_names.append(fname)
                segs.append(Segment(SEG_META_NUM, fname, 1, col, src=src))
                col += 1
            else:
                raise Exception('Invalid feature type: {}'.format(fname))
        self.use_acr = bool(internal_features_config.get('article_content_embeddings', False))
        self.use_item_emb = bool(internal_features_config.get('item_clicked_embeddings', False))
        self.use_recency = bool(internal_features_config.get('recency', False))
        self.use_novelty = bool(internal_features_config.get('novelty', False))
        if self.use_acr:
            segs.append(Segment(SEG_ACR, 'acr', self.acr_dim, col)); col += self.acr_dim
        if self.use_item_emb:
            segs.append(Segment(SEG_ITEM_EMB, 'item_emb', self.item_emb_dim, col, card=self.num_items,
                                param='items_embedding')); col += self.item_emb_dim
        if self.use_recency:
            segs.append(Segment(SEG_RECENCY, 'recency', 1, col)); col += 1
        if self.use_novelty:
            segs.append(Segment(SEG_NOVELTY, 'novelty', 1, col)); col += 1
        self.segments = segs
        self.F = col
        # ---- internal (HBM) order: ITEM side first - the wide segments at 4-float aligned offsets, then the narrow
        # item segments (metadata, recency, novelty) - and the user-CONTEXT segments last, starting at the 4-float
        # aligned column ctx_col0: the item half [0, ctx_col0) and the context half [ctx_col0, Fp) of a row (and the
        # matching row blocks of W1) can then be used as separate, TMA-aligned GEMM operands (per-unique-id CAR layer 1)
        ctx_kinds = (SEG_CTX_OHE, SEG_CTX_EMBED, SEG_CTX_NUM, SEG_CTX_ZERO)
        icol = 0
        for s in segs:
            if s.kind in (SEG_ACR, SEG_ITEM_EMB):
                icol = round_up(icol, 4)
                s.int_col = icol
                icol += s.width
        for s in segs:
            if s.kind not in (SEG_ACR, SEG_ITEM_EMB) and s.kind not in ctx_kinds:
                s.int_col = icol
                icol += s.width
        icol = round_up(icol, 4)
        self.ctx_col0 = icol
        for s in segs:
            if s.kind in ctx_kinds:
                s.int_col = icol
                icol += s.width
        self.F_int = icol
        self.Fp = round_up(icol, 4)
        # int2log[c] = logical column of internal column c (or -1 for padding)
        self.int2log = np.full(self.Fp, -1, dtype=np.int64)
        for s in segs:
            self.int2log[s.int_col:s.int_col + s.width] = np.arange(s.log_col, s.log_col + s.width)
        self.log2int = np.zeros(self.F, dtype=np.int64)
        valid = self.int2log >= 0
        self.log2int[self.int2log[valid]] = np.nonzero(valid)[0]

    @property
    def acr_ld(self) -> int:
        return round_up(self.acr_dim, 4)

    @property
    def item_emb_ld(self) -> int:
        return round_up(self.item_emb_dim, 4)


# ---------------------------------------------------------------------------
# Parameters
# ---------------------------------------------------------------------------
INIT_XAVIER = 'xavier'                 # tf.contrib.layers.xavier_initializer (scope default nar_model.py:210)
INIT_VAR_SCALING = 'variance_scaling'  # contrib variance_scaling_initializer(): trunc normal, std sqrt(1.3*2/fan_in)
INIT_LECUN_UNIFORM = 'lecun_uniform'   # tf.initializers.lecun_uniform: U(+-sqrt(3/fan_in))
INIT_ZEROS = 'zeros'
INIT_ONES = 'ones'

# padded hidden sizes Hp the session-cell recurrence kernels accept (csrc/rnn.cu shape_ok)
HP_SIZES = (32, 64, 128, 256, 512, 1024)


@dataclass
class ParamTensor:
    key: str                      # short key used by kernels ('W1', 'rnn0/Wx' ...)
    tf_name: str                  # TF variable name (SURVEY.md Appendix B)
    logical_shape: Tuple[int, ...]
    init: str
    reg: bool
    rows: int                     # internal rows
    ld: int                       # internal leading dimension (floats)
    offset: int = 0               # offset in the flat buffer (floats)
    # how the logical tensor maps into the internal one
    row_map: Optional[np.ndarray] = None   # internal row index for each logical row
    col_map: Optional[np.ndarray] = None   # internal col index for each logical col
    part_rows: Optional[Tuple[int, int]] = None   # rows of the logical tensor this one holds (RNN kernel split)
    into: Optional[str] = None    # key of the tensor whose storage this one fills (same rows and ld, none of its own)

    @property
    def size(self) -> int:
        return self.rows * self.ld


class ParamLayout:
    """Flat-buffer layout.  ``tensors`` in buffer order; regularised ones first."""

    def __init__(self, plan: FeaturePlan, CAR_embedding_size: int, rnn_units: int, rnn_num_layers: int,
                 rnn_cell: str = 'ugrnn', residual: bool = False):
        self.plan = plan
        self.rnn_cell = rnn_cell
        self.residual = bool(residual)
        C = int(CAR_embedding_size)
        H = int(rnn_units)
        self.C, self.H, self.layers = C, H, int(rnn_num_layers)
        self.Cp = round_up(C, 4)
        # the recurrence kernels (csrc/rnn.cu) run Hp = 32, 64, ..., 1024: the state is padded to the smallest of those
        if not 1 <= H <= HP_SIZES[-1]:
            raise ValueError('rnn_units=%d: must be in [1, %d]' % (H, HP_SIZES[-1]))
        self.Hp = min(s for s in HP_SIZES if s >= H)
        if self.Cp != C:
            raise ValueError('CAR_embedding_size must be a multiple of 4')
        Hp = self.Hp
        F, Fp = plan.F, plan.Fp
        reg: List[ParamTensor] = []
        noreg: List[ParamTensor] = []
        # --- small categorical embeddings (nar_model.py:736-742) ---
        for s in plan.segments:
            if s.kind in (1, 5):   # CTX_EMBED, META_EMBED
                scope = 'main/user_items_contextual_features/'
                tf_name = scope + ('features/' if s.kind == 1 else 'item_features/features/') + \
                    '{}_cat_embedding/{}_embedding'.format(s.name, s.name)
                reg.append(ParamTensor(s.param, tf_name, (s.card, s.width), INIT_XAVIER, True,
                                       rows=s.card, ld=s.width))
        if plan.use_item_emb:
            # nar_model.py:911-919
            reg.append(ParamTensor('items_embedding',
                                   'main/user_items_contextual_features/item_features/item_cat_embedding/items_embedding',
                                   (plan.num_items, plan.item_emb_dim), INIT_XAVIER, True,
                                   rows=plan.num_items, ld=plan.item_emb_ld,
                                   col_map=np.arange(plan.item_emb_dim)))
        # nar_model.py:887-907
        scs = 'main/user_items_contextual_features/input_features_center_scale/'
        reg.append(ParamTensor('gamma', scs + 'gamma_scale', (F,), INIT_ONES, True, rows=1, ld=Fp,
                               col_map=plan.log2int.copy()))
        reg.append(ParamTensor('beta', scs + 'beta_center', (F,), INIT_ZEROS, True, rows=1, ld=Fp,
                               col_map=plan.log2int.copy()))
        # nar_model.py:374-388
        reg.append(ParamTensor('W1', 'main/CAR/PreCAR_representation/kernel', (F, C), INIT_VAR_SCALING, True,
                               rows=Fp, ld=C, row_map=plan.log2int.copy()))
        noreg.append(ParamTensor('b1', 'main/CAR/PreCAR_representation/bias', (C,), INIT_ZEROS, False, rows=1, ld=C))
        reg.append(ParamTensor('W2', 'main/CAR/CAR_representation/kernel', (C, C), INIT_XAVIER, True, rows=C, ld=C))
        noreg.append(ParamTensor('b2', 'main/CAR/CAR_representation/bias', (C,), INIT_ZEROS, False, rows=1, ld=C))
        # nar_model.py:1308-1342, not regularised.  Per cell: its TF scope, then per TF kernel [in+H, n*H] and bias [n*H] the
        # prefix, the n column blocks, the bias initialiser and the key of the recurrent block:
        #   tf.contrib.rnn.UGRNNCell    kernel (gate | candidate)
        #   tf.nn.rnn_cell.GRUCell      gates/kernel (r | u), bias 1.0; candidate/kernel (:1315, commented alternative)
        #   tf.nn.rnn_cell.LSTMCell     kernel (i | j | f | o); forget_bias 1.0 is a constant inside the cell (:1316, idem)
        # Every column block goes to an Hp-wide block.  The input rows of a layer's kernels fill one Wx [in, G*Hp] and its
        # biases one b [G*Hp] (G = 2, 3 or 4: one input projection per layer).  The recurrent rows of each kernel are a block
        # of their own: the GRU's candidate multiplies r*h, not h, so its Whc is a separate product.
        cells = {'ugrnn': ('ugrnn_cell/', [('', 2, INIT_ZEROS, 'Wh')]),
                 'gru': ('gru_cell/', [('gates/', 2, INIT_ONES, 'Wh'), ('candidate/', 1, INIT_ZEROS, 'Whc')]),
                 'lstm': ('lstm_cell/', [('', 4, INIT_ZEROS, 'Wh')])}
        if rnn_cell not in cells:
            raise ValueError('rnn_cell=%r: one of %s' % (rnn_cell, sorted(cells)))
        scope, kernels = cells[rnn_cell]
        G = sum(n for _, n, _, _ in kernels)
        if self.residual:
            # build_rnn(residual_connections=True) (nar_model.py:1319-1323): layer 0 is InputProjectionWrapper(ResidualWrapper(
            # cell), H), whose scope holds the projection's _Linear kernel [C, H] (the scope's xavier) and bias [H] (zeros)
            # and the cell's variables; layers > 0 keep their names (ResidualWrapper opens no scope).  DESIGN.md section 15
            proj = 'main/RNN/rnn/multi_rnn_cell/cell_0/input_projection_wrapper/'
            noreg.append(ParamTensor('rnn0/Wp', proj + 'kernel', (C, H), INIT_XAVIER, False, rows=C, ld=Hp,
                                     col_map=np.arange(H)))
            noreg.append(ParamTensor('rnn0/bp', proj + 'bias', (H,), INIT_ZEROS, False, rows=1, ld=Hp, col_map=np.arange(H)))
        for i in range(self.layers):
            n_in = C if (i == 0 and not self.residual) else H
            n_in_p = C if (i == 0 and not self.residual) else Hp
            base = 'main/RNN/rnn/multi_rnn_cell/cell_{}/'.format(i) + \
                ('input_projection_wrapper/' if (i == 0 and self.residual) else '') + scope
            wx, b = 'rnn%d/Wx' % i, 'rnn%d/b' % i
            g0 = 0
            for prefix, n, b_init, wh in kernels:
                k, cols = base + prefix + 'kernel', np.concatenate([g * Hp + np.arange(H) for g in range(n)])
                noreg.append(ParamTensor(wx, k, (n_in + H, n * H), INIT_XAVIER, False, rows=n_in_p, ld=G * Hp,
                                         col_map=g0 * Hp + cols, part_rows=(0, n_in), row_map=np.arange(n_in),
                                         into=wx if g0 else None))
                noreg.append(ParamTensor('rnn%d/%s' % (i, wh), k, (n_in + H, n * H), INIT_XAVIER, False, rows=Hp, ld=n * Hp,
                                         col_map=cols, part_rows=(n_in, n_in + H), row_map=np.arange(H)))
                noreg.append(ParamTensor(b, base + prefix + 'bias', (n * H,), b_init, False, rows=1, ld=G * Hp,
                                         col_map=g0 * Hp + cols, into=b if g0 else None))
                g0 += n
        # nar_model.py:410-426
        reg.append(ParamTensor('W3', 'main/session_representation/FC1/kernel', (H, 512), INIT_VAR_SCALING, True,
                               rows=Hp, ld=512, row_map=np.arange(H)))
        noreg.append(ParamTensor('b3', 'main/session_representation/FC1/bias', (512,), INIT_ZEROS, False, rows=1, ld=512))
        reg.append(ParamTensor('W4', 'main/session_representation/FC2/kernel', (512, C), INIT_XAVIER, True, rows=512, ld=C))
        noreg.append(ParamTensor('b4', 'main/session_representation/FC2/bias', (C,), INIT_ZEROS, False, rows=1, ld=C))
        # nar_model.py:447-473
        dims = [C, 128, 64, 32, 1]
        for li in range(4):
            init = INIT_LECUN_UNIFORM if li == 3 else INIT_VAR_SCALING
            base = 'main/recommendations_ranking/matching_dense_layer_{}/'.format(li + 1)
            ld = round_up(dims[li + 1], 4)
            reg.append(ParamTensor('M%d' % (li + 1), base + 'kernel', (dims[li], dims[li + 1]), init, True,
                                   rows=dims[li], ld=ld, col_map=np.arange(dims[li + 1])))
            noreg.append(ParamTensor('c%d' % (li + 1), base + 'bias', (dims[li + 1],), INIT_ZEROS, False,
                                     rows=1, ld=ld, col_map=np.arange(dims[li + 1])))
        self.tensors: List[ParamTensor] = reg + noreg
        off = 0
        self.by_key: Dict[str, ParamTensor] = {}
        for t in self.tensors:
            if t.into is not None:
                t.offset = self.by_key[t.into].offset
                continue
            t.offset = off
            off += round_up(t.size, 4)
            if t.reg:
                self.reg_end = off
            self.by_key[t.key] = t
        self.total = off

    # ---- logical <-> internal -------------------------------------------------
    def logical_names(self) -> List[str]:
        seen, out = set(), []
        for t in self.tensors:
            if t.tf_name not in seen:
                seen.add(t.tf_name); out.append(t.tf_name)
        return out

    def to_internal(self, logical: Dict[str, np.ndarray]) -> np.ndarray:
        flat = np.zeros(self.total, dtype=np.float32)
        for t in self.tensors:
            w = np.asarray(logical[t.tf_name], dtype=np.float32)
            assert tuple(w.shape) == tuple(t.logical_shape), (t.tf_name, w.shape, t.logical_shape)
            if w.ndim == 1:
                w = w[None, :]
            if t.part_rows is not None:
                w = w[t.part_rows[0]:t.part_rows[1]]
            dst = flat[t.offset:t.offset + t.size].reshape(t.rows, t.ld)
            rmap = t.row_map if t.row_map is not None else np.arange(w.shape[0])
            cmap = t.col_map if t.col_map is not None else np.arange(w.shape[1])
            dst[np.ix_(rmap, cmap)] = w
        return flat

    def to_logical(self, flat: np.ndarray) -> Dict[str, np.ndarray]:
        out: Dict[str, np.ndarray] = {}
        flat = np.asarray(flat)
        for t in self.tensors:
            src = flat[t.offset:t.offset + t.size].reshape(t.rows, t.ld)
            nrows = (t.part_rows[1] - t.part_rows[0]) if t.part_rows is not None else \
                (t.logical_shape[0] if len(t.logical_shape) == 2 else 1)
            ncols = t.logical_shape[-1]
            rmap = t.row_map if t.row_map is not None else np.arange(nrows)
            cmap = t.col_map if t.col_map is not None else np.arange(ncols)
            w = src[np.ix_(rmap, cmap)]
            if t.part_rows is not None:
                if t.tf_name not in out:
                    out[t.tf_name] = np.zeros(t.logical_shape, dtype=flat.dtype)
                out[t.tf_name][t.part_rows[0]:t.part_rows[1]] = w
            elif len(t.logical_shape) == 1:
                out[t.tf_name] = w[0].copy()
            else:
                out[t.tf_name] = w.copy()
        return out

    # ---- initialisation (reference initialisers, numpy RandomState) --------------
    def init_logical(self, seed: int = 42) -> Dict[str, np.ndarray]:
        rs = np.random.RandomState(seed)
        out: Dict[str, np.ndarray] = {}
        for t in self.tensors:
            if t.tf_name in out:
                continue
            shp = t.logical_shape
            if t.init == INIT_ZEROS:
                w = np.zeros(shp, np.float32)
            elif t.init == INIT_ONES:
                w = np.ones(shp, np.float32)
            else:
                fan_in, fan_out = (shp[0], shp[1]) if len(shp) == 2 else (shp[0], shp[0])
                if t.init == INIT_XAVIER:
                    lim = math.sqrt(6.0 / (fan_in + fan_out))
                    w = rs.uniform(-lim, lim, size=shp)
                elif t.init == INIT_LECUN_UNIFORM:
                    lim = math.sqrt(3.0 / fan_in)
                    w = rs.uniform(-lim, lim, size=shp)
                elif t.init == INIT_VAR_SCALING:
                    std = math.sqrt(1.3 * 2.0 / fan_in)
                    w = rs.normal(0.0, 1.0, size=shp)
                    bad = np.abs(w) > 2.0           # truncated normal: redraw beyond 2 sigma
                    while bad.any():
                        w[bad] = rs.normal(0.0, 1.0, size=int(bad.sum()))
                        bad = np.abs(w) > 2.0
                    w = w * std
                else:
                    raise ValueError(t.init)
                w = w.astype(np.float32)
            out[t.tf_name] = w
        return out
