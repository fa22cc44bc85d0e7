"""TEST INFRASTRUCTURE - CPU restatement of the NAR training graph (torch-CPU, fp32 or fp64).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this module; the product path never does and fails loudly without its CUDA
library.

Pinning (SURVEY.md section 8c).  The reference arithmetic lives in TensorFlow 1.12.3 (requirements.txt:5), which
cannot be installed here (Python 3.12, no network), and the reference holds no test, golden vector or fixture for
logits / loss / gradients / Adam.  What this file is checked against:
 (a) outputs of the reference's OWN model code: nar_model.py's NARModuleModel is imported unmodified and its
     constructor executed on an eager stand-in for the TF-1.x API (tests/golden/tf1_shim.py, generator
     tests/golden/make_model_golden.py, fixtures tests/golden/model_golden.npz); tests/test_oracle_reference_model.py
     compares logits, loss, the intermediates the reference exposes, every gradient, the first Adam step, and the
     EVAL ranking / recall@n / MRR@n (train, float32, cold start, novelty regulariser, 2 RNN layers, internal-feature switches, GRU cell substituted, dropout with the
     reference run's masks handed over, eval): 1e-7 in float64.  That pins the WIRING to the reference.  The per-op TF kernel semantics inside the stand-in (moments,
     leaky_relu, UGRNNCell, dynamic_rnn, AdamOptimizer ...) are a restatement of the TF documentation, so "what
     TensorFlow itself would compute" remains unpinned;
 (b) hand-derived known answers (tests/test_oracle.py), finite-difference gradients, invariants from the code;
 (c) the evaluation metrics (HR@n / MRR@n) against the reference's own numpy classes
     (tests/golden/make_metrics_golden.py).
The cosine scorer is a switch the reference does not contain as running code: (b) only.  The GRU branch is placed in the
graph by the reference code (the stand-in substitutes its GRUCell for UGRNNCell); the cell formula is the TF docs', restated.  Dropout: the
sites and scaling are pinned by (a); the masks themselves are this repo's counter-based spec (oracle/dropout_ref.py).
Every function cites the lines it follows.

Restated: nar_module/nar/nar_model.py:219-245 (inputs/masks), :730-773 (get_features),
:887-907 (scale/centre), :921-994 (item features), :996-1039 (normalisation), :1055-1089
(recency), :1134-1193 (novelty), :374-405 (CAR), :1308-1342 + tf.contrib.rnn.UGRNNCell
(RNN), :410-438 (FC), :444-517 (scorer + softmax), :639-704 (loss), :706-722 (Adam).
It computes on every padded position like the reference does (masked only in the loss).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as Fn

from chameleon_recsys_b200.hparams import ARTICLE_REQ_FEATURES, SESSION_REQ_SEQ_FEATURES, get_embedding_size

LEAKY_ALPHA = 0.2       # tf.nn.leaky_relu default
MS_PER_DAY = 1000.0 * 60.0 * 60.0 * 24.0


def _t(x, dtype):
    return torch.as_tensor(np.asarray(x)).to(dtype)


class NarOracle:
    """Pure function of (params, batch, state) -> loss / logits / grads; plus TF-Adam."""

    def __init__(self, session_features_config, articles_features_config, internal_features_config,
                 content_article_embeddings_matrix, articles_metadata, *, negative_samples,
                 softmax_temperature=1.0, reg_weight_decay=0.0, recent_clicks_for_normalization=1000,
                 elapsed_days_smooth_log_base=1.3, popularity_smooth_log_base=2.0, CAR_embedding_size=256,
                 rnn_units=256, rnn_num_layers=1, max_cardinality_for_ohe=10, lr=1e-3,
                 rnn_cell='ugrnn', ranking='mlp', dtype=torch.float32, keep_prob=1.0, novelty_reg_factor=0.0,
                 dropout_seed=42, int2log=None):
        self.scfg = session_features_config
        self.acfg = articles_features_config
        self.icfg = internal_features_config
        self.dtype = dtype
        self.acr = _t(content_article_embeddings_matrix, torch.float32).to(dtype)
        self.meta = {k: torch.as_tensor(np.asarray(v)) for k, v in articles_metadata.items()}
        self.K = int(negative_samples)
        self.tau = float(softmax_temperature)
        self.reg = float(reg_weight_decay)
        self.n_norm = int(recent_clicks_for_normalization)
        self.rec_base = float(elapsed_days_smooth_log_base)
        self.pop_base = float(popularity_smooth_log_base)
        self.C = int(CAR_embedding_size)
        self.H = int(rnn_units)
        self.layers = int(rnn_num_layers)
        self.max_ohe = int(max_cardinality_for_ohe)
        self.lr = float(lr)
        self.rnn_cell = rnn_cell
        self.ranking = ranking
        self.keep_prob = float(keep_prob)
        self.nov_factor = float(novelty_reg_factor)
        self.dropout_seed = int(dropout_seed)
        # internal (HBM) column -> logical column of the product's feature rows: the dropout spec is indexed by the former
        self.int2log = None if int2log is None else np.asarray(int2log, dtype=np.int64)
        self._drop = None          # (step,) while a training forward with dropout runs
        self.mask_override = None
        self._kinks = None
        self.V = int(articles_features_config['article_id']['cardinality'])
        self.adam_m: Dict[str, torch.Tensor] = {}
        self.adam_v: Dict[str, torch.Tensor] = {}
        self.step = 0

    # ------------------------------------------------------------------ params
    def set_params(self, logical: Dict[str, np.ndarray]):
        self.params = {k: _t(v, torch.float32).to(self.dtype).clone().requires_grad_(True)
                       for k, v in logical.items()}
        self.adam_m = {k: torch.zeros_like(v) for k, v in self.params.items()}
        self.adam_v = {k: torch.zeros_like(v) for k, v in self.params.items()}
        self.step = 0

    def get_params(self) -> Dict[str, np.ndarray]:
        return {k: v.detach().cpu().numpy().copy() for k, v in self.params.items()}

    def _p(self, name):
        return self.params[name]

    def regularised(self, name: str) -> bool:
        """l2_regularizer is attached to Dense kernels, all embeddings, gamma, beta; not to
        biases nor to the RNN (nar_model.py:378,386,414,426,450-471,740,894,898,917)."""
        return (('/RNN/' not in name) and not name.endswith('/bias'))

    # ------------------------------------------------------------------ features
    def _log_base(self, x, base):
        # nar_model.py:28-34
        return torch.log(x) / math.log(base) if self.dtype == torch.float64 else \
            torch.log(x) / torch.log(torch.tensor(base, dtype=self.dtype))

    def get_features(self, inputs: Dict[str, torch.Tensor], features_config, features_to_ignore, scope: str):
        """nar_model.py:730-773."""
        feats = []
        for fname, fc in features_config.items():
            if fname in features_to_ignore:
                continue
            if fc['type'] == 'categorical':
                size = fc['cardinality']
                ids = inputs[fname].long()
                if size <= self.max_ohe:
                    oh = torch.zeros(ids.shape + (size,), dtype=self.dtype)
                    ok = (ids >= 0) & (ids < size)
                    oh.scatter_(-1, ids.clamp(0, size - 1).unsqueeze(-1), ok.to(self.dtype).unsqueeze(-1))
                    feats.append(oh)
                else:
                    table = self._p(scope + '{}_cat_embedding/{}_embedding'.format(fname, fname))
                    feats.append(table[ids])
            elif fc['type'] == 'numerical':
                feats.append(inputs[fname].to(self.dtype).unsqueeze(-1))
            else:
                raise Exception('Invalid feature type: {}'.format(fname))
        if feats:
            return torch.cat(feats, dim=-1)
        return None

    def _elapsed_days(self, creation_dates, reference_timestamps):
        # nar_model.py:1055-1060 : int64 -> float32 cast BEFORE the subtraction
        ref32 = reference_timestamps.to(torch.float32)
        cre32 = creation_dates.to(torch.float32)
        return torch.relu((ref32 - cre32) / torch.tensor(MS_PER_DAY, dtype=torch.float32)).to(self.dtype)

    def _normalize_values(self, x, stats):
        # nar_model.py:1011-1039 + :996-1009 ; tf.nn.moments = population variance
        stats = stats.reshape(-1)
        mean = stats.mean()
        var = ((stats - mean) ** 2).mean()
        std = torch.sqrt(var + 1e-24)
        z = (x - mean) / std
        zs = (stats - mean) / std
        mn, mx = zs.min(), zs.max()
        eps = 1e-24
        scaled = (z - mn + eps) / torch.clamp(mx - mn, min=2 * eps)
        return scaled * 2.0 - 1.0

    def _buffer_last(self, buffer):
        nz = buffer[buffer != 0]
        return nz[:self.n_norm]

    def item_features(self, item_ids, events_timestamp, max_ts, buffer, pop_norm):
        """nar_model.py:921-994.  item_ids [...] i64; events_timestamp broadcastable i64 [..., 1]."""
        feats = []
        meta_vals = {f: self.meta[f][item_ids] for f in self.acfg if f not in ARTICLE_REQ_FEATURES}
        if meta_vals:
            feats.append(self.get_features(meta_vals, self.acfg, ARTICLE_REQ_FEATURES,
                                           'main/user_items_contextual_features/item_features/features/'))
        if self.icfg['article_content_embeddings']:
            feats.append(self.acr[item_ids])
        if self.icfg['item_clicked_embeddings']:
            feats.append(self._p('main/user_items_contextual_features/item_features/item_cat_embedding/items_embedding')[item_ids])
        nonpad = (item_ids != 0)
        last = self._buffer_last(buffer)
        if self.icfg['recency']:
            created = self.meta['created_at_ts'][item_ids].unsqueeze(-1)
            days = self._elapsed_days(created, events_timestamp)
            sm = self._log_base(days + 1.0, self.rec_base)
            if last.numel() == 0:
                stats = sm[nonpad]                                   # tf.cond :1082 (first batch only)
            else:
                rdays = self._elapsed_days(self.meta['created_at_ts'][last], max_ts)
                stats = self._log_base(rdays + 1.0, self.rec_base)
            feats.append(self._normalize_values(sm, stats))
        if self.icfg['novelty']:
            nov = -self._log_base(pop_norm[item_ids].unsqueeze(-1), self.pop_base)
            if last.numel() == 0:
                stats = nov[nonpad]
            else:
                stats = -self._log_base(pop_norm[last], self.pop_base)
            feats.append(self._normalize_values(nov, stats))
        return torch.cat(feats, dim=-1)

    # ------------------------------------------------------------------ dropout (spec: oracle/dropout_ref.py)
    def _dropout(self, x, tensor_id, row_key, feature_rows=False, t=None):
        """tf.layers.dropout(rate = 1 - keep_prob, training=True) with the counter-based masks of dropout_ref.
        ``mask_override`` (tests/test_oracle_reference_model.py): keep-masks recorded from a run of the reference code,
        keyed by tensor id (RNN outputs: (id, time step)), in the reference's column order."""
        if self._drop is None or self.keep_prob >= 1.0:
            return x
        if self.mask_override is not None:
            m = self.mask_override[tensor_id if t is None else (tensor_id, t)]
            return x * torch.as_tensor(np.asarray(m)).to(self.dtype) / self.keep_prob
        from . import dropout_ref
        n_cols = x.shape[-1]
        if feature_rows:
            Fp = len(self.int2log)
            mi = dropout_ref.keep_mask(self.dropout_seed, self._drop, tensor_id, row_key, Fp, self.keep_prob)
            valid = self.int2log >= 0
            m = np.zeros(mi.shape[:-1] + (n_cols,), dtype=bool)
            m[..., self.int2log[valid]] = mi[..., valid]
        else:
            m = dropout_ref.keep_mask(self.dropout_seed, self._drop, tensor_id, row_key, n_cols, self.keep_prob)
        return x * torch.as_tensor(m).to(self.dtype) / self.keep_prob

    # ------------------------------------------------------------------ layers
    def _dense(self, x, name, act, kink=None):
        y = x @ self._p(name + '/kernel') + self._p(name + '/bias')
        if act == 'leaky':
            k = None if (self._kinks is None or kink is None) else self._kinks.get(kink)
            if k is not None:
                # Kink alignment (tests): leaky_relu is not differentiable at 0, and a 1e-5 difference in a pre-activation that
                # happens to sit at the kink flips its slope between 1 and 0.2 - measured: forward noise of 1e-6 of the
                # tensor max moves the ORACLE's own matching_dense_layer_1/bias gradient by 10 %.  A gradient comparison is
                # only meaningful at identical slope choices, so the caller may hand over the other implementation's choices
                # (sign of its stored activations) for the valid positions; padded positions keep the oracle's own.
                m = (y > 0)
                m[self._kinks['valid']] = torch.as_tensor(k, dtype=torch.bool)
                return torch.where(m, y, LEAKY_ALPHA * y)
            return Fn.leaky_relu(y, LEAKY_ALPHA)
        if act == 'tanh':
            return torch.tanh(y)
        return y

    def CAR(self, x, kink=None):
        # nar_model.py:374-403
        return self._dense(self._dense(x, 'main/CAR/PreCAR_representation', 'leaky', kink),
                           'main/CAR/CAR_representation', 'tanh')

    def rnn(self, x, lengths, pos_key=None):
        """nar_model.py:1308-1342: MultiRNNCell of UGRNNCell inside dynamic_rnn(sequence_length); every cell wrapped in
        DropoutWrapper(output_keep_prob) (:1330-1333): the OUTPUT of a cell is dropped (what the next layer / FC1
        sees), the state it carries to the next time step is not."""
        B, T, _ = x.shape
        H = self.H
        states = [torch.zeros(B, H, dtype=self.dtype) for _ in range(self.layers)]
        outs = []
        for t in range(T):
            inp = x[:, t]
            new_states = []
            for i in range(self.layers):
                if self.rnn_cell == 'gru':
                    # tf.nn.rnn_cell.GRUCell (the cell nar_model.py:1315 keeps commented out; north_star's "session GRU"):
                    # [r, u] = sigmoid([x, h] Wg + bg) ; c = tanh([x, r*h] Wc + bc) ; h' = u*h + (1-u)*c
                    base = 'main/RNN/rnn/multi_rnn_cell/cell_{}/gru_cell/'.format(i)
                    gi = torch.cat([inp, states[i]], dim=1) @ self._p(base + 'gates/kernel') + self._p(base + 'gates/bias')
                    r, u = torch.sigmoid(gi[:, :H]), torch.sigmoid(gi[:, H:])
                    c = torch.tanh(torch.cat([inp, r * states[i]], dim=1) @ self._p(base + 'candidate/kernel') +
                                   self._p(base + 'candidate/bias'))
                    h = u * states[i] + (1.0 - u) * c
                    new_states.append(h)
                    inp = h if pos_key is None else self._dropout(h, 8 + i, pos_key[:, t], t=t)
                    continue
                base = 'main/RNN/rnn/multi_rnn_cell/cell_{}/ugrnn_cell/'.format(i)
                m = torch.cat([inp, states[i]], dim=1) @ self._p(base + 'kernel') + self._p(base + 'bias')
                g_act, c_act = m[:, :H], m[:, H:]
                c = torch.tanh(c_act)
                g = torch.sigmoid(g_act + 1.0)                     # forget_bias = 1.0
                h = g * states[i] + (1.0 - g) * c
                new_states.append(h)
                inp = h if pos_key is None else self._dropout(h, 8 + i, pos_key[:, t], t=t)
            alive = (t < lengths).to(self.dtype).unsqueeze(-1)
            outs.append(inp * alive)                                # zero output past the length
            states = [alive * ns + (1.0 - alive) * s for ns, s in zip(new_states, states)]
        return torch.stack(outs, dim=1)

    def scorer(self, cand, pred, kink=None):
        # nar_model.py:447-500 (cand [...,C] already multiplied outside for 'mlp')
        if self.ranking == 'cosine':
            return (Fn.normalize(cand, dim=-1) * Fn.normalize(pred, dim=-1)).sum(-1, keepdim=True)
        z = cand * pred
        base = 'main/recommendations_ranking/matching_dense_layer_'
        z = self._dense(z, base + '1', 'leaky', None if kink is None else 'z1_' + kink)
        z = self._dense(z, base + '2', 'leaky', None if kink is None else 'z2_' + kink)
        z = self._dense(z, base + '3', 'leaky', None if kink is None else 'z3_' + kink)
        return self._dense(z, base + '4', None)

    # ------------------------------------------------------------------ forward
    def forward(self, features: Dict[str, np.ndarray], labels: Dict[str, np.ndarray], negatives: np.ndarray,
                buffer: np.ndarray, pop_norm: np.ndarray, sum_mask_global: Optional[float] = None,
                train_step: Optional[int] = None, session0: int = 0, kinks: Optional[dict] = None):
        """-> dict with total_loss, xe_loss, reg_loss, logits [B,T,1+K] (already / temperature), mask, ...
        ``train_step`` (the optimiser step number, 1-based) switches dropout on (training mode, keep_prob < 1);
        ``session0`` = global index of the first session (data-parallel shards draw the masks of their own rows)."""
        self._drop = int(train_step) if (train_step is not None and self.keep_prob < 1.0) else None
        self._kinks = kinks          # see _dense: {'valid': bool [B,T], 'h1_in' / 'h1_pos' / 'h1_neg' / 'f1' / 'z{1,2,3}_{pos,neg}': slopes}
        item_clicked = torch.as_tensor(features['item_clicked']).long()
        event_ts = torch.as_tensor(features['event_timestamp']).long().unsqueeze(-1)
        lengths = torch.as_tensor(features['session_size']).long() - 1          # :227
        B, T = item_clicked.shape
        mask = (torch.arange(T)[None, :] < lengths[:, None])                     # :231
        max_ts = event_ts.max()                                                  # :235
        next_item = torch.as_tensor(labels['label_next_item']).long()
        neg = torch.as_tensor(negatives).long()
        buf = torch.as_tensor(np.asarray(buffer)).long()
        pop = _t(np.asarray(pop_norm, dtype=np.float32), torch.float32).to(self.dtype)   # placeholder is float32

        inputs = {k: torch.as_tensor(v) for k, v in features.items()}
        ctx = self.get_features(inputs, self.scfg['sequence_features'], SESSION_REQ_SEQ_FEATURES,
                                'main/user_items_contextual_features/features/')
        if ctx is None:
            ctx = torch.zeros(B, T, 1, dtype=self.dtype)                         # :325
        gamma = self._p('main/user_items_contextual_features/input_features_center_scale/gamma_scale')
        beta = self._p('main/user_items_contextual_features/input_features_center_scale/beta_center')

        pos_key = (np.arange(B, dtype=np.int64)[:, None] + session0) * T + np.arange(T, dtype=np.int64)[None, :]
        Kn = neg.shape[2]
        f_in = self.item_features(item_clicked, event_ts, max_ts, buf, pop)                        # :328
        x_in = torch.cat([ctx, f_in], dim=2) * gamma + beta                                        # :332-333
        x_in = self._dropout(x_in, 1, pos_key, feature_rows=True)                                  # :338-340
        f_pos = self.item_features(next_item, max_ts, max_ts, buf, pop)                            # :343
        x_pos = torch.cat([ctx, f_pos], dim=2) * gamma + beta
        x_pos = self._dropout(x_pos, 2, pos_key, feature_rows=True)                                # :351-353
        f_neg = self.item_features(neg, max_ts, max_ts, buf, pop)                                  # :356
        ctx_t = ctx.unsqueeze(2).expand(B, T, neg.shape[2], ctx.shape[-1])
        x_neg = torch.cat([ctx_t, f_neg], dim=3) * gamma + beta                                    # :360-364
        x_neg = self._dropout(x_neg, 3, pos_key[:, :, None] * Kn + np.arange(Kn, dtype=np.int64), feature_rows=True)   # :367-369

        e_in, e_pos, e_neg = self.CAR(x_in, 'h1_in'), self.CAR(x_pos, 'h1_pos'), self.CAR(x_neg, 'h1_neg')   # :382-403
        r = self.rnn(e_in, lengths, pos_key if self._drop is not None else None)                   # :408
        fc1 = self._dense(r, 'main/session_representation/FC1', 'leaky', 'f1')                     # :411
        fc1 = self._dropout(fc1, 4, pos_key)                                                       # :417-419
        pred = self._dense(fc1, 'main/session_representation/FC2', 'tanh')                         # :423-438
        s_pos = self.scorer(e_pos, pred, 'pos')                                                    # :478-485
        s_neg = self.scorer(e_neg, pred.unsqueeze(2), 'neg').squeeze(-1)                           # :493-500
        logits = torch.cat([s_pos, s_neg], dim=2) / self.tau                                       # :511-514
        logp = torch.log_softmax(logits, dim=-1)                                                   # :515, :660
        m = mask.to(self.dtype)
        denom = m.sum() if sum_mask_global is None else torch.tensor(float(sum_mask_global), dtype=self.dtype)
        xe = -(logp[:, :, 0] * m).sum() / denom                                                    # :660-664
        reg = torch.zeros((), dtype=self.dtype)
        if self.reg > 0.0:
            for name, w in self.params.items():
                if self.regularised(name):
                    reg = reg + self.reg * (w ** 2).sum() / 2.0                                    # l2_regularizer
        total = xe + reg                                                                           # :667
        nov_reg = torch.zeros((), dtype=self.dtype)
        if self.nov_factor > 0.0:
            # nar_model.py:517 (softmax over the NEGATIVES only), :531-544 (raw novelty of the negatives), :673-683
            neg_prob = torch.softmax(s_neg / self.tau, dim=-1)
            nov = -self._log_base(pop[neg], self.pop_base)
            nov_reg = self.nov_factor * ((neg_prob * nov).sum(-1) * m).sum() / denom
            total = total - nov_reg
        self._drop = None
        self._kinks = None
        return {'total_loss': total, 'xe_loss': xe, 'reg_loss': reg, 'nov_reg_loss': nov_reg, 'logits': logits, 'mask': mask,
                'x_in': x_in, 'x_pos': x_pos, 'x_neg': x_neg, 'e_in': e_in, 'e_pos': e_pos, 'e_neg': e_neg,
                'rnn_out': r, 'pred': pred, 'probs': torch.softmax(logits, dim=-1)}

    # ------------------------------------------------------------------ eval (ModeKeys.EVAL)
    @staticmethod
    def rank_and_metrics(out, labels: Dict[str, np.ndarray], negatives: np.ndarray, top_n: int):
        """rank_items_by_predicted_prob (nar_model.py:777-795: tf.nn.top_k over all 1+K candidates = descending
        probability, ties to the lower index) and the per-batch sums behind sparse_recall_at_top_k (:835-840) and
        define_mrr_metric (:862-885).  -> predicted_item_ids [B,T,1+K], predicted_item_probs, hits, rr_sum, count"""
        probs = out['probs'].detach().cpu().numpy()
        mask = out['mask'].cpu().numpy().astype(bool)
        ids = np.concatenate([np.asarray(labels['label_next_item'])[..., None], np.asarray(negatives)], axis=2)
        order = np.argsort(-probs, axis=2, kind='stable')                       # top_k order
        pred_ids = np.take_along_axis(ids, order, axis=2)
        pred_probs = np.take_along_axis(probs, order, axis=2)
        rank_of_pos = np.argmax(order == 0, axis=2)                             # 0-based rank of the positive
        found = (rank_of_pos < top_n) & mask
        hits = float(found.sum())
        rr = float((1.0 / (rank_of_pos + 1.0))[found].sum())
        return pred_ids, pred_probs, hits, rr, float(mask.sum())

    # ------------------------------------------------------------------ train
    def compute_gradients(self, out) -> Dict[str, torch.Tensor]:
        names = list(self.params.keys())
        grads = torch.autograd.grad(out['total_loss'], [self.params[n] for n in names], allow_unused=True)
        return {n: (g if g is not None else torch.zeros_like(self.params[n])) for n, g in zip(names, grads)}

    def apply_gradients(self, grads: Dict[str, torch.Tensor]):
        """tf.train.AdamOptimizer(lr, 0.9, 0.999, 1e-8) (nar_model.py:708-722): epsilon outside the
        bias-corrected sqrt; sparse gradients are applied densely (moments of every row decay)."""
        b1, b2, eps = 0.9, 0.999, 1e-8
        self.step += 1
        t = self.step
        lr_t = self.lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
        with torch.no_grad():
            for n, p in self.params.items():
                g = grads[n]
                self.adam_m[n].mul_(b1).add_(g, alpha=1.0 - b1)
                self.adam_v[n].mul_(b2).addcmul_(g, g, value=1.0 - b2)
                p.sub_(lr_t * self.adam_m[n] / (self.adam_v[n].sqrt() + eps))

    def train_step(self, features, labels, negatives, buffer, pop_norm, sum_mask_global=None, kinks=None):
        out = self.forward(features, labels, negatives, buffer, pop_norm, sum_mask_global, train_step=self.step + 1, kinks=kinks)
        grads = self.compute_gradients(out)
        self.apply_gradients(grads)
        return out, grads
