"""TEST INFRASTRUCTURE - CPU reference of NarEngine.recommend (ModeKeys.PREDICT) on top of oracle/nar_oracle.py.

Only tests/ and tools/ may import this module; the product path never does.  It is the plain every-row form: each
(query, candidate) feature row is materialised and run through NarOracle's CAR / scorer exactly as NarOracle.forward
runs a sampled negative - no PC + PI decomposition - and the top-n rule is restated in numpy.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from chameleon_recsys_b200.hparams import SESSION_REQ_SEQ_FEATURES
from oracle.nar_oracle import NarOracle, _t


def topn_rule(scores: np.ndarray, cand: np.ndarray, top_n: int, excluded=None):
    """Top-n of every row of ``scores`` [Q, N] over the candidate ids ``cand`` [N]: descending score, ties to the lower
    candidate index (tf.nn.top_k); ``excluded[q]`` = ids query q never returns; probabilities = softmax over the
    non-excluded candidates; slots beyond the non-excluded count hold id 0, score -inf, prob 0.
    -> (ids, scores, probs) [Q, top_n] (float64 scores / probs)."""
    scores = np.asarray(scores, dtype=np.float64)
    Q = scores.shape[0]
    ids = np.zeros((Q, top_n), dtype=np.int64)
    sc = np.full((Q, top_n), -np.inf)
    pr = np.zeros((Q, top_n))
    for q in range(Q):
        keep = np.ones(cand.size, dtype=bool) if excluded is None else ~np.isin(cand, np.asarray(list(excluded[q]), dtype=np.int64))
        idx = np.flatnonzero(keep)
        if idx.size == 0:
            continue
        s = scores[q, idx]
        e = np.exp(s - s.max())
        p = e / e.sum()
        order = np.argsort(-s, kind='stable')[:top_n]
        k = order.size
        ids[q, :k], sc[q, :k], pr[q, :k] = cand[idx[order]], s[order], p[order]
    return ids, sc, pr


def recommend(orc: NarOracle, features: Dict[str, np.ndarray], buffer: np.ndarray, pop_norm: np.ndarray, candidates,
              top_n: int, positions: str = 'last', exclude_session_clicks: bool = True):
    """Every-row form of NarEngine.recommend with the weights of ``orc``: for each query position (positions='last': the
    last valid position t = session_size - 2 of every session; 'all': every valid position, session-major) and each
    candidate id, the feature row concat(context(b, t), item_features(id, ts = batch max event_timestamp)) * gamma + beta
    goes through CAR and the scorer like a sampled negative of that position (nar_model.py:356-364, :374-405,
    :444-515), then / temperature.  Recency / novelty statistics: the recent-clicks buffer, or - empty buffer - the
    candidate rows themselves (the negatives' tf.cond, :1082 / :1179).  candidates: None = distinct nonzero buffer ids,
    'catalog' = 1 .. V-1, else the given ids.
    -> dict(query_session, query_position [Q], candidates [N], scores [Q, N], x [Q, N, F], predicted_item_ids /
    predicted_item_scores / predicted_item_probs [Q, top_n])."""
    item_clicked = np.asarray(features['item_clicked'], dtype=np.int64)
    B, T = item_clicked.shape
    buf = np.asarray(buffer, dtype=np.int64).reshape(-1)
    if candidates is None:
        cand = np.unique(buf[buf != 0])
    elif isinstance(candidates, str):
        assert candidates == 'catalog', candidates
        cand = np.arange(1, orc.V, dtype=np.int64)
    else:
        cand = np.asarray(candidates, dtype=np.int64)
    lengths = np.clip(np.asarray(features['session_size'], dtype=np.int64) - 1, 0, T)
    if positions == 'last':
        qs = np.flatnonzero(lengths > 0)
        qt = lengths[qs] - 1
    else:
        qs, qt = np.nonzero(np.arange(T)[None, :] < lengths[:, None])
    Q, N = qs.size, cand.size
    # the session branch only: labels / negatives are placeholders (nonzero, so that an empty buffer's per-row-group
    # statistics of the unused positive / negative rows are defined)
    labels = {'label_next_item': item_clicked, 'label_last_item': np.zeros(B, dtype=np.int64)}
    with torch.no_grad():
        out = orc.forward(features, labels, item_clicked[:, :, None], buffer, pop_norm)
        pred = out['pred'][qs, qt]                                                                 # [Q, C]
        inputs = {k: torch.as_tensor(v) for k, v in features.items()}
        ctx = orc.get_features(inputs, orc.scfg['sequence_features'], SESSION_REQ_SEQ_FEATURES,
                               'main/user_items_contextual_features/features/')
        if ctx is None:
            ctx = torch.zeros(B, T, 1, dtype=orc.dtype)
        gamma = orc._p('main/user_items_contextual_features/input_features_center_scale/gamma_scale')
        beta = orc._p('main/user_items_contextual_features/input_features_center_scale/beta_center')
        max_ts = torch.as_tensor(features['event_timestamp']).long().max()
        pop = _t(np.asarray(pop_norm, dtype=np.float32), torch.float32).to(orc.dtype)
        ids = torch.as_tensor(cand).long()[None, :].expand(Q, N)
        f_c = orc.item_features(ids, max_ts, max_ts, torch.as_tensor(buf).long(), pop)            # :356 with ids = candidates
        cq = ctx[torch.as_tensor(qs), torch.as_tensor(qt)]
        x = torch.cat([cq[:, None, :].expand(Q, N, cq.shape[-1]), f_c], dim=2) * gamma + beta     # :360-364
        scores = (orc.scorer(orc.CAR(x), pred[:, None, :]).squeeze(-1) / orc.tau).numpy()        # :493-514
    excl = None
    if exclude_session_clicks:
        excl = [set(item_clicked[b, :t + 1].tolist()) for b, t in zip(qs, qt)]
    pid, psc, ppr = topn_rule(scores, cand, int(top_n), excl)
    return {'query_session': qs, 'query_position': qt, 'candidates': cand, 'scores': scores, 'x': x.numpy(),
            'predicted_item_ids': pid, 'predicted_item_scores': psc, 'predicted_item_probs': ppr}
