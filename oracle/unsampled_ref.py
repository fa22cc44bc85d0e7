"""TEST INFRASTRUCTURE - CPU reference of the unsampled evaluation (NarEngine.rank_labels, DESIGN.md section 13).

Only tests/ and tools/ may import this module; the product path never does.  The competitor sets restate what the
reference sampler's support is (nar_model.py:1220-1304: the batch's clicks and labels plus the recent-clicks buffer, minus
the session's own ids by get_neg_items_session's tf.setdiff1d); the scores come from the every-row oracle of
NarEngine.recommend (oracle/recommend_ref.py); the metrics are the reference's HitRate, MRR and NDCG (metrics.py:40-134)
on a ranked list with a single relevant item.
"""
from __future__ import annotations

from typing import Dict

import numpy as np


def pool(item_clicked, label_last_item, buffer) -> np.ndarray:
    """Sorted distinct nonzero ids of item_clicked [B, T], label_last_item [B] and the recent-clicks buffer."""
    ids = np.concatenate([np.asarray(a, dtype=np.int64).reshape(-1) for a in (item_clicked, label_last_item, buffer)])
    return np.unique(ids[ids != 0])


def competitor_sets(item_clicked, label_last_item, buffer) -> list:
    """Per session b: the pool minus every id of its row [item_clicked[b, :] | label_last_item[b]] (sorted)."""
    ic = np.asarray(item_clicked, dtype=np.int64)
    ll = np.asarray(label_last_item, dtype=np.int64).reshape(-1)
    p = pool(ic, ll, buffer)
    return [np.setdiff1d(p, np.append(ic[b], ll[b])) for b in range(ic.shape[0])]


def queries(features, labels):
    """The queries (b, t) in session-major order: valid positions t < session_size - 1 with label_next_item != 0."""
    ic = np.asarray(features['item_clicked'])
    T = ic.shape[1]
    lengths = np.clip(np.asarray(features['session_size'], dtype=np.int64) - 1, 0, T)
    lab = np.asarray(labels['label_next_item'], dtype=np.int64)
    qs, qt = np.nonzero((np.arange(T)[None, :] < lengths[:, None]) & (lab != 0))
    return qs, qt


def rank_rule(label_score: float, competitor_scores) -> int:
    """Competitors strictly above the label (ties go to the label: it is index 0 of tf.nn.top_k's input)."""
    return int(np.count_nonzero(np.asarray(competitor_scores) > label_score))


def metric_values(ranks, top_n: int) -> Dict[str, np.ndarray]:
    """Per query: the reference's HitRate, MRR and NDCG terms of a ranked list whose only relevant item is at ``rank``."""
    r = np.asarray(ranks, dtype=np.int64)
    hit = r < top_n
    return {'hitrate': hit.astype(np.float64),
            'mrr': np.where(hit, 1.0 / (r + 1.0), 0.0),
            'ndcg': np.where(hit, 1.0 / np.log2(r + 2.0), 0.0)}


def unsampled(orc, features, labels, buffer, pop_norm, top_n: int, candidates=None) -> dict:
    """Every query of the batch ranked against its competitor set, scored in the precision of ``orc`` (NarOracle) as
    NarEngine.recommend scores a candidate.  ``candidates`` None = the pool.
    -> dict(qs, qt [Q], candidates [N], scores [Q', N] for every valid position, rank [Q], gap [Q] = the smallest
    |competitor - label| score difference (inf without competitors), n_comp [Q], and the four metrics)."""
    from oracle.recommend_ref import recommend
    ic = np.asarray(features['item_clicked'], dtype=np.int64)
    ll = np.asarray(labels['label_last_item'], dtype=np.int64).reshape(-1)
    cand = pool(ic, ll, buffer) if candidates is None else np.sort(np.asarray(candidates, dtype=np.int64))
    ref = recommend(orc, features, buffer, pop_norm, cand, 1, positions='all', exclude_session_clicks=False)
    row = {(int(b), int(t)): i for i, (b, t) in enumerate(zip(ref['query_session'], ref['query_position']))}
    qs, qt = queries(features, labels)
    lab = np.asarray(labels['label_next_item'], dtype=np.int64)
    ranks, gaps, n_comp = [], [], []
    for b, t in zip(qs, qt):
        j = np.searchsorted(cand, lab[b, t])
        if j >= cand.size or cand[j] != lab[b, t]:
            continue
        s = ref['scores'][row[(int(b), int(t))]]
        comp = ~np.isin(cand, np.append(ic[b], ll[b]))
        comp[j] = False
        ranks.append(rank_rule(s[j], s[comp]))
        gaps.append(np.abs(s[comp] - s[j]).min() if comp.any() else np.inf)
        n_comp.append(int(comp.sum()))
    ranks = np.asarray(ranks, dtype=np.int64)
    v = metric_values(ranks, top_n)
    Q = max(ranks.size, 1)
    return {'qs': qs, 'qt': qt, 'candidates': cand, 'scores': ref['scores'], 'rank': ranks, 'gap': np.asarray(gaps),
            'n_comp': np.asarray(n_comp, dtype=np.int64),
            'unsampled_hitrate_at_n': v['hitrate'].sum() / Q, 'unsampled_mrr_at_n': v['mrr'].sum() / Q,
            'unsampled_ndcg_at_n': v['ndcg'].sum() / Q, 'unsampled_candidates_per_query': float(np.sum(n_comp)) / Q}
