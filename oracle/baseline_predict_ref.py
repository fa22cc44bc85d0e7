"""TEST INFRASTRUCTURE - CPU reference of the baselines' recommendations (BaselineTables.recommend, Estimator.predict with
``recommender=<suffix>``, DESIGN.md section 16).

Only tests/ and tools/ may import this module; the product path never does.  A query (b, t) has the valid set
``candidates`` minus item_clicked[b, 0..t] (when excluding the session's clicks); each baseline scores the valid ids as
the sampled oracles score a candidate (``BaselinesRef._scores``, ``SknnRef.item_scores``) and the output is the first
``top_n`` admissible ids in its strict order - ``(score desc, tie asc)`` for the five table baselines, ``(score desc, first
neighbour asc, id asc)`` for the session kNN ones - then id 0 with score NaN, as the reference's
``_get_top_n_valid_items`` pads with 0.
"""
from __future__ import annotations

import numpy as np


def valid_set(candidates, item_clicked, b: int, t: int, exclude: bool) -> list:
    cand = [int(c) for c in np.asarray(candidates, dtype=np.int64).reshape(-1)]
    if not exclude:
        return cand
    row = set(int(x) for x in np.asarray(item_clicked)[b, :t + 1])
    return [c for c in cand if c not in row]


def ranked(ref, suffix: str, item_clicked, b: int, t: int, valid, buffer=None, articles_pop=None, hist=None) -> list:
    """[(score, key, id)] of the admissible ids of ``valid`` in the baseline's order.  ``ref``: a BaselinesRef (the five
    table baselines) or an SknnRef (``suffix`` 'v-sknn' / 'sknn')."""
    from oracle.baselines_ref import BaselinesRef
    ic = np.asarray(item_clicked, dtype=np.int64)
    if isinstance(ref, BaselinesRef):
        hc, hf = BaselinesRef._hist(buffer) if hist is None else hist
        keys = [(sc, (tie, c), c) for sc, tie, c in ref._scores(suffix, int(ic[b, t]), valid, hc, hf, articles_pop)]
    else:
        scores, first = ref.item_scores(ic[b, :t + 1].tolist())
        keys = [(scores[c], (first[c], c), c) for c in dict.fromkeys(valid) if c in scores]
    return sorted(keys, key=lambda k: (-k[0], k[1]))


def recommend(ref, suffix: str, item_clicked, q_pos, candidates, top_n: int, buffer=None, articles_pop=None,
              exclude: bool = True):
    """-> (ids [Q, top_n] int64, scores [Q, top_n] float64) for the queries at flat positions ``q_pos`` = b*T + t."""
    ic = np.asarray(item_clicked, dtype=np.int64)
    T = ic.shape[1]
    q_pos = np.asarray(q_pos, dtype=np.int64).reshape(-1)
    ids = np.zeros((q_pos.size, top_n), np.int64)
    scores = np.full((q_pos.size, top_n), np.nan)
    hist = None
    from oracle.baselines_ref import BaselinesRef
    if isinstance(ref, BaselinesRef):
        hist = BaselinesRef._hist(buffer)
    for q, pos in enumerate(q_pos.tolist()):
        b, t = divmod(pos, T)
        r = ranked(ref, suffix, ic, b, t, valid_set(candidates, ic, b, t, exclude), buffer, articles_pop, hist)[:top_n]
        ids[q, :len(r)] = [k[2] for k in r]
        scores[q, :len(r)] = [k[0] for k in r]
    return ids, scores

