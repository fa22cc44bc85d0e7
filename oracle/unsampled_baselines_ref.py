"""TEST INFRASTRUCTURE - CPU reference of the baselines' unsampled evaluation (BaselineTables.rank_unsampled, DESIGN.md
section 14).

Only tests/ and tools/ may import this module; the product path never does.  The pool and the competitor sets are those of
oracle/unsampled_ref.py (the reference sampler's support); each baseline scores the label and its competitors as the
sampled oracles score a candidate (``BaselinesRef._scores``, ``SknnRef.item_scores``), and ranks them in the same strict
orders: ``(score desc, tie asc)`` for the five table baselines, ``(score desc, first neighbour asc, id asc)`` for the
session kNN ones.  A label the baseline does not admit is a miss (rank MISS).
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from oracle.unsampled_ref import metric_values, pool as make_pool

MISS = 0x7fffffff


def _keys_table(ref, suffix, item, ids, hc, hf, pop) -> dict:
    """{id: (score, tie)} of the admissible ids (BaselinesRef._scores)."""
    return {c: (sc, tie) for sc, tie, c in ref._scores(suffix, int(item), ids, hc, hf, pop)}


def _rank(keys: dict, label: int, comp, sort_key) -> tuple:
    """-> (rank of the label among the admissible competitors, or MISS; the pessimistic and optimistic ranks over every
    order of equal scores: the competitors with a score >= / > the label's)."""
    if label not in keys:
        return MISS, MISS, MISS
    kl = sort_key(label, keys[label])
    rank = lo = hi = 0
    for c in comp:
        if c in keys:
            kc = sort_key(c, keys[c])
            rank += kc < kl
            lo += kc[0] <= kl[0]
            hi += kc[0] < kl[0]
    return rank, lo, hi


def ranks(ref, suffix: str, item_clicked, label_next, label_last_item, buffer, articles_pop=None,
          candidates: Optional[np.ndarray] = None) -> dict:
    """Every query (b, t) with label_next != 0 ranked against ``candidates`` (default: the pool of the batch) minus the label
    and its session's row [item_clicked[b, :] | label_last_item[b]].  ``ref``: a BaselinesRef (the five table baselines)
    or an SknnRef (``suffix`` 'v-sknn' / 'sknn'), holding the state the batch is scored against.
    -> dict(q [Q] flat positions b*T+t, rank [Q] (MISS for a label the baseline does not admit), rank_lo [Q] (every
    competitor of the label's score counted above it: the pessimistic rank over all orders of ties), rank_hi [Q] (the
    optimistic one), n_comp [Q])."""
    from oracle.baselines_ref import BaselinesRef
    ic = np.asarray(item_clicked, dtype=np.int64)
    ln = np.asarray(label_next, dtype=np.int64)
    ll = np.asarray(label_last_item, dtype=np.int64).reshape(-1)
    B, T = ic.shape
    cand = make_pool(ic, ll, buffer) if candidates is None else np.unique(np.asarray(candidates, dtype=np.int64))
    cand = cand[cand != 0]
    table = isinstance(ref, BaselinesRef)
    if table:
        hc, hf = BaselinesRef._hist(buffer)
    qs, rk, lo, hi, n_comp = [], [], [], [], []
    for b in range(B):
        row = set(np.append(ic[b], ll[b]).tolist())
        for t in range(T):
            label = int(ln[b, t])
            if label == 0:
                continue
            comp = [int(c) for c in cand if int(c) != label and int(c) not in row]
            if table:
                keys = _keys_table(ref, suffix, ic[b, t], [label] + comp, hc, hf, articles_pop)
                r, r_lo, r_hi = _rank(keys, label, comp, lambda c, k: (-k[0], k[1]))
            else:
                scores, first = ref.item_scores(ic[b, :t + 1].tolist())
                keys = {x: (scores[x], first[x]) for x in [label] + comp if x in scores}
                r, r_lo, r_hi = _rank(keys, label, comp, lambda c, k: (-k[0], k[1], c))
            qs.append(b * T + t)
            rk.append(r)
            lo.append(r_lo)
            hi.append(r_hi)
            n_comp.append(len(comp))
    return {k: np.asarray(v, dtype=np.int64)
            for k, v in (('q', qs), ('rank', rk), ('rank_lo', lo), ('rank_hi', hi), ('n_comp', n_comp))}


def histogram(r: dict, top_n: int) -> np.ndarray:
    """The [top_n + 2] accumulator of BaselineTables.rank_unsampled for the ranks of ``ranks``."""
    h = np.zeros(top_n + 2, dtype=np.int64)
    rk = r['rank']
    np.add.at(h, rk[rk < top_n], 1)
    h[top_n] = rk.size
    h[top_n + 1] = int(r['n_comp'].sum())
    return h


def metrics(r: dict, top_n: int) -> Dict[str, float]:
    """Mean hit rate, MRR and NDCG at ``top_n`` of the ranks, and their pessimistic (``_lo``) / optimistic (``_hi``)
    bounds over every order of equal scores."""
    out = {}
    Q = max(r['rank'].size, 1)
    for name, rk in (('', r['rank']), ('_lo', r['rank_lo']), ('_hi', r['rank_hi'])):
        v = metric_values(rk, top_n)
        for k in ('hitrate', 'mrr', 'ndcg'):
            out[k + name] = float(v[k].sum()) / Q
    out['candidates_per_query'] = float(r['n_comp'].sum()) / Q
    return out
