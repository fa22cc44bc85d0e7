"""Plain-Python restatement of the evaluation hook's hit rate by session position (the reference's
``HitRateBySessionPosition``, metrics.py, reported by evaluation.py ``compute_metrics_results``).

A query is a cell (b, t) with a nonzero label; its position is p = t + 1.  Per recommender and position: ``total[p]``
queries, ``hits[p]`` of them with the label among the first ``top_n`` ids of the list, and ``norm_pop[p]`` the sum of
``pop[label]``.  The reference starts that sum from ``int`` 0 and adds ``np.float32`` scalars, so it is a float32 sum in
the order batch -> session -> cell, and its mean is divided in float32; here every add is rounded to float32 explicitly.
Keys exist for the positions with a query only; the model's (suffix '') also carry ``clicks_at_pos_PP`` and
``avg_norm_pop_by_pos_PP``.
"""
from __future__ import annotations

from collections import defaultdict

import numpy as np


class ByPositionRef:
    """Streaming accumulator over ``rows`` recommenders (what the hook keeps per evaluation)."""

    def __init__(self, rows, top_n):
        self.rows, self.top_n = int(rows), int(top_n)

    def begin(self):
        self.hits = [defaultdict(int) for _ in range(self.rows)]
        self.total = [defaultdict(int) for _ in range(self.rows)]
        self.norm_pop = [defaultdict(lambda: np.float32(0.0)) for _ in range(self.rows)]

    def add(self, row, lists, labels, T, pos=None, pop=None):
        """``lists`` [Q, len] and ``labels`` [Q] of recommender ``row`` in session-major order; query q sits at
        ``pos[q] % T`` (flat b*T + t) or, without ``pos``, at ``q % T``.  ``pop`` [V] float32: add the labels' popularity."""
        labels = np.asarray(labels).reshape(-1)
        lists = np.asarray(lists).reshape(labels.size, -1)
        for q, label in enumerate(labels.tolist()):
            if label == 0:
                continue
            p = int(pos[q] if pos is not None else q) % T + 1
            self.total[row][p] += 1
            if label in lists[q, :self.top_n].tolist():
                self.hits[row][p] += 1
            if pop is not None:
                self.norm_pop[row][p] = np.float32(self.norm_pop[row][p] + np.float32(pop[label]))

    def results(self, row, suffix='') -> dict:
        out = {}
        for p in sorted(self.total[row]):
            q = self.total[row][p]
            out['hitrate_at_n_by_pos%s_%02d' % ('_' + suffix if suffix else '', p)] = self.hits[row][p] / float(q)
            if not suffix:
                out['clicks_at_pos_%02d' % p] = q
                out['avg_norm_pop_by_pos_%02d' % p] = float(np.float32(self.norm_pop[row][p]) / np.float32(q))
        return out
