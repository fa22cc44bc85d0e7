"""Plain-Python restatement of the evaluation hook's list metrics (the reference's metrics.py, as built by
``ItemsStateUpdaterHook.create_eval_metrics``): NDCG, item coverage, ESI-R, ESI-RR, EILD-R and EILD-RR.

A query is a position whose label is nonzero; its list is a row of ids.  The first ``m = min(top_n, len(row))`` ids
are scored; NDCG's ideal counts the label's occurrences over the whole row (for the model the row is the full ranked
candidate list, for a baseline its 0-padded top-n).  ``disc(k) = 1 / log2(k + 2)``; ``rel(x)`` is 1 for the label and
``neg_relevance`` otherwise; ``D(i, j)`` is sklearn's ``cosine_distances / 2`` of the ACR rows in fp64 (a row of norm 0
has cosine 0).  The novelty and diversity sums run over ``i < m - 1`` only, like the reference's ``range(0, len - 1)``.
Coverage is |recommended ids| / |clicked ids|: the clicked set starts as the recent-clicks buffer (0 included while it
holds padding) and gains every batch's nonzero labels and clicks; the recommended set gains every scored id, 0 included.
"""
from __future__ import annotations

import math

import numpy as np

VALUES = ('ndcg', 'esi-r', 'esi-rr', 'eild-r', 'eild-rr')


def disc(k: int) -> float:
    return 1.0 / math.log2(k + 2)


def distances(acr, norms, ids) -> np.ndarray:
    x = acr[np.asarray(ids, dtype=np.int64)]
    nn = np.outer(norms[ids], norms[ids])
    dot = x @ x.T
    cos = np.where(nn > 0, dot / np.where(nn > 0, nn, 1.0), 0.0)
    return np.clip(1.0 - cos, 0.0, 2.0) / 2.0


def list_values(row, label, top_n, pop, acr, norms, neg_relevance):
    """The five per-query values of one query."""
    row = [int(v) for v in row]
    m = min(top_n, len(row))
    lst = row[:m]
    occ = row.count(label)
    dcg = sum(disc(i) for i in range(m) if lst[i] == label)
    idcg = sum(disc(i) for i in range(min(m, occ)))
    ndcg = dcg / idcg if idcg > 0 else 0.0
    D = distances(acr, norms, lst)
    rel = [1.0 if x == label else neg_relevance for x in lst]
    w = esi = esi_rr = eild = eild_rr = 0.0
    for i in range(m - 1):
        di = disc(i)
        nov = -math.log2(float(pop[lst[i]])) * di
        num = den = num_rr = den_rr = 0.0
        for j in range(m):
            if j == i:
                continue
            wj = disc(max(0, j - i - 1))
            num += D[i, j] * wj
            den += wj
            if j > i:
                num_rr += D[i, j] * wj * rel[j]
                den_rr += wj * rel[j]
        esi += nov
        esi_rr += nov * rel[i]
        eild += num / den * di
        eild_rr += num_rr / den_rr * di * rel[i]
        w += di
    return ndcg, esi / w, esi_rr / w, eild / w, eild_rr / w


class EvalMetricsRef:
    """Streaming accumulator over ``rows`` recommenders sharing one clicked set (what the hook keeps per evaluation)."""

    def __init__(self, rows, top_n, acr, neg_relevance=0.1):
        self.rows, self.top_n, self.neg_relevance = int(rows), int(top_n), float(neg_relevance)
        self.acr = np.asarray(acr, dtype=np.float64)
        self.norms = np.sqrt((self.acr * self.acr).sum(axis=1))

    def begin(self, buffer):
        self.sums = np.zeros((self.rows, len(VALUES)))
        self.count = np.zeros(self.rows, dtype=np.int64)
        self.recommended = [set() for _ in range(self.rows)]
        self.clicked = set(int(v) for v in np.asarray(buffer).reshape(-1))

    def add_lists(self, row, lists, labels, pop):
        """``lists`` [Q, len] id rows and ``labels`` [Q] of recommender ``row``; ``pop`` the normalised popularity the
        batch was fed with."""
        lists = np.asarray(lists).reshape(len(np.asarray(labels).reshape(-1)), -1)
        for lst, label in zip(lists, np.asarray(labels).reshape(-1).tolist()):
            if label == 0:
                continue
            self.sums[row] += list_values(lst, label, self.top_n, pop, self.acr, self.norms, self.neg_relevance)
            self.count[row] += 1
            self.recommended[row].update(int(v) for v in lst[:self.top_n])

    def add_clicks(self, item_clicked, label_next):
        for a in (label_next, item_clicked):
            a = np.asarray(a).reshape(-1)
            self.clicked.update(int(v) for v in a[a != 0])

    def per_query_means(self, row) -> dict:
        c = self.count[row]
        return {k: (self.sums[row, i] / c if c else float('nan')) for i, k in enumerate(VALUES)}

    def results(self, row) -> dict:
        out = self.per_query_means(row)
        out['recommended'] = len(self.recommended[row])
        out['clicked'] = len(self.clicked)
        out['coverage'] = out['recommended'] / out['clicked'] if out['clicked'] else float('nan')
        return out
