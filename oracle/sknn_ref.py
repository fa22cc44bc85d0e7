"""Plain-Python restatement of the reference's session-based kNN baseline (benchmarks/session_knn.py, V-SkNN with
``first_session_clicks_decay='div'``, SkNN with ``'same'``) driven by nar_model.py:1609-1632, with the tie rules of
csrc/sknn.cu:

* neighbours of equal similarity: the HIGHER session id first (the reference's order whenever the 'recent' cut applied:
  it pre-sorts by id descending and Python's sort is stable; otherwise its order is CPython set iteration order);
* items of equal score: first the rank of the first kept neighbour copy that contains the item (the reference's dict
  insertion order), then the LOWER article id (standing in for the iteration order of a Python set of ints).

Everything else is the reference's own arithmetic: the buffer of the last ``sessions_buffer_size`` sessions in insertion
order with its item -> session-ids map (an eviction discards ``(x, id)`` for every item of the evicted entry, even when a
newer entry with the same id holds ``x``), the candidate list with one copy per position of the active session whose
item maps to the session and ``find_session_on_buffer`` (a leftmost binary search over the buffer in insertion order,
which misses ids that are not ascending), the similarity against the full item set of the entry that search finds, the
``0 < sim < 1`` filter and the neighbour cut over copies, and item scores summed copy by copy in neighbour order.

Per batch the HR / MRR sums are taken from the label's rank histogram in a fixed order (what the device kernel does),
and ``bounds`` gives the pessimistic / optimistic HR and MRR over every order of equal item scores.
"""
from __future__ import annotations

import copy
from collections import defaultdict
from math import sqrt

import numpy as np

KNN_SUFFIXES = ('v-sknn', 'sknn')


class SknnRef:
    def __init__(self, sessions_buffer_size=3000, candidate_sessions_sample_size=1000,
                 nearest_neighbor_session_for_scoring=500, similarity='cosine', first_session_clicks_decay='div'):
        self.S = int(sessions_buffer_size)
        self.C = int(candidate_sessions_sample_size)
        self.NN = int(nearest_neighbor_session_for_scoring)
        self.similarity = similarity
        self.decay = first_session_clicks_decay
        self.buffer = []                        # [(session_id, frozenset of item ids)], oldest first
        self.map = defaultdict(set)             # item -> session ids

    @property
    def suffix(self):
        return 'sknn' if self.decay == 'same' else 'v-sknn'

    # ---- training
    def update(self, session_ids, all_items):
        """One batch: ``all_items`` [B, T1] (item_clicked | label, 0 = padding), ``session_ids`` [B]."""
        new = [(int(s), frozenset(int(x) for x in row if x != 0)) for s, row in zip(session_ids, np.asarray(all_items))]
        self.buffer.extend(new)
        for s, items in new:
            for x in items:
                self.map[x].add(s)
        while len(self.buffer) > self.S:
            s, items = self.buffer.pop(0)
            for x in items:
                self.map[x].discard(s)

    def export(self) -> dict:
        """The buffer in insertion order: ids [n], lens [n], items [n, W] (sorted, 0-padded), live [n, W] (item x of
        entry e is live when (x, id_e) is in the map)."""
        n = len(self.buffer)
        W = max([len(it) for _, it in self.buffer] + [1])
        ids = np.array([s for s, _ in self.buffer], dtype=np.int64)
        lens = np.array([len(it) for _, it in self.buffer], dtype=np.int64)
        items = np.zeros((n, W), dtype=np.int64)
        live = np.zeros((n, W), dtype=bool)
        for e, (s, it) in enumerate(self.buffer):
            xs = sorted(it)
            items[e, :len(xs)] = xs
            live[e, :len(xs)] = [s in self.map.get(x, ()) for x in xs]
        return {'ids': ids, 'lens': lens, 'items': items, 'live': live}

    def snapshot(self):
        self._chk = copy.deepcopy((self.buffer, self.map))

    def restore(self):
        self.buffer, self.map = self._chk
        del self._chk

    # ---- neighbours
    def find(self, session_id) -> int:
        """find_session_on_buffer: leftmost binary search over the buffer in insertion order."""
        left, right = 0, len(self.buffer)
        while left < right:
            mid = (left + right) // 2
            if session_id > self.buffer[mid][0]:
                left = mid + 1
            else:
                right = mid
        return left if left != len(self.buffer) and self.buffer[left][0] == session_id else -1

    def _sim(self, P, items):
        sP = set(P)
        if self.decay == 'same':
            num = len(sP & items)
        else:
            num = 0
            for pos, x in enumerate(reversed(P)):
                if x in items:
                    num += 1 / (pos + 1)
        den = sqrt(len(sP)) * sqrt(len(items)) if self.similarity == 'cosine' else len(sP | items)
        return num / den

    def candidates(self, P) -> dict:
        """{session id: copies} after the 'recent' cut."""
        m = defaultdict(int)
        for x in P:
            for s in self.map.get(int(x), ()):
                if self.find(s) != -1:
                    m[s] += 1
        total = sum(m.values())
        if self.C > 0 and total > self.C:
            left, cut = self.C, {}
            for s in sorted(m, reverse=True):
                if left == 0:
                    break
                cut[s] = min(m[s], left)
                left -= cut[s]
            m = cut
        return dict(m)

    def neighbors(self, P, cut=True) -> list:
        """[(session id, similarity)] with one entry per kept copy, in neighbour order (``cut=False``: before the
        nearest-neighbour cut)."""
        P = [int(x) for x in P]
        scored = []
        for s, c in self.candidates(P).items():
            sim = self._sim(P, self.buffer[self.find(s)][1])
            if 0.0 < sim < 1.0:
                scored.append((sim, s, c))
        scored.sort(key=lambda v: (-v[0], -v[1]))
        out = [(s, sim) for sim, s, c in scored for _ in range(c)]
        return out[:self.NN] if cut else out

    def item_scores(self, P):
        """-> ({item: score}, {item: rank of the first kept neighbour copy holding it})."""
        scores, first = {}, {}
        for r, (s, sim) in enumerate(self.neighbors(P)):
            for x in self.buffer[self.find(s)][1]:
                scores[x] = scores.get(x, 0) + sim
                first.setdefault(x, r)
        return scores, first

    def predict(self, P, valid, top_n, scored=None) -> list:
        """Top-n of ``valid`` (label + negatives) for the active session ``P``, 0-padded (``scored``: item_scores(P))."""
        scores, first = self.item_scores(P) if scored is None else scored
        valid = {int(v) for v in valid}
        ranked = sorted((x for x in scores if x in valid), key=lambda x: (-scores[x], first[x], x))
        top = ranked[:top_n]
        return top + [0] * (top_n - len(top))

    # ---- one evaluation batch
    def score(self, item_clicked, label_next, negatives, top_n) -> dict:
        """-> {'ids' [B*T, top_n], 'hist' [top_n+1], 'hits', 'rr', 'count', 'bounds' (hr_lo, hr_hi, rr_lo, rr_hi) sums}
        over the queries (b, t) with label_next != 0."""
        item_clicked = np.asarray(item_clicked, dtype=np.int64)
        label_next = np.asarray(label_next, dtype=np.int64)
        negatives = np.asarray(negatives, dtype=np.int64)
        B, T = item_clicked.shape
        ids = np.zeros((B * T, top_n), dtype=np.int64)
        hist = np.zeros(top_n + 1, dtype=np.int64)
        lo, hi = [0.0, 0.0], [0.0, 0.0]
        for b in range(B):
            for t in range(T):
                label = int(label_next[b, t])
                if label == 0:
                    continue
                P = item_clicked[b, :t + 1].tolist()
                valid = [label] + negatives[b, t].tolist()
                scored = self.item_scores(P)
                top = self.predict(P, valid, top_n, scored)
                ids[b * T + t] = top
                hist[top_n] += 1
                if label in top:
                    hist[top.index(label)] += 1
                scores = scored[0]
                if label in scores:
                    vs = {int(v) for v in valid if int(v) in scores}
                    better = sum(1 for v in vs if scores[v] > scores[label])
                    equal = sum(1 for v in vs if scores[v] == scores[label]) - 1
                    for acc, r in ((hi, better), (lo, better + equal)):
                        if r < top_n:
                            acc[0] += 1
                            acc[1] += 1.0 / (r + 1)
        rr = 0.0
        for r in range(top_n):
            rr += float(hist[r]) / float(r + 1)
        return {'ids': ids, 'hist': hist, 'hits': float(hist[:top_n].sum()), 'rr': rr, 'count': float(hist[top_n]),
                'bounds': (lo[0], hi[0], lo[1], hi[1])}
