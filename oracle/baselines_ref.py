"""numpy restatement of the five baseline recommenders of the evaluation hook (the reference's
benchmarks/{recently_popular,item_cooccurrences,item_knn,content_based,sequential_rules}.py driven by
nar_model.py:1609-1650), with the tie rules of csrc/baselines.cu:

* pop_recent: count in the recent-clicks buffer desc, then first index in the buffer (Counter.most_common order);
* coocurrent, item_knn, cb: score desc, then the HIGHER article id (a stable sort followed by the reference's [::-1]);
* sr: weight desc, then the order in which the rule past -> active was first inserted (batch, session, i, j).

Tables: co-occurrence = sessions in which (a, c) occur at two different positions of concat(item_clicked,
label_last_item) (each distinct ordered pair once per session, like SciPy's fancy-index +=); sequential rules = sum
of 1/(i-j) over j < i <= j + max_clicks_dist, kept as integers in units of 1/lcm(1..max_clicks_dist).

Per batch the HR / MRR sums are taken from the label's rank histogram in a fixed order (what the device kernel
does), and ``bounds`` gives the pessimistic / optimistic HR and MRR over every order of equal scores.
"""
from __future__ import annotations

import copy
import math
from functools import reduce

import numpy as np

SUFFIXES = ('pop_recent', 'coocurrent', 'item_knn', 'cb', 'sr')


def lcm_upto(n: int) -> int:
    return reduce(lambda x, y: x * y // math.gcd(x, y), range(1, n + 1), 1)


class BaselinesRef:
    def __init__(self, num_items, acr=None, max_clicks_dist=10, reg_lambda=20.0, alpha=0.75):
        self.num_items = num_items
        self.acr = None if acr is None else np.asarray(acr, dtype=np.float64)
        self.D = int(max_clicks_dist)
        self.unit = lcm_upto(self.D)
        self.reg_lambda, self.alpha = float(reg_lambda), float(alpha)
        self.cooc, self.sr_w, self.sr_first = {}, {}, {}
        self.batch_seq = 0

    # ---- tables
    def update(self, all_items):
        all_items = np.asarray(all_items, dtype=np.int64)
        T1 = all_items.shape[1]
        seq = self.batch_seq
        for b, row in enumerate(all_items):
            x = [int(v) for v in row if v != 0]
            pairs = {(x[p], x[q]) for p in range(len(x)) for q in range(len(x)) if p != q}
            for pr in pairs:
                self.cooc[pr] = self.cooc.get(pr, 0) + 1
            for i in range(1, len(x)):
                for j in range(max(0, i - self.D), i):
                    pr = (x[j], x[i])
                    self.sr_w[pr] = self.sr_w.get(pr, 0) + self.unit // (i - j)
                    key = (seq << 32) | ((b * T1 + i) * T1 + j)
                    self.sr_first[pr] = min(self.sr_first.get(pr, key), key)
        self.batch_seq += 1

    def export(self) -> dict:
        keys = sorted(set(self.cooc) | set(self.sr_w))
        big = np.iinfo(np.int64).max
        return {'keys': np.array([(a << 32) | c for a, c in keys], dtype=np.int64),
                'cooc': np.array([self.cooc.get(k, 0) for k in keys], dtype=np.int64),
                'sr_w': np.array([self.sr_w.get(k, 0) for k in keys], dtype=np.int64),
                'sr_first': np.array([self.sr_first.get(k, big) for k in keys], dtype=np.int64)}

    def snapshot(self):
        self._chk = copy.deepcopy((self.cooc, self.sr_w, self.sr_first, self.batch_seq))

    def restore(self):
        self.cooc, self.sr_w, self.sr_first, self.batch_seq = self._chk
        del self._chk

    def cooc_dense(self) -> np.ndarray:
        m = np.zeros((self.num_items, self.num_items), dtype=np.int64)
        for (a, c), v in self.cooc.items():
            m[a, c] = v
        return m

    def sr_rules(self) -> dict:
        return {k: v / self.unit for k, v in self.sr_w.items()}

    # ---- scoring
    def _scores(self, suffix, item, cands, hist_count, hist_first, pop):
        """-> [(score, tie, id)] of the admissible candidates (first occurrence of each id)."""
        out, seen = [], set()
        for c in cands:
            c = int(c)
            if c in seen:
                continue
            seen.add(c)
            if suffix == 'pop_recent':
                if hist_count.get(c, 0) > 0:
                    out.append((float(hist_count[c]), hist_first[c], c))
            elif suffix == 'cb':
                na, nc = np.linalg.norm(self.acr[item]), np.linalg.norm(self.acr[c])
                cos = float(np.dot(self.acr[item], self.acr[c]) / (na * nc)) if na * nc > 0 else 0.0
                out.append((cos, -c, c))
            elif suffix == 'sr':
                w = self.sr_w.get((item, c), 0)
                if w > 0:
                    out.append((float(w), self.sr_first[(item, c)], c))
            else:
                co = self.cooc.get((item, c), 0)
                if co > 0:
                    if suffix == 'coocurrent':
                        out.append((float(co), -c, c))
                    else:
                        norm = np.power(pop[c] + self.reg_lambda, self.alpha) * \
                            np.power(pop[item] + self.reg_lambda, 1.0 - self.alpha)
                        out.append((float(co / norm), -c, c))
        return out

    def candidate_scores(self, suffix, item, cands, buffer_ids, articles_pop) -> dict:
        """{id: score} of the admissible candidates ``cands`` of a query whose current click is ``item``."""
        hc, hf = self._hist(buffer_ids)
        return {c: sc for sc, _, c in self._scores(suffix, int(item), cands, hc, hf, articles_pop)}

    @staticmethod
    def _hist(buffer_ids):
        hist_count, hist_first = {}, {}
        for i, v in enumerate(np.asarray(buffer_ids, dtype=np.int64).reshape(-1).tolist()):
            if v != 0:
                hist_count[v] = hist_count.get(v, 0) + 1
                hist_first.setdefault(v, i)
        return hist_count, hist_first

    def score(self, item_clicked, label_next, negatives, buffer_ids, articles_pop, top_n, suffixes=SUFFIXES) -> dict:
        """One evaluation batch against the current tables -> {suffix: {'ids' [B*T, top_n], 'hist' [top_n+1],
        'hits', 'rr', 'count', 'bounds' (hr_lo, hr_hi, rr_lo, rr_hi) sums}}."""
        item_clicked = np.asarray(item_clicked, dtype=np.int64)
        label_next = np.asarray(label_next, dtype=np.int64)
        negatives = np.asarray(negatives, dtype=np.int64)
        B, T = item_clicked.shape
        hist_count, hist_first = self._hist(buffer_ids)
        res = {}
        for sfx in suffixes:
            ids = np.zeros((B * T, top_n), dtype=np.int64)
            hist = np.zeros(top_n + 1, dtype=np.int64)
            lo = [0.0, 0.0]
            hi = [0.0, 0.0]
            for b in range(B):
                for t in range(T):
                    label = int(label_next[b, t])
                    if label == 0:
                        continue
                    item = int(item_clicked[b, t])
                    cands = [label] + negatives[b, t].tolist()
                    sc = self._scores(sfx, item, cands, hist_count, hist_first, articles_pop)
                    ranked = sorted(sc, key=lambda s: (-s[0], s[1]))
                    top = [s[2] for s in ranked[:top_n]]
                    ids[b * T + t, :len(top)] = top
                    hist[top_n] += 1
                    if label in top:
                        hist[top.index(label)] += 1
                    lab = [s for s in sc if s[2] == label]
                    if lab:
                        better = sum(1 for s in sc if s[0] > lab[0][0])
                        equal = sum(1 for s in sc if s[0] == lab[0][0]) - 1
                        for acc, r in ((hi, better), (lo, better + equal)):
                            if r < top_n:
                                acc[0] += 1
                                acc[1] += 1.0 / (r + 1)
            rr = 0.0
            for r in range(top_n):
                rr += float(hist[r]) / float(r + 1)
            res[sfx] = {'ids': ids, 'hist': hist, 'hits': float(hist[:top_n].sum()), 'rr': rr, 'count': float(hist[top_n]),
                        'bounds': (lo[0], hi[0], lo[1], hi[1])}
        return res
