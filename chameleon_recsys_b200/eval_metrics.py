"""NDCG, item coverage, ESI-R / ESI-RR novelty and EILD-R / EILD-RR content diversity of the evaluation hook, on the GPU
(the six metrics the reference's ``ItemsStateUpdaterHook.create_eval_metrics`` adds to HR / MRR, nar_model.py:1696-1721,
metrics.py).  Definitions and the reference's quirks: DESIGN.md section 10; spec: oracle/eval_metrics_ref.py.

``EvalMetrics`` accumulates them for several recommenders (rows) over one evaluation: each batch's top-n id lists go in
with ``add_lists`` straight from the device buffers that hold them (the model's ranked candidates, the baselines'
``out_ids``), the batch's clicks with ``add_clicks``, and ``results`` reads the accumulator once at the end.

``ByPosition`` does the same for the hit rate by session position (the reference's ``HitRateBySessionPosition``, switch
``eval_metrics_by_session_position``; DESIGN.md section 11, spec oracle/by_position_ref.py).

``unsampled_results`` turns the integer rank histogram of ``NarEngine.rank_labels`` into the unsampled hit rate, MRR and
NDCG (switch ``eval_unsampled_metrics``; DESIGN.md section 13, spec oracle/unsampled_ref.py).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from ._lib import check

KEYS = ('ndcg_at_n', 'esi-r_at_n', 'esi-rr_at_n', 'content_eild-r_at_n', 'content_eild-rr_at_n')
COVERAGE_KEY = 'item_coverage_at_n'
MAX_TOP_N = 64             # list positions the kernel scores per query
MAX_LIST_SMEM = 200 * 1024 # the list kernel's shared memory per query: top_n^2 fp64 distances, top_n fp32 ACR rows
_N_VALUES = 6              # accumulator columns: the five sums of KEYS, then the query count


def _p(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def metric_names(suffix: str = '') -> list:
    """The result keys of one recommender: no suffix for the model, ``<key>_<suffix>`` for a baseline."""
    return [k + ('_' + suffix if suffix else '') for k in KEYS + (COVERAGE_KEY,)]


def check_params(top_n, neg_relevance):
    if int(top_n) < 2:
        raise ValueError('eval_extended_metrics needs eval_metrics_top_n >= 2 (novelty and diversity average over the '
                         'first top_n - 1 items), not %r' % (top_n,))
    if int(top_n) > MAX_TOP_N:
        raise ValueError('eval_extended_metrics supports eval_metrics_top_n <= %d, not %r' % (MAX_TOP_N, top_n))
    if neg_relevance is None or not float(neg_relevance) > 0:
        raise ValueError('eval_extended_metrics needs eval_negative_sample_relevance > 0, not %r' % (neg_relevance,))


class EvalMetrics:
    """Accumulator of ``rows`` recommenders.  ``acr`` [V, ld] float32 device tensor (first ``acr_dim`` columns used);
    ``acr_norm`` its fp64 row norms when the caller already has them (computed here otherwise)."""

    def __init__(self, rows: int, num_items: int, acr: torch.Tensor, acr_dim: int, top_n: int, neg_relevance: float,
                 acr_norm: Optional[torch.Tensor] = None, err: Optional[torch.Tensor] = None):
        check_params(top_n, neg_relevance)
        smem = 8 * int(top_n) ** 2 + 4 * int(top_n) * int(acr_dim)
        if smem > MAX_LIST_SMEM:
            raise ValueError('eval_extended_metrics holds top_n ACR rows per query in %d bytes of shared memory; top_n %d '
                             'with acr_dim %d needs %d' % (MAX_LIST_SMEM, int(top_n), int(acr_dim), smem))
        self.rows, self.num_items, self.top_n = int(rows), int(num_items), int(top_n)
        self.neg_relevance = float(neg_relevance)
        self.acr, self.acr_dim = acr, int(acr_dim)
        self.dev = acr.device
        self.lib = _lib.load()
        self.words = (self.num_items + 31) // 32
        stream = C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)
        if acr_norm is None:
            acr_norm = torch.empty(acr.shape[0], dtype=torch.float64, device=self.dev)
            check(self.lib.nar_baselines_row_norms(_p(acr), acr.shape[0], self.acr_dim, acr.shape[1], _p(acr_norm), stream),
                  'nar_baselines_row_norms')
        self.acr_norm = acr_norm
        self.err = torch.zeros(1, dtype=torch.int32, device=self.dev) if err is None else err
        self.acc = torch.zeros(self.rows, _N_VALUES, dtype=torch.float64, device=self.dev)
        # bitmaps: the recommended ids of each row, then the clicked ids shared by all rows
        self.bits = torch.zeros(self.rows + 1, self.words, dtype=torch.int32, device=self.dev)
        self._scratch = torch.empty(0, dtype=torch.float64, device=self.dev)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def _mark(self, ids: torch.Tensor, skip_zero: bool):
        ids = ids.to(self.dev, torch.int64).contiguous().view(-1)
        check(self.lib.nar_eval_metrics_mark(_p(ids), ids.numel(), self.num_items, int(skip_zero), _p(self.bits[self.rows]),
                                             _p(self.err), self._stream()), 'nar_eval_metrics_mark')

    def begin(self, buffer):
        """Start an evaluation: zero the sums and the recommended sets; the clicked set = the ids of the recent-clicks
        ``buffer`` (0 included while it holds padding)."""
        self.acc.zero_()
        self.bits.zero_()
        self._mark(torch.as_tensor(buffer), skip_zero=False)

    def add_lists(self, ids: torch.Tensor, labels: torch.Tensor, pop: torch.Tensor, row0: int = 0,
                  row_mask: Optional[int] = None, label_stride: int = 1):
        """Score one batch's lists of the rows ``row0 ..``: ``ids`` [rows, Q, len] or [Q, len] int64 device (the first
        min(top_n, len) ids of a query are its list; NDCG's ideal counts the label over all len), ``labels``
        [Q * label_stride] int64 device (query q's label at q * label_stride; 0 = no query), ``pop`` [V] float32 device
        normalised recent popularity the batch was fed with.  ``row_mask`` (bit r: row row0 + r) defaults to all."""
        ids3 = ids if ids.dim() == 3 else ids.unsqueeze(0)
        rows, nq, length = ids3.shape
        assert ids3.dtype == torch.int64 and ids3.stride(2) == 1 and 0 <= row0 and row0 + rows <= self.rows
        assert labels.dtype == torch.int64 and labels.is_contiguous() and pop.dtype == torch.float32
        if nq == 0:
            return
        mask = (1 << rows) - 1 if row_mask is None else int(row_mask)
        need = rows * nq * _N_VALUES
        if self._scratch.numel() < need:
            self._scratch = torch.empty(need, dtype=torch.float64, device=self.dev)
        s = self._stream()
        check(self.lib.nar_eval_metrics_lists(
            _p(ids3), ids3.stride(0), ids3.stride(1), rows, mask, nq, length, self.top_n, _p(labels), label_stride,
            _p(pop), _p(self.acr), self.acr_dim, self.acr.shape[1], _p(self.acr_norm), self.num_items, self.neg_relevance,
            _p(self._scratch), _p(self.bits[row0]), _p(self.err), s), 'nar_eval_metrics_lists')
        check(self.lib.nar_eval_metrics_reduce(_p(self._scratch), rows, mask, nq, _p(self.acc[row0]), s),
              'nar_eval_metrics_reduce')

    def add_clicks(self, item_clicked: torch.Tensor, label_next: torch.Tensor):
        """The batch's nonzero clicks and next-click labels join the clicked set."""
        self._mark(item_clicked, skip_zero=True)
        self._mark(label_next, skip_zero=True)

    def results(self) -> list:
        """Per row: {KEYS..., COVERAGE_KEY} - the per-query means (nan without queries) and |recommended| / |clicked|;
        plus 'queries', 'recommended' and 'clicked' counts.  Raises ValueError when an id was outside [0, num_items)."""
        counts = torch.empty(self.rows + 1, dtype=torch.int64, device=self.dev)
        check(self.lib.nar_eval_metrics_popcount(_p(self.bits), self.rows + 1, self.words, _p(counts), self._stream()),
              'nar_eval_metrics_popcount')
        acc, counts, err = self.acc.cpu().numpy(), counts.cpu().numpy(), int(self.err.item())
        if err == 1:
            raise ValueError('evaluation metrics: an article id lies outside [0, num_items)')
        clicked = int(counts[self.rows])
        out = []
        for r in range(self.rows):
            q = float(acc[r, _N_VALUES - 1])
            res: Dict[str, float] = {k: (float(acc[r, i]) / q if q else float('nan')) for i, k in enumerate(KEYS)}
            res[COVERAGE_KEY] = int(counts[r]) / clicked if clicked else float('nan')
            res.update(queries=int(q), recommended=int(counts[r]), clicked=clicked)
            out.append(res)
        return out


MAX_POSITIONS = 1024       # session positions (T) the by-position kernel counts per batch
BY_POSITION_KEY = 'hitrate_at_n_by_pos'


def check_by_position_params(top_n):
    if not 1 <= int(top_n) <= MAX_TOP_N:
        raise ValueError('eval_metrics_by_session_position needs 1 <= eval_metrics_top_n <= %d, not %r'
                         % (MAX_TOP_N, top_n))


class ByPosition:
    """Hit rate at n by session position of ``rows`` recommenders over one evaluation.  Position p = t + 1 of a query
    (b, t) with a nonzero label; per row and position the query count and the hits (label among the first n ids of the
    list), and for the lists added with ``pop`` (the model's) the float32 sum of the labels' normalised popularity."""

    def __init__(self, rows: int, num_items: int, top_n: int, device, err: Optional[torch.Tensor] = None):
        check_by_position_params(top_n)
        self.rows, self.num_items, self.top_n = int(rows), int(num_items), int(top_n)
        self.dev = torch.device(device)
        self.lib = _lib.load()
        self.err = torch.zeros(1, dtype=torch.int32, device=self.dev) if err is None else err
        self.counts = torch.zeros(2, self.rows, MAX_POSITIONS, dtype=torch.int64, device=self.dev)   # hits, queries
        self.norm_pop = torch.zeros(MAX_POSITIONS, dtype=torch.float32, device=self.dev)

    def begin(self):
        self.counts.zero_()
        self.norm_pop.zero_()

    def add(self, ids: torch.Tensor, labels: torch.Tensor, T: int, pos_idx: Optional[torch.Tensor] = None,
            sess_off: Optional[torch.Tensor] = None, pop: Optional[torch.Tensor] = None, row0: int = 0,
            row_mask: Optional[int] = None, label_stride: int = 1):
        """Count one batch's lists of the rows ``row0 ..``: ``ids`` [rows, Q, len] or [Q, len] int64 device, ``labels``
        [Q * label_stride] int64 device (0 = no query).  Query q sits at position ``pos_idx[q] % T`` (int32 flat b*T + t,
        the model's compacted rows), or at ``q % T`` without ``pos_idx`` (a [B*T] grid).  ``pop`` [V] float32 device with
        ``sess_off`` [B + 1] int32 (session b's rows start at sess_off[b]): the labels' popularity joins the position
        sums, session by session in order.  ``row_mask`` (bit r: row row0 + r) defaults to all."""
        ids3 = ids if ids.dim() == 3 else ids.unsqueeze(0)
        rows, nq, length = ids3.shape
        assert ids3.dtype == torch.int64 and ids3.stride(2) == 1 and 0 <= row0 and row0 + rows <= self.rows
        assert labels.dtype == torch.int64 and labels.is_contiguous()
        assert pos_idx is None or (pos_idx.dtype == torch.int32 and pos_idx.is_contiguous() and pos_idx.numel() >= nq)
        assert pop is None or (pop.dtype == torch.float32 and sess_off is not None and sess_off.dtype == torch.int32)
        if int(T) > MAX_POSITIONS:
            raise ValueError('eval_metrics_by_session_position counts at most %d session positions, not %d'
                             % (MAX_POSITIONS, T))
        if nq == 0:
            return
        mask = (1 << rows) - 1 if row_mask is None else int(row_mask)
        check(self.lib.nar_eval_by_position(
            _p(ids3), ids3.stride(0), ids3.stride(1), rows, mask, nq, length, self.top_n, _p(labels), label_stride,
            _p(pos_idx), int(T), _p(sess_off), 0 if sess_off is None else sess_off.numel() - 1, _p(pop), self.num_items,
            _p(self.counts[0, row0]), _p(self.counts[1, row0]), MAX_POSITIONS, _p(self.norm_pop), _p(self.err),
            C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)), 'nar_eval_by_position')

    def results(self, names) -> Dict[str, float]:
        """``names`` [(row, suffix)]: ``hitrate_at_n_by_pos[_<suffix>]_PP`` = hits / queries for every position p with a
        query (PP = '%02d' % p); for the empty suffix (the model) also ``clicks_at_pos_PP`` = queries and
        ``avg_norm_pop_by_pos_PP`` = the float32 popularity sum / queries, divided in float32.  Raises ValueError when an
        id was outside [0, num_items)."""
        counts, norm_pop, err = self.counts.cpu().numpy(), self.norm_pop.cpu().numpy(), int(self.err.item())
        if err == 1:
            raise ValueError('evaluation metrics: an article id lies outside [0, num_items)')
        out: Dict[str, float] = {}
        for row, s in names:
            hits, total = counts[0, row], counts[1, row]
            for t in np.flatnonzero(total):
                p, q = int(t) + 1, int(total[t])
                out['%s%s_%02d' % (BY_POSITION_KEY, '_' + s if s else '', p)] = int(hits[t]) / float(q)
                if not s:
                    out['clicks_at_pos_%02d' % p] = q
                    out['avg_norm_pop_by_pos_%02d' % p] = float(np.float32(norm_pop[t]) / np.float32(q))
        return out


# ------------------------------------------------------------------ unsampled hit rate, MRR and NDCG (DESIGN.md section 13)
UNSAMPLED_KEYS = ('unsampled_hitrate_at_n', 'unsampled_mrr_at_n', 'unsampled_ndcg_at_n', 'unsampled_candidates_per_query')


def unsampled_results(hist, top_n: int) -> Dict[str, float]:
    """The unsampled metrics from the integer accumulator of NarEngine.rank_labels (hist [top_n + 2]: the count of each
    rank r < top_n, the ranked queries, their competitors), summed in float64 in rank order: the same bits for any blocking
    and from run to run.  NaN for every key without a query."""
    h = [int(v) for v in np.asarray(hist, dtype=np.int64).reshape(-1)]
    n = int(top_n)
    q = h[n]
    if q == 0:
        return {k: float('nan') for k in UNSAMPLED_KEYS}
    hits = mrr = ndcg = 0.0
    for r in range(n):
        hits += float(h[r])
        mrr += h[r] / (r + 1.0)
        ndcg += h[r] / float(np.log2(r + 2.0))
    return dict(zip(UNSAMPLED_KEYS, (hits / q, mrr / q, ndcg / q, h[n + 1] / q)))


def unsampled_bench_keys(suffix: str):
    """The per-baseline unsampled keys of ``suffix`` (switch ``eval_unsampled_benchmarks``; DESIGN.md section 14)."""
    return tuple('%s_%s' % (k, suffix) for k in UNSAMPLED_KEYS[:3])


def unsampled_bench_results(hist, rows) -> Dict[str, float]:
    """The unsampled metrics of the baselines from their integer accumulator hist [n_rows, top_n + 2] (one row per baseline,
    laid out as NarEngine.rank_labels' histogram): ``rows`` = [(suffix, row)].  -> each baseline's
    ``unsampled_<metric>_at_n_<suffix>`` and ``unsampled_candidates_per_query``, the same for every baseline (they share the
    queries and the competitor sets)."""
    h = np.asarray(hist, dtype=np.int64)
    top_n = h.shape[1] - 2
    out: Dict[str, float] = {}
    for sfx, row in rows:
        r = unsampled_results(h[row], top_n)
        out.update(zip(unsampled_bench_keys(sfx), (r[k] for k in UNSAMPLED_KEYS[:3])))
        out['unsampled_candidates_per_query'] = r['unsampled_candidates_per_query']
    return out
