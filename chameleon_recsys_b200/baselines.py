"""Baseline recommenders of the evaluation hook, on the GPU (reference: nar_trainer_gcom.py:280-300,
nar_model.py:1399-1407, 1609-1632, benchmarks/*.py).

``BaselineTables`` owns what the baselines learn from the click stream - one pair table in HBM shared by the
co-occurrence, item-kNN and sequential-rules baselines (csrc/baselines.cu) - and scores every evaluation batch for all
enabled baselines in one launch.  It hangs off the ``ClickedItemsState`` (``state.baselines``) like the reference's
``items_coocurrences`` / ``benchmarks_states``, so ``save_state_checkpoint`` / ``restore_state_checkpoint`` snapshot and
restore it around an evaluation.

Baselines, by the reference's suffixes: ``pop_recent``, ``coocurrent``, ``item_knn`` (``reg_lambda``, ``alpha``), ``cb``
(content-based cosine of the ACR rows), ``sr`` (``max_clicks_dist`` <= 20, ``dist_between_clicks_decay='div'``), and the
session-based kNN baselines ``v-sknn`` (``first_session_clicks_decay='div'``) and ``sknn`` (``'same'``) with the
reference's ``sessions_buffer_size`` (<= 4096), ``candidate_sessions_sample_size``, ``sampling_strategy='recent'``,
``nearest_neighbor_session_for_scoring`` and ``similarity`` ('cosine' / 'jaccard'); each kNN suffix keeps its own ring of
recent sessions (sknn.py, csrc/sknn.cu) and needs the batches' session ids.  Ties, scores and timing: DESIGN.md
section 9.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import check
from .sknn import KNN_SUFFIXES, SessionKNN, parse_params as _knn_params

SUFFIXES = ('pop_recent', 'coocurrent', 'item_knn', 'cb', 'sr')
DEFAULT_PARAMS = {'pop_recent': {}, 'coocurrent': {}, 'item_knn': {'reg_lambda': 20, 'alpha': 0.75}, 'cb': {},
                  'sr': {'max_clicks_dist': 10, 'dist_between_clicks_decay': 'div'}}
_TABLE_USERS = ('coocurrent', 'item_knn', 'sr')
_EMPTY = -1


def parse_classifiers(classifiers) -> Dict[str, dict]:
    """The hook's ``eval_benchmark_classifiers`` list ``[{'recommender': <suffix>, 'params': {...}}]`` (or bare suffixes)
    -> {suffix: params} in request order.  Raises for unknown names and unsupported parameters."""
    out: Dict[str, dict] = {}
    for clf in classifiers:
        name, params = (clf, {}) if isinstance(clf, str) else (clf['recommender'], dict(clf.get('params') or {}))
        if name == 'vsknn':
            raise NotImplementedError("there is no 'vsknn' baseline: the session-based kNN baselines are named by the "
                                      "reference's suffixes, 'v-sknn' (decay 'div') and 'sknn' (decay 'same')")
        if name in KNN_SUFFIXES:
            out[name] = _knn_params(name, params)
            continue
        if name not in SUFFIXES:
            raise ValueError('unknown baseline recommender %r (expected one of %s)'
                             % (name, ', '.join(SUFFIXES + KNN_SUFFIXES)))
        p = dict(DEFAULT_PARAMS[name])
        p.update({k: v for k, v in params.items() if k in p})
        if name == 'sr':
            if p['dist_between_clicks_decay'] != 'div':
                raise ValueError("sequential rules: only dist_between_clicks_decay='div' is supported, not %r"
                                 % (p['dist_between_clicks_decay'],))
            if not 1 <= int(p['max_clicks_dist']) <= 20:
                raise ValueError('sequential rules: max_clicks_dist must lie in [1, 20], not %r' % (p['max_clicks_dist'],))
        out[name] = p
    return out


def _p(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


class BaselineTables:
    """Device state + scoring of the enabled baselines.  ``acr`` [V, ld] float32 device tensor (the engine's resident
    ACR table, first ``acr_dim`` columns used)."""

    def __init__(self, classifiers, num_items: int, acr: Optional[torch.Tensor] = None, acr_dim: int = 0,
                 device=None, capacity: int = 1 << 16):
        self.params = parse_classifiers(classifiers)
        self.enabled: List[str] = list(self.params)
        self.num_items = int(num_items)
        self.dev = torch.device('cuda', torch.cuda.current_device() if device is None else device)
        self.lib = _lib.load()
        self.mask = sum(1 << SUFFIXES.index(s) for s in self.enabled if s in SUFFIXES)
        self.uses_table = any(s in _TABLE_USERS for s in self.enabled)
        # rows of the metrics accumulator: SUFFIXES, then KNN_SUFFIXES when a kNN baseline is enabled
        self.n_rows = len(SUFFIXES) + (len(KNN_SUFFIXES) if any(s in KNN_SUFFIXES for s in self.enabled) else 0)
        sr = self.params.get('sr', DEFAULT_PARAMS['sr'])
        self.max_clicks_dist = int(sr['max_clicks_dist'])
        knn = self.params.get('item_knn', DEFAULT_PARAMS['item_knn'])
        self.reg_lambda, self.alpha = float(knn['reg_lambda']), float(knn['alpha'])
        d = self.dev
        self.err = torch.zeros(1, dtype=torch.int32, device=d)
        self.knn = {s: SessionKNN(s, self.params[s], self.num_items, self.lib, d, self.err)
                    for s in self.enabled if s in KNN_SUFFIXES}
        self.trains = self.uses_table or bool(self.knn)           # some baseline learns from the training batches
        self.acr, self.acr_dim, self.acr_norm = None, int(acr_dim), None
        if 'cb' in self.enabled:
            if acr is None:
                raise ValueError("the 'cb' baseline needs the ACR content matrix")
            self.acr = acr
            self.acr_norm = torch.empty(acr.shape[0], dtype=torch.float64, device=d)
            check(self.lib.nar_baselines_row_norms(_p(acr), acr.shape[0], self.acr_dim, acr.shape[1], _p(self.acr_norm),
                                                   C.c_void_p(torch.cuda.current_stream(d).cuda_stream)),
                  'nar_baselines_row_norms')
        if 'pop_recent' in self.enabled:
            self.hist_count = torch.empty(self.num_items, dtype=torch.int32, device=d)
            self.hist_first = torch.empty(self.num_items, dtype=torch.int32, device=d)
        self._occ_host = torch.zeros(2, dtype=torch.int64).pin_memory()
        self._ready: Optional[torch.cuda.Event] = None
        self.cap = 0
        self._alloc(max(16, 1 << (int(capacity) - 1).bit_length()), torch.cuda.current_stream(d))
        self.batch_seq = 0

    # ---- table storage
    def _alloc(self, cap: int, stream):
        with torch.cuda.stream(stream):
            t = [torch.empty(cap, dtype=torch.int64, device=self.dev) for _ in range(4)]
            self.count = torch.zeros(1, dtype=torch.int64, device=self.dev)
        check(self.lib.nar_baselines_clear(*[_p(x) for x in t], cap, C.c_void_p(stream.cuda_stream)), 'nar_baselines_clear')
        self.keys, self.cooc, self.sr_w, self.sr_first = t
        self.cap = cap
        self._occ = 0              # occupancy known on the host
        self._pending = []         # [(event, slot, pairs of the batches folded after the reading)] since the reading
        self._pairs_since = 0

    def _tables(self):
        return [self.keys, self.cooc, self.sr_w, self.sr_first]

    def _wait(self, stream):
        if self._ready is not None:
            stream.wait_event(self._ready)

    def _mark(self, stream):
        self._ready = torch.cuda.Event()
        self._ready.record(stream)

    def _occupancy_bound(self) -> int:
        """Upper bound of the occupied slots without waiting for the GPU: the newest completed occupancy reading (a
        pinned copy queued behind each update) plus the pairs of every batch folded after it."""
        while self._pending and self._pending[0][0].query():
            ev, slot, pairs_after = self._pending.pop(0)
            self._occ = int(self._occ_host[slot])
            self._pairs_since = pairs_after
        return self._occ + self._pairs_since

    def _grow(self, need: int, stream):
        new_cap = self.cap
        while need > new_cap // 2:
            new_cap *= 2
        if new_cap == self.cap:
            return
        with torch.cuda.stream(stream):
            t = [torch.empty(new_cap, dtype=torch.int64, device=self.dev) for _ in range(4)]
        check(self.lib.nar_baselines_rehash(*[_p(x) for x in self._tables()], self.cap, *[_p(x) for x in t], new_cap,
                                            _p(self.err), C.c_void_p(stream.cuda_stream)), 'nar_baselines_rehash')
        for x in self._tables():
            x.record_stream(stream)           # the old table is freed only after the rehash has read it
        self.keys, self.cooc, self.sr_w, self.sr_first = t
        self.cap = new_cap

    # ---- training: fold one batch
    def update(self, all_items: torch.Tensor, lens: Optional[Sequence[int]] = None, stream=None,
               after: Optional[torch.cuda.Event] = None, session_ids=None):
        """Fold one batch (``all_items`` [Bg, T+1] int64 device = item_clicked | label_last_item) into the pair table and
        the kNN rings on ``stream`` (default: the current stream), after ``after``.  ``lens`` = the sessions' click counts
        (for the growth bound; default T+1 each).  ``session_ids`` [Bg] (host array or tensor) is required when a kNN
        baseline is enabled; host ids go up through a pinned copy on ``stream``.  Queues work only: no host
        synchronisation."""
        if self.knn and session_ids is None:
            raise ValueError('the session kNN baselines (%s) need the batch\'s session ids' % ', '.join(self.knn))
        self.batch_seq += 1
        if not self.trains:
            return
        s = torch.cuda.current_stream(self.dev) if stream is None else stream
        Bg, T1 = all_items.shape
        assert all_items.dtype == torch.int64 and all_items.is_contiguous()
        if after is not None:
            s.wait_event(after)
        self._wait(s)
        if self.knn:
            if torch.is_tensor(session_ids) and session_ids.is_cuda:
                sids = session_ids.to(self.dev, torch.int64).contiguous().view(-1)
            else:
                host = torch.as_tensor(np.ascontiguousarray(np.asarray(session_ids, dtype=np.int64).reshape(-1)))
                with torch.cuda.stream(s):
                    sids = host.pin_memory().to(self.dev, non_blocking=True)
            sids.record_stream(s)
            all_items.record_stream(s)
            for ring in self.knn.values():
                ring.update(all_items, sids, s)
        if not self.uses_table:
            self._mark(s)
            return
        lens = np.full(Bg, T1, dtype=np.int64) if lens is None else np.asarray(lens, dtype=np.int64)
        pairs = int(np.sum(lens * (lens - 1)))
        bound = self._occupancy_bound() + pairs
        if bound > self.cap // 2:
            self._grow(bound, s)
        for x in self._tables() + [self.count]:
            x.record_stream(s)
        all_items.record_stream(s)
        check(self.lib.nar_baselines_update(*[_p(x) for x in self._tables()], self.cap, _p(self.count), _p(all_items), Bg,
                                            T1, self.num_items, self.max_clicks_dist, self.batch_seq - 1, _p(self.err),
                                            C.c_void_p(s.cuda_stream)), 'nar_baselines_update')
        self._pairs_since += pairs
        slot = self.batch_seq & 1
        with torch.cuda.stream(s):
            self._occ_host[slot:slot + 1].copy_(self.count, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(s)
        self._pending.append((ev, slot, 0))
        # pairs folded after this reading: those of later batches (added as they come)
        for i in range(len(self._pending) - 1):
            e, sl, pa = self._pending[i]
            self._pending[i] = (e, sl, pa + pairs)
        self._mark(s)

    # ---- evaluation: score one batch
    def score(self, item_clicked: torch.Tensor, label_next: torch.Tensor, negatives: torch.Tensor, buffer_ids,
              articles_pop, top_n: int, metrics: torch.Tensor, out_ids: Optional[torch.Tensor] = None):
        """Rank label + negatives [B, T, K] of every query (label != 0) for every enabled baseline against the current
        tables, ``buffer_ids`` (recent-clicks buffer) and ``articles_pop``; ``metrics`` [n_rows, 3] fp64 device
        accumulator (rows in SUFFIXES order, then KNN_SUFFIXES when a kNN baseline is enabled) += {hits, sum of
        reciprocal ranks, queries}.  ``out_ids`` [n_rows, B*T, top_n] int64: the top-n ids per query (0-padded).  Runs on
        the current stream."""
        s = torch.cuda.current_stream(self.dev)
        self._wait(s)
        d = self.dev
        B, T = item_clicked.shape
        K = negatives.shape[2] if negatives.dim() == 3 else 0
        assert metrics.dtype == torch.float64 and metrics.numel() >= 3 * self.n_rows
        ic = item_clicked.to(d, torch.int64).contiguous()
        ln = label_next.to(d, torch.int64).contiguous()
        ng = negatives.to(d, torch.int64).contiguous()
        stream = C.c_void_p(s.cuda_stream)
        if 'pop_recent' in self.enabled:
            buf = torch.as_tensor(np.asarray(buffer_ids, dtype=np.int64) if not torch.is_tensor(buffer_ids) else buffer_ids)
            buf = buf.to(d, torch.int64).contiguous().view(-1)
            check(self.lib.nar_baselines_buffer_hist(_p(buf), buf.numel(), self.num_items, _p(self.hist_count),
                                                     _p(self.hist_first), _p(self.err), stream), 'nar_baselines_buffer_hist')
        pop = None
        if 'item_knn' in self.enabled:
            pop = torch.as_tensor(np.asarray(articles_pop, dtype=np.int64) if not torch.is_tensor(articles_pop) else articles_pop)
            pop = pop.to(d, torch.int64).contiguous()
        if out_ids is not None:
            assert out_ids.dtype == torch.int64 and out_ids.shape == (self.n_rows, B * T, top_n) and out_ids.is_contiguous()
        for sfx, ring in self.knn.items():
            row = len(SUFFIXES) + KNN_SUFFIXES.index(sfx)
            ring.score(ic, ln, ng, B, T, K, top_n, metrics.view(-1)[3 * row:3 * row + 3],
                       None if out_ids is None else out_ids[row], s)
        if not self.mask:
            return
        hist = torch.empty(5 * (top_n + 1), dtype=torch.int64, device=d)
        check(self.lib.nar_baselines_score(
            *[_p(x) for x in self._tables()], self.cap, _p(ic), _p(ln), _p(ng), B, T, K,
            _p(getattr(self, 'hist_count', None)), _p(getattr(self, 'hist_first', None)), _p(pop), _p(self.acr),
            self.acr_dim, 0 if self.acr is None else self.acr.shape[1], _p(self.acr_norm), self.num_items, self.reg_lambda,
            self.alpha, self.mask, int(top_n), _p(hist), _p(metrics), _p(out_ids), _p(self.err), stream),
            'nar_baselines_score')

    @staticmethod
    def row(sfx: str) -> int:
        """Row of baseline ``sfx`` in the metrics accumulator and in ``out_ids``."""
        return SUFFIXES.index(sfx) if sfx in SUFFIXES else len(SUFFIXES) + KNN_SUFFIXES.index(sfx)

    def results(self, metrics: torch.Tensor) -> Dict[str, float]:
        """{'hitrate_at_n_<suffix>', 'mrr_at_n_<suffix>'} of the enabled baselines from an [n_rows, 3] accumulator."""
        m = metrics.view(-1, 3).cpu().numpy()
        out = {}
        for sfx in self.enabled:
            h, rr, cnt = m[self.row(sfx)]
            cnt = max(float(cnt), 1.0)
            out['hitrate_at_n_%s' % sfx] = float(h) / cnt
            out['mrr_at_n_%s' % sfx] = float(rr) / cnt
        return out

    # ---- snapshot / restore (ClickedItemsState.save_state_checkpoint / restore_state_checkpoint)
    def snapshot(self):
        s = torch.cuda.current_stream(self.dev)
        self._wait(s)
        self._chk = ([x.clone() for x in self._tables()], self.count.clone(), self.cap, self.batch_seq, self._occ,
                     self._pairs_since, list(self._pending))
        for ring in self.knn.values():
            ring.snapshot()

    def restore(self):
        s = torch.cuda.current_stream(self.dev)
        self._wait(s)
        tabs, cnt, self.cap, self.batch_seq, self._occ, self._pairs_since, self._pending = self._chk
        del self._chk
        self.keys, self.cooc, self.sr_w, self.sr_first = tabs
        self.count = cnt
        for ring in self.knn.values():
            ring.restore()
        self._ready = None

    def clear(self):
        self.batch_seq = 0
        for ring in self.knn.values():
            ring.clear()
        self._alloc(self.cap, torch.cuda.current_stream(self.dev))

    # ---- export / load (checkpoints, tests): occupied entries sorted by key
    def check_errors(self):
        torch.cuda.current_stream(self.dev).synchronize()
        e = int(self.err.item())
        if e == 1:
            raise ValueError('baselines: an article id lies outside [0, num_items)')
        if e == 2:
            raise RuntimeError('baselines: pair table overflow')

    def export(self) -> Dict[str, np.ndarray]:
        s = torch.cuda.current_stream(self.dev)
        self._wait(s)
        self.check_errors()
        occ = self.keys != _EMPTY
        keys, order = torch.sort(self.keys[occ])
        vals = {n: t[occ][order].cpu().numpy() for n, t in (('cooc', self.cooc), ('sr_w', self.sr_w), ('sr_first', self.sr_first))}
        return {'keys': keys.cpu().numpy(), **vals, 'batch_seq': np.asarray(self.batch_seq, dtype=np.int64)}

    def export_knn(self, suffix: str) -> Dict[str, np.ndarray]:
        """The ring of kNN ``suffix`` in insertion order: ids [n], lens [n], items [n, W] (sorted sets, 0-padded), live
        [n, W] (the pair (item, session id) is in the reference's item -> sessions map)."""
        s = torch.cuda.current_stream(self.dev)
        self._wait(s)
        self.check_errors()
        return self.knn[suffix].export()

    def load(self, arrays: Dict[str, np.ndarray]):
        """Replace the tables by exported ones (a kNN ring without saved arrays starts empty)."""
        if self.knn:
            s = torch.cuda.current_stream(self.dev)
            self._wait(s)
            for sfx, ring in self.knn.items():
                pre = 'sknn_%s_' % sfx
                ring.load({k[len(pre):]: v for k, v in arrays.items() if k.startswith(pre)})
            self._mark(s)
        if 'keys' not in arrays:
            self.batch_seq = int(arrays.get('batch_seq', 0))
            return
        n = int(arrays['keys'].size)
        cap = max(16, 1 << (max(1, 2 * n) - 1).bit_length())
        s = torch.cuda.current_stream(self.dev)
        self._wait(s)
        self._alloc(cap, s)
        src = [torch.from_numpy(np.ascontiguousarray(arrays[k], dtype=np.int64)).to(self.dev)
               for k in ('keys', 'cooc', 'sr_w', 'sr_first')]
        if n:
            # the exported entries form a (dense) table of capacity n: rehash them into the new one
            big = 1 << (n - 1).bit_length()
            pad = [torch.cat([x, torch.full((big - n,), v, dtype=torch.int64, device=self.dev)])
                   for x, v in zip(src, (_EMPTY, 0, 0, np.iinfo(np.int64).max))]
            check(self.lib.nar_baselines_rehash(*[_p(x) for x in pad], big, *[_p(x) for x in self._tables()], self.cap,
                                                _p(self.err), C.c_void_p(s.cuda_stream)), 'nar_baselines_rehash')
            self.count.fill_(n)
            self._occ = n
        self.batch_seq = int(arrays.get('batch_seq', 0))
        self._mark(s)

    def state_arrays(self) -> Dict[str, np.ndarray]:
        out = self.export() if self.uses_table else {'batch_seq': np.asarray(self.batch_seq, dtype=np.int64)}
        for sfx in self.knn:
            out.update({'sknn_%s_%s' % (sfx, k): v for k, v in self.export_knn(sfx).items()})
        return out
