"""The per-session evaluation logs of the reference hook (nar_model.py:1529-1581; trainer flags
``save_eval_sessions_negative_samples`` / ``save_eval_sessions_recommendations``), packed on the GPU.

``SessionLogs`` appends to the two lists the hook was given exactly the dicts the reference appends:

* negatives log: ``{'session_id': str, 'negative_items': [[K ids] per query]}``;
* recommendations log: ``{'session_id': str, 'next_click_labels': [...], 'predicted_item_ids': [[1 + K]],
  'predicted_item_probs': [[1 + K]], 'predicted_item_norm_pop': [[1 + K]]}``

for every session of every batch (empty lists for a session without a query).  Per batch: one kernel
(nar_eval_session_logs_pack) filters, rounds, gathers and packs into one device buffer, one asynchronous copy brings it to
a pinned slot, and the slot becomes Python lists only later - ``drain`` - so the GPU is never held up by it.  Buffer layout,
copy size and what overlaps what: DESIGN.md section 12; spec: oracle/session_logs_ref.py.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from ._lib import check

NEGATIVES, RECOMMENDATIONS = 1, 2          # flag bits of the kernel
_HEADER_WORDS = 4                          # int32 {Q, err, 0, 0}


def _p(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


class SessionLogs:
    """``negatives_log`` / ``recommendations_log``: the lists to append to (None = that log is off; at least one is on)."""

    def __init__(self, num_items: int, device, negatives_log: Optional[list] = None,
                 recommendations_log: Optional[list] = None):
        if negatives_log is None and recommendations_log is None:
            raise ValueError('SessionLogs needs at least one of the two lists')
        self.num_items = int(num_items)
        self.dev = torch.device(device)
        self.negatives_log, self.recommendations_log = negatives_log, recommendations_log
        self.flags = (NEGATIVES if negatives_log is not None else 0) | (RECOMMENDATIONS if recommendations_log is not None else 0)
        self.lib = _lib.load()
        self.packed: Optional[torch.Tensor] = None     # device buffer, sized for B * T queries
        self.slots = [None, None]                      # pinned host copies of it, batch n in slot n & 1
        self.n = 0
        self.pending = None
        self.d2h_bytes = 0                             # bytes of the last batch's device-to-host copy

    def layout(self, B: int, rows: int, K: int) -> np.ndarray:
        """int64 [9]: byte offsets of {counts, neg, labels, ids, probs, pops}, total bytes, Kp, Wp (sections of ``rows``
        rows; nar_eval_session_logs_layout)."""
        o = np.zeros(9, dtype=np.int64)
        check(self.lib.nar_eval_session_logs_layout(int(B), int(rows), int(K), self.flags, C.c_void_p(o.ctypes.data)),
              'nar_eval_session_logs_layout')
        return o

    def begin(self):
        """Start an evaluation: nothing pending, the error flag cleared."""
        self.n, self.pending = 0, None
        if self.packed is not None:
            self.packed[:4 * _HEADER_WORDS].zero_()

    def _ensure(self, nbytes: int):
        if self.packed is None or self.packed.numel() < nbytes:
            self.packed = torch.zeros(nbytes, dtype=torch.uint8, device=self.dev)
            self.slots = [torch.empty(nbytes, dtype=torch.uint8, pin_memory=True) for _ in range(2)]

    def add(self, session_ids, label_next: torch.Tensor, pos_idx: torch.Tensor, sess_off: torch.Tensor, L: int,
            negatives: Optional[torch.Tensor] = None, pred_ids: Optional[torch.Tensor] = None,
            pred_probs: Optional[torch.Tensor] = None, cand: Optional[torch.Tensor] = None, cand_stride: int = 1,
            pop: Optional[torch.Tensor] = None):
        """Queue one batch: ``session_ids`` [B] (host), ``label_next`` [B, T] int64, ``pos_idx`` [>= L] int32 (flat
        b * T + t of compact row r), ``sess_off`` [B + 1] int32, ``negatives`` [B, T, K] int64, ``pred_ids`` /
        ``pred_probs`` [L, 1 + K] int64 / float32 (the ranked candidates of the compact rows), ``cand`` int64 with row r's
        label at ``r * cand_stride``, ``pop`` [num_items] float32 - device tensors, the ones of the enabled logs required.
        Launches the pack kernel and the copy on the current stream, then turns the PREVIOUS batch into list entries."""
        if session_ids is None:
            raise ValueError('the per-session evaluation logs need the session_id feature')
        sids = np.asarray(session_ids).reshape(-1)
        B, T = label_next.shape
        L = int(L)
        assert sids.size == B and sess_off.numel() == B + 1 and label_next.dtype == torch.int64 and label_next.is_contiguous()
        assert pos_idx.dtype == torch.int32 and sess_off.dtype == torch.int32 and pos_idx.numel() >= L
        neg_on, rec_on = bool(self.flags & NEGATIVES), bool(self.flags & RECOMMENDATIONS)
        if L == 0:                                         # no valid position: every session's entry is empty
            self.drain()
            self._append(sids, np.zeros(B, dtype=np.int64), [], [], [], [], [])
            self.n += 1
            self.d2h_bytes = 0
            return
        if neg_on:
            assert negatives is not None and negatives.dtype == torch.int64 and negatives.is_contiguous() and \
                tuple(negatives.shape[:2]) == (B, T)
            K = negatives.shape[2]
        if rec_on:
            assert pred_ids is not None and pred_ids.dtype == torch.int64 and pred_ids.is_contiguous() and \
                pred_ids.shape[0] == L and pred_probs.dtype == torch.float32 and pred_probs.is_contiguous() and \
                pred_probs.shape == pred_ids.shape and cand.dtype == torch.int64 and pop.dtype == torch.float32 and \
                pop.numel() >= self.num_items
            K = pred_ids.shape[1] - 1
        self._ensure(int(self.layout(B, B * T, K)[6]))
        o = self.layout(B, L, K)
        stream = torch.cuda.current_stream(self.dev)
        check(self.lib.nar_eval_session_logs_pack(
            _p(pred_ids), _p(pred_probs), _p(cand), int(cand_stride), _p(pos_idx), _p(sess_off), _p(pop), _p(negatives),
            _p(label_next), B, K, L, self.num_items, self.flags, _p(self.packed), C.c_void_p(stream.cuda_stream)),
            'nar_eval_session_logs_pack')
        # the copy is sized from L, which the host knows: Q <= L, with equality unless a label inside a session is 0
        nbytes = int(o[6])
        slot = self.slots[self.n & 1]
        slot[:nbytes].copy_(self.packed[:nbytes], non_blocking=True)
        copied = torch.cuda.Event()
        copied.record(stream)
        self.d2h_bytes = nbytes
        self.drain()                                       # batch n - 1, now that batch n is queued
        self.pending = (slot, copied, sids, B, L, K, o)
        self.n += 1

    def drain(self):
        """Turn the pending batch's pinned slot into list entries (waits for its copy only).  Raises ValueError when a
        ranked id lay outside [0, num_items)."""
        if self.pending is None:
            return
        slot, copied, sids, B, L, K, o = self.pending
        self.pending = None
        copied.synchronize()
        buf = slot.numpy()
        hdr = buf[:4 * _HEADER_WORDS].view(np.int32)
        Q = int(hdr[0])
        if hdr[1] != 0:
            raise ValueError('session logs: a ranked article id lies outside [0, num_items)')
        counts = buf[o[0]:o[0] + 4 * B].view(np.int32).astype(np.int64)
        Kp, Wp, W = int(o[7]), int(o[8]), K + 1

        def rows(i, dtype, width, keep):
            esz = np.dtype(dtype).itemsize
            return buf[o[i]:o[i] + L * width * esz].view(dtype).reshape(L, width)[:Q, :keep].tolist()

        neg = rows(1, np.int64, Kp, K) if self.flags & NEGATIVES else []
        labels = ids = probs = pops = []
        if self.flags & RECOMMENDATIONS:
            labels = buf[o[2]:o[2] + 8 * L].view(np.int64)[:Q].tolist()
            ids, probs, pops = rows(3, np.int64, Wp, W), rows(4, np.float32, Wp, W), rows(5, np.float32, Wp, W)
        self._append(sids, counts, neg, labels, ids, probs, pops)

    def _append(self, sids, counts, neg, labels, ids, probs, pops):
        ends = np.cumsum(counts).tolist()
        start = 0
        for sid, end in zip(sids.tolist(), ends):
            sid = str(sid)               # the reference: numeric session ids as str, large ints are not serialisable
            if self.negatives_log is not None:
                self.negatives_log.append({'session_id': sid, 'negative_items': neg[start:end]})
            if self.recommendations_log is not None:
                self.recommendations_log.append({'session_id': sid, 'next_click_labels': labels[start:end],
                                                 'predicted_item_ids': ids[start:end],
                                                 'predicted_item_probs': probs[start:end],
                                                 'predicted_item_norm_pop': pops[start:end]})
            start = end

    def end(self):
        self.drain()
