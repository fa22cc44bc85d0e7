"""Device state of the session-based kNN baseline (the reference's benchmarks/session_knn.py; V-SkNN with the 'div'
decay, suffix ``v-sknn``, SkNN with 'same', suffix ``sknn``): the ring of the last ``sessions_buffer_size`` sessions
(csrc/sknn.cu).  ``baselines.BaselineTables`` owns one ``SessionKNN`` per enabled kNN suffix and calls it on its
streams; the ring's head and entry count are kept here on the host (they follow from the batch sizes, so nothing is
read back)."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from ._lib import check

KNN_SUFFIXES = ('v-sknn', 'sknn')
KNN_DEFAULT_PARAMS = {'sessions_buffer_size': 3000, 'candidate_sessions_sample_size': 1000, 'sampling_strategy': 'recent',
                      'nearest_neighbor_session_for_scoring': 500, 'similarity': 'cosine'}
MAX_SESSIONS = 4096        # ring slots the score kernel's shared memory holds (about 28 bytes per slot)
MAX_T = 64                 # positions of an active session: one bit each of a uint64 mask
WIDTH = 65                 # item slots per ring entry: concat(item_clicked, label_last_item) with T <= 64


def _p(t) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def parse_params(name: str, params: dict) -> dict:
    """Defaults of the reference trainer (nar_trainer_gcom.py:285-292) updated by ``params``, validated."""
    p = dict(KNN_DEFAULT_PARAMS, first_session_clicks_decay='div' if name == 'v-sknn' else 'same')
    p.update({k: v for k, v in params.items() if k in p})
    decay = p['first_session_clicks_decay']
    if decay not in ('same', 'div'):
        raise ValueError("session kNN: only first_session_clicks_decay 'same' (sknn) or 'div' (v-sknn) is supported, "
                         "not %r" % (decay,))
    if ('sknn' if decay == 'same' else 'v-sknn') != name:
        raise ValueError("session kNN: first_session_clicks_decay=%r is the %r baseline, not %r"
                         % (decay, 'sknn' if decay == 'same' else 'v-sknn', name))
    if p['sampling_strategy'] != 'recent':
        raise ValueError("session kNN: only sampling_strategy='recent' is supported (the reference's 'random' draws "
                         "from Python's random module and cannot be reproduced), not %r" % (p['sampling_strategy'],))
    if p['similarity'] not in ('cosine', 'jaccard'):
        raise ValueError("session kNN: similarity must be 'cosine' or 'jaccard', not %r" % (p['similarity'],))
    if not 1 <= int(p['sessions_buffer_size']) <= MAX_SESSIONS:
        raise ValueError('session kNN: sessions_buffer_size must lie in [1, %d] (the scoring kernel keeps one entry per '
                         'buffered session in shared memory), not %r' % (MAX_SESSIONS, p['sessions_buffer_size']))
    for k in ('candidate_sessions_sample_size', 'nearest_neighbor_session_for_scoring'):
        if int(p[k]) < 0:
            raise ValueError('session kNN: %s must be >= 0, not %r' % (k, p[k]))
    return p


class SessionKNN:
    """The ring of one kNN suffix: ids [S] int64, lens [S] int32, items [S, WIDTH] int32 (sorted set, +x live / -x
    discarded from the item -> sessions map), plus staging scratch of the same shape."""

    def __init__(self, suffix: str, params: dict, num_items: int, lib, dev, err):
        self.suffix, self.params = suffix, params
        self.S = int(params['sessions_buffer_size'])
        self.sample_size = int(params['candidate_sessions_sample_size'])
        self.nn = int(params['nearest_neighbor_session_for_scoring'])
        self.decay_div = int(params['first_session_clicks_decay'] == 'div')
        self.jaccard = int(params['similarity'] == 'jaccard')
        self.num_items, self.lib, self.dev, self.err = int(num_items), lib, dev, err
        self.ids = torch.zeros(self.S, dtype=torch.int64, device=dev)
        self.lens = torch.zeros(self.S, dtype=torch.int32, device=dev)
        self.items = torch.zeros(self.S, WIDTH, dtype=torch.int32, device=dev)
        self.st_ids, self.st_lens, self.st_items = (torch.zeros_like(x) for x in (self.ids, self.lens, self.items))
        self.head = 0
        self.count = 0

    def _tensors(self):
        return [self.ids, self.lens, self.items, self.st_ids, self.st_lens, self.st_items]

    def update(self, all_items: torch.Tensor, session_ids: torch.Tensor, stream):
        """Append one batch (``all_items`` [B, T1] int64 device, ``session_ids`` [B] int64 device) on ``stream``."""
        B, T1 = all_items.shape
        if B > self.S:
            raise ValueError('session kNN: a batch of %d sessions does not fit a buffer of %d' % (B, self.S))
        if T1 > WIDTH:
            raise ValueError('session kNN: sessions of more than %d clicks are not supported' % (WIDTH - 1))
        if session_ids.numel() != B:
            raise ValueError('session kNN: %d session ids for a batch of %d sessions' % (session_ids.numel(), B))
        if B == 0:
            return
        for x in self._tensors():
            x.record_stream(stream)
        check(self.lib.nar_sknn_update(*[_p(x) for x in self._tensors()[:3]], self.S, WIDTH, self.head, self.count,
                                       *[_p(x) for x in self._tensors()[3:]], _p(all_items), _p(session_ids), B, T1,
                                       self.num_items, _p(self.err), C.c_void_p(stream.cuda_stream)), 'nar_sknn_update')
        evicted = max(0, self.count + B - self.S)
        self.head = (self.head + evicted) % self.S
        self.count += B - evicted

    def score(self, ic, ln, ng, B, T, K, top_n, metrics_row: torch.Tensor, out_ids, stream):
        """``metrics_row`` [3] fp64 device += {hits, sum of reciprocal ranks, queries}; ``out_ids`` [B*T, top_n] or None."""
        hist = torch.empty(top_n + 1, dtype=torch.int64, device=self.dev)
        check(self.lib.nar_sknn_score(_p(self.ids), _p(self.lens), _p(self.items), self.S, WIDTH, self.head, self.count,
                                      _p(ic), _p(ln), _p(ng), B, T, K, self.num_items, self.sample_size, self.nn,
                                      self.decay_div, self.jaccard, int(top_n), _p(hist), _p(metrics_row), _p(out_ids),
                                      _p(self.err), C.c_void_p(stream.cuda_stream)), 'nar_sknn_score')

    # ---- snapshot / restore / export / load
    def snapshot(self):
        self._chk = (self.ids.clone(), self.lens.clone(), self.items.clone(), self.head, self.count)

    def restore(self):
        self.ids, self.lens, self.items, self.head, self.count = self._chk
        del self._chk

    def clear(self):
        self.head = self.count = 0

    def export(self) -> Dict[str, np.ndarray]:
        """The buffer in insertion order: ids [n], lens [n], items [n, WIDTH] (sorted set, 0-padded), live [n, WIDTH]."""
        idx = (self.head + torch.arange(self.count, device=self.dev)) % self.S
        items = self.items[idx].cpu().numpy().astype(np.int64)
        return {'ids': self.ids[idx].cpu().numpy(), 'lens': self.lens[idx].cpu().numpy().astype(np.int64),
                'items': np.abs(items), 'live': items > 0}

    def load(self, arrays: Dict[str, np.ndarray]):
        """Replace the ring by an exported one (``{}``: empty)."""
        n = int(arrays['ids'].size) if 'ids' in arrays else 0
        if n > self.S:
            raise ValueError('session kNN: a saved buffer of %d sessions does not fit sessions_buffer_size %d' % (n, self.S))
        self.head, self.count = 0, n
        if n:
            items = np.zeros((n, WIDTH), dtype=np.int64)
            w = min(WIDTH, arrays['items'].shape[1])
            signed = np.where(arrays['live'], arrays['items'], -arrays['items'])
            items[:, :w] = signed[:, :w]
            self.ids[:n] = torch.from_numpy(np.ascontiguousarray(arrays['ids'], dtype=np.int64)).to(self.dev)
            self.lens[:n] = torch.from_numpy(np.asarray(arrays['lens'], dtype=np.int32)).to(self.dev)
            self.items[:n] = torch.from_numpy(items.astype(np.int32)).to(self.dev)
