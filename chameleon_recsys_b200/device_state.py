"""Device-resident ``ClickedItemsState`` (SURVEY.md section 8f #1).

The recent-clicks buffer and the recent-popularity vector live in HBM (two ping-pong slots: the step in flight reads
one while the update for the next step writes the other) and are advanced by one single-CTA kernel per step
(``nar_state_update``, csrc/state.cu) from the batch arrays that are already staged for the step.  Same arithmetic as
the host class (clicked_items_state.py, itself pinned against the reference's).  ``Estimator.train`` keeps the state
here by default (``NarEngine.attach_device_state``; ``NAR_DEVICE_STATE=0`` keeps the hook's host update and its 0.34 MB
per-step upload of buffer + popularity) and writes it back to the host object when training returns.  Covered by
tests/test_device_state.py (runs on a GPU box), bit for bit against oracle/clicked_items_state_ref.py.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import check
from .clicked_items_state import ClickedItemsState


class DeviceClickedItemsState:
    def __init__(self, host: ClickedItemsState, device=None):
        self.dev = torch.device('cuda', torch.cuda.current_device() if device is None else device)
        self.hours_ms = int(host.recent_clicks_buffer_hours * 1000 * 60 * 60)
        self.cap = int(host.recent_clicks_buffer_max_size)
        self.num_items = int(host.num_items)
        self.min_norm = 1.0 / host.recent_clicks_for_normalization
        buf = np.ascontiguousarray(host.pop_recent_clicks_buffer, dtype=np.int64)
        d = self.dev
        self.items = [torch.from_numpy(buf[:, 0].copy()).to(d), torch.zeros(self.cap, dtype=torch.int64, device=d)]
        self.ts = [torch.from_numpy(buf[:, 1].copy()).to(d), torch.zeros(self.cap, dtype=torch.int64, device=d)]
        pn = np.asarray(host.get_articles_recent_pop_norm(), dtype=np.float64)
        self.pop_norm = [torch.from_numpy(pn.astype(np.float32)).to(d), torch.zeros(self.num_items, device=d)]
        self.pop_norm64 = [torch.from_numpy(pn.copy()).to(d), torch.zeros(self.num_items, dtype=torch.float64, device=d)]
        self.recent_pop = torch.from_numpy(np.asarray(host.get_articles_recent_pop(), dtype=np.int64)).to(d)
        self.articles_pop = torch.from_numpy(np.asarray(host.get_articles_pop(), dtype=np.int64).copy()).to(d)
        self.err = torch.zeros(1, dtype=torch.int32, device=d)
        self.cur = 0

    # what the step reads
    def buffer_ids(self) -> torch.Tensor:
        return self.items[self.cur]

    def articles_recent_pop_norm(self) -> torch.Tensor:
        return self.pop_norm[self.cur]

    def update(self, all_items: torch.Tensor, event_ts: torch.Tensor, has_clicks: bool = True, stream=None):
        """Advance the state by one batch: ``all_items`` [Bg,T+1] = [item_clicked | label_last_item], ``event_ts``
        [Bg,T] (device, int64).  ``has_clicks`` False (nothing but padding) leaves the state alone like the hook does."""
        if not has_clicks:
            return
        assert all_items.dtype == torch.int64 and event_ts.dtype == torch.int64 and all_items.is_contiguous() and event_ts.is_contiguous()
        Bg, T1 = all_items.shape
        o, n = self.cur, self.cur ^ 1
        s = torch.cuda.current_stream() if stream is None else stream
        p = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731
        check(_lib.load().nar_state_update(p(self.items[o]), p(self.ts[o]), self.cap, p(all_items), p(event_ts), Bg, T1 - 1,
                                           self.hours_ms, p(self.items[n]), p(self.ts[n]), p(self.recent_pop),
                                           p(self.pop_norm[n]), p(self.pop_norm64[n]), p(self.articles_pop), self.num_items,
                                           self.min_norm, p(self.err), C.c_void_p(s.cuda_stream)), 'nar_state_update')
        self.cur = n

    def to_host(self, host: ClickedItemsState) -> ClickedItemsState:
        """Write the device state back into a host object (checkpoints, evaluation hooks)."""
        torch.cuda.synchronize(self.dev)
        if int(self.err.item()) != 0:
            raise ValueError('nar_state_update saw an article id outside [0, num_items)')
        host.pop_recent_clicks_buffer = np.stack([self.items[self.cur].cpu().numpy(), self.ts[self.cur].cpu().numpy()], axis=1)
        host.articles_recent_pop = self.recent_pop.cpu().numpy()
        host.articles_recent_pop_norm = self.pop_norm64[self.cur].cpu().numpy()
        host.articles_pop = self.articles_pop.cpu().numpy()
        return host
