"""Host state of the recent-clicks buffer and recent popularity.

Mirror of the hot-path part of the reference class of the same name (nar_module/nar/clicked_items_state.py:10-250):
same constructor, same method names, same arrays.  The update itself (``update_items_state`` :187-250, and the
hook's batch flattening nar_model.py:1635-1646) is ONE C pass in libnar_b200 (``nar_host_state_update[_batch]``,
csrc/host_state.cu, host code, ~40 us per G1 step); there is no numpy fallback - without the library every update
raises.  The numpy specification it is bit-checked against lives with the test infrastructure
(oracle/clicked_items_state_ref.py, pinned to fixtures produced by the reference class itself).
The co-occurrence matrix (:252-255) and the baselines' own state (``benchmarks_states``) are the device pair table of
``baselines.BaselineTables``, kept in ``self.baselines`` when the hook enables baseline recommenders and snapshot /
restored with the rest.  Out of scope (SURVEY.md section 8, row a-14): cold-start bookkeeping (:97-123, :196-203).
"""
from __future__ import annotations

import numpy as np


class ClickedItemsState:

    def __init__(self, recent_clicks_buffer_hours, recent_clicks_buffer_max_size,
                 recent_clicks_for_normalization, num_items):
        self.recent_clicks_buffer_hours = recent_clicks_buffer_hours
        self.recent_clicks_buffer_max_size = recent_clicks_buffer_max_size
        self.recent_clicks_for_normalization = recent_clicks_for_normalization
        self.num_items = num_items
        self.baselines = None                 # baselines.BaselineTables when baseline recommenders are enabled
        self.reset_state()

    def reset_state(self):
        if self.baselines is not None:
            self.baselines.clear()
        self.articles_pop = np.zeros(shape=[self.num_items], dtype=np.int64)
        self.articles_recent_pop = np.zeros(shape=[self.num_items], dtype=np.int64)
        # empty buffer: pop / (0 + 1) floored at 1 / recent_clicks_for_normalization (clicked_items_state.py:240-246)
        self.articles_recent_pop_norm = np.full(self.num_items, 1.0 / self.recent_clicks_for_normalization, dtype=np.float64)
        self.pop_recent_clicks_buffer = np.zeros(shape=[self.recent_clicks_buffer_max_size, 2], dtype=np.int64)
        self.pop_recent_buffer_article_id_column = 0
        self.pop_recent_buffer_timestamp_column = 1
        self.current_step = 0

    # -- checkpoint around eval (clicked_items_state.py:49-79), hot-path fields only
    def save_state_checkpoint(self):
        self.articles_pop_chkp = np.copy(self.articles_pop)
        self.pop_recent_clicks_buffer_chkp = np.copy(self.pop_recent_clicks_buffer)
        self.current_step_chkp = self.current_step
        if self.baselines is not None:
            self.baselines.snapshot()

    def restore_state_checkpoint(self):
        self.articles_pop = self.articles_pop_chkp
        del self.articles_pop_chkp
        self.pop_recent_clicks_buffer = self.pop_recent_clicks_buffer_chkp
        del self.pop_recent_clicks_buffer_chkp
        self.current_step = self.current_step_chkp
        if self.baselines is not None:
            self.baselines.restore()
        # NB: like the reference, recent_pop / recent_pop_norm are NOT restored here;
        # they are recomputed by the next update_items_state().

    # -- getters (clicked_items_state.py:81-108)
    def get_articles_pop(self):
        return self.articles_pop

    def get_articles_recent_pop(self):
        return self.articles_recent_pop

    def get_articles_recent_pop_norm(self):
        return self.articles_recent_pop_norm

    def get_recent_clicks_buffer(self):
        return self.pop_recent_clicks_buffer[:, self.pop_recent_buffer_article_id_column]

    def increment_current_step(self):
        self.current_step += 1

    def get_current_step(self):
        return self.current_step

    def get_max_timestamp_recent_clicks(self):
        return np.max(self.pop_recent_clicks_buffer[:, self.pop_recent_buffer_timestamp_column])

    # -- update (clicked_items_state.py:187-250): the C pass
    @staticmethod
    def _lib():
        from . import _lib as nl
        return nl.load()                      # raises NarError when the library is not built

    def update_items_state(self, batch_clicked_items, batch_clicked_timestamps):
        """One call per step with the batch's non-padded clicks in batch order (what the hook hands over)."""
        lib = self._lib()
        items = np.ascontiguousarray(batch_clicked_items, dtype=np.int64).reshape(-1)
        ts = np.ascontiguousarray(batch_clicked_timestamps, dtype=np.int64).reshape(-1)
        if items.size != ts.size:
            raise ValueError('items / timestamps differ in length')
        if items.size == 0:
            raise ValueError('update_items_state needs at least one click (np.min of an empty batch in the reference)')
        self._call(lambda buf, scratch, recent, norm, pop, hours_ms: lib.nar_host_state_update(
            buf.ctypes.data, buf.shape[0], items.ctypes.data, ts.ctypes.data, items.size, hours_ms, scratch.ctypes.data,
            recent.ctypes.data, norm.ctypes.data, pop.ctypes.data, self.num_items,
            1.0 / self.recent_clicks_for_normalization))

    def update_from_batch(self, clicked_items, clicked_timestamps, last_item_label):
        """ItemsStateUpdaterHook.after_run in one call (nar_model.py:1635-1650): the padded [B,T] batch + [B,1] last
        labels are flattened, padding dropped and folded in, in one pass.  A batch of nothing but padding leaves the
        state alone like the hook does."""
        lib = self._lib()
        ci = np.ascontiguousarray(clicked_items, dtype=np.int64)
        if ci.ndim != 2:
            raise ValueError('clicked_items must be [B, T]')
        ct = np.ascontiguousarray(clicked_timestamps, dtype=np.int64)
        ll = np.ascontiguousarray(last_item_label, dtype=np.int64).reshape(-1)
        B, T = ci.shape
        if ct.shape != (B, T) or ll.shape != (B,):
            raise ValueError('clicked_timestamps must be [B, T] and last_item_label [B, 1]')
        if not (ci.any() or ll.any()):
            return
        bs = getattr(self, '_batch_scratch', None)
        if bs is None or bs.size < 2 * B * (T + 1):
            bs = self._batch_scratch = np.empty(2 * B * (T + 1), dtype=np.int64)
        self._call(lambda buf, scratch, recent, norm, pop, hours_ms: lib.nar_host_state_update_batch(
            buf.ctypes.data, buf.shape[0], ci.ctypes.data, ct.ctypes.data, ll.ctypes.data, B, T, hours_ms, bs.ctypes.data,
            scratch.ctypes.data, recent.ctypes.data, norm.ctypes.data, pop.ctypes.data, self.num_items,
            1.0 / self.recent_clicks_for_normalization))

    def _call(self, fn):
        buf = self.pop_recent_clicks_buffer
        if buf.dtype != np.int64 or not buf.flags['C_CONTIGUOUS'] or not buf.flags['WRITEABLE']:
            buf = np.ascontiguousarray(buf, dtype=np.int64).copy()
        if buf.shape != (self.recent_clicks_buffer_max_size, 2):
            raise ValueError('pop_recent_clicks_buffer must be [recent_clicks_buffer_max_size, 2]')
        scratch = getattr(self, '_scratch', None)
        if scratch is None or scratch.shape != buf.shape:
            scratch = self._scratch = np.empty_like(buf)
        # two alternating output sets: fresh 368 KB arrays per step cost more (page faults) than the update itself, and
        # whoever still holds the previous step's arrays (a feed dict) keeps seeing that step's values
        flip = self._flip = 1 - getattr(self, '_flip', 0)
        outs = getattr(self, '_outs', None)
        if outs is None or outs[0][0].size != self.num_items:
            outs = self._outs = [(np.empty(self.num_items, dtype=np.int64), np.empty(self.num_items, dtype=np.float64))
                                 for _ in range(2)]
        recent, norm = outs[flip]
        pop = self.articles_pop
        if pop.dtype != np.int64 or not pop.flags['C_CONTIGUOUS'] or not pop.flags['WRITEABLE']:
            pop = np.ascontiguousarray(pop, dtype=np.int64).copy()
        hours_ms = int(self.recent_clicks_buffer_hours * 1000 * 60 * 60)
        rc = fn(buf, scratch, recent, norm, pop, hours_ms)
        if rc != 0:
            raise ValueError('nar_host_state_update failed (%d): article id outside [0, num_items)?' % rc)
        self.pop_recent_clicks_buffer = buf
        self.articles_recent_pop = recent
        self.articles_recent_pop_norm = norm
        self.articles_pop = pop


def batch_clicks_for_state_update(clicked_items, clicked_timestamps, last_item_label):
    """ItemsStateUpdaterHook.after_run, train-mode part (nar_model.py:1635-1646): the hook's flattening, for callers
    that hand ``update_items_state`` the reference's way ([B,T] ids / timestamps + [B,1] last label ->
    (items_nonzero, timestamps_nonzero), the last label carrying its session's maximum timestamp)."""
    allc = np.concatenate([clicked_items, last_item_label], axis=1).reshape(-1)
    ts = np.concatenate([clicked_timestamps, np.max(clicked_timestamps, axis=1).reshape(-1, 1)], axis=1).reshape(-1)
    keep = np.nonzero(allc)
    return allc[keep], ts[keep]
