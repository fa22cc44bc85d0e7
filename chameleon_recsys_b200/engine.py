"""Device engine of the NAR hot path: owns the HBM-resident state (weights, Adam slots, ACR table, metadata), stages
one batch per step and hands the whole step to libnar_b200's C engine (csrc/engine.cu) - ONE call per phase
(``nar_engine_prepare`` / ``nar_engine_step`` / ``nar_engine_apply``) instead of ~50 per-kernel host round trips.
torch = allocator + streams + NCCL plumbing only.

Step order follows the reference graph (nar_module/nar/nar_model.py, SURVEY.md Appendix A):
  sampler (:265-276) -> features (:314-370) -> CAR (:374-405) -> RNN (:408, :1308-1342) ->
  FC1/FC2 (:410-438) -> scorer (:444-517) -> loss (:639-704) -> Adam (:706-722)
with one structural difference: only the valid positions (mask == 1) are materialised.  Padded positions never reach
the loss (:660-664), so skipping them changes no output.  With ``dedup`` (default) the first CAR layer is computed once
per distinct negative id and once per position instead of once per candidate row (csrc/car.cu).

HBM layout of a step: see csrc/engine.cu (row layouts) - all activations live in one workspace the C side carves.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import numpy as np
import torch

from . import ops
from ._lib import FeaturePlanC, ModelCfg, NarError, StepIO, check
from .dp import shard_sessions
from .plan import (SEG_ACR, SEG_CTX_EMBED, SEG_ITEM_EMB, SEG_META_EMBED, FeaturePlan, ParamLayout, round_up)

_NP2T = {np.int64: torch.int64, np.float32: torch.float32, np.int32: torch.int32}


def set_plan_columns(p: FeaturePlanC, pl: FeaturePlan):
    """Write the column part of the C plan ``p`` from ``pl``: the column -> segment map and the column ranges outside the
    wide (vector-copied) segments."""
    if pl.Fp > len(p.col_seg):
        raise NarError('feature rows wider than NAR_MAX_COLS')
    cs = np.full(len(p.col_seg), 255, dtype=np.uint8)
    wide = np.zeros(pl.Fp, dtype=bool)
    for i, s in enumerate(pl.segments):
        cs[s.int_col:s.int_col + s.width] = i
        if s.kind in (SEG_ACR, SEG_ITEM_EMB):
            wide[s.int_col:s.int_col + s.width] = True
    C.memmove(p.col_seg, cs.ctypes.data, len(p.col_seg))
    edges = np.flatnonzero(np.diff(np.concatenate([[True], wide, [True]]).astype(np.int8)))
    ranges = list(zip(edges[0::2], edges[1::2]))
    if len(ranges) > 4:
        raise NarError('more than 4 narrow column ranges')
    p.n_narrow = len(ranges)
    for i, (a, b) in enumerate(ranges):
        p.narrow_begin[i], p.narrow_end[i] = int(a), int(b)


class NarEngine:
    use_side_stream = True          # stage_ahead always stages on the side stream; kept for bench.py, which reads it

    def __init__(self, plan: FeaturePlan, layout: ParamLayout, content_article_embeddings_matrix: np.ndarray,
                 articles_metadata: Dict[str, np.ndarray], *, negative_samples: int, negative_sample_from_buffer: int,
                 softmax_temperature: float, reg_weight_decay: float, lr: float,
                 recent_clicks_buffer_max_size: int, recent_clicks_for_normalization: int,
                 elapsed_days_smooth_log_base: float = 1.3, popularity_smooth_log_base: float = 2.0,
                 ranking: str = 'mlp', rnn_cell: str = 'ugrnn', sampler_seed: int = 42, device: Optional[int] = None,
                 fwd_precision: int = 4, bwd_precision: int = 1, process_group=None, max_batch: int = 0,
                 dedup: bool = True, keep_prob: float = 1.0, novelty_reg_factor: float = 0.0,
                 dropout_seed: Optional[int] = None):
        if not torch.cuda.is_available():
            raise NarError('NarEngine needs a CUDA (sm_90a) device; there is no CPU fallback')
        if rnn_cell not in ('ugrnn', 'gru', 'lstm'):
            raise ValueError("rnn_cell=%r: 'ugrnn' (the reference's UGRNNCell, nar_model.py:1318), 'gru' (GRUCell, :1315) or "
                             "'lstm' (LSTMCell, :1316)" % rnn_cell)
        if rnn_cell != getattr(layout, 'rnn_cell', 'ugrnn'):
            raise ValueError('ParamLayout was built for rnn_cell=%r' % getattr(layout, 'rnn_cell', 'ugrnn'))
        self.rnn_cell = rnn_cell
        if ranking not in ('mlp', 'cosine'):
            raise ValueError(ranking)
        self.dev = torch.device('cuda', torch.cuda.current_device() if device is None else device)
        self.plan, self.layout = plan, layout
        self.K = int(negative_samples)
        self.n_from_buffer = int(negative_sample_from_buffer)
        self.tau = float(softmax_temperature)
        self.reg = float(reg_weight_decay)
        self.lr = float(lr)
        self.buf_len = int(recent_clicks_buffer_max_size)
        self.n_norm = int(recent_clicks_for_normalization)
        self.lb_rec, self.lb_nov = float(elapsed_days_smooth_log_base), float(popularity_smooth_log_base)
        self.ranking = ranking
        self.seed = int(sampler_seed)
        # forward GEMMs: 3 = 3xTF32, 4 = bf16x3 (bf16 hi + lo pieces on the kind::f16 path: same error compensation at twice
        # the tensor rate and 2/3 of the operand bytes; logits within 3e-5 of fp32 instead of 3e-6 - the bar is 1e-3)
        self.fwd_prec, self.bwd_prec = int(fwd_precision), int(bwd_precision)
        self.pg = process_group
        self.world = torch.distributed.get_world_size(process_group) if process_group is not None else 1
        self.rank = torch.distributed.get_rank(process_group) if process_group is not None else 0
        # data parallel: contiguous session shards with equal numbers of valid positions (dp.shard_bounds); 0 = equal session counts
        self.dp_balance = os.environ.get('NAR_DP_BALANCE', '1') == '1'
        self.C, self.H, self.Hp, self.layers = layout.C, layout.H, layout.Hp, layout.layers
        self.V = plan.num_items
        # per-unique-id CAR layer 1 (exact; csrc/car.cu).  dedup=False materialises every candidate row instead.
        self.dedup = bool(dedup)
        # dropout (nar_model.py:338-340, :417-419, :1330-1333): masks are drawn per candidate row, so the rows cannot be
        # shared between candidates - training with keep_prob < 1 materialises every row
        self.keep_prob = float(keep_prob)
        if not (0.0 < self.keep_prob <= 1.0):
            raise ValueError('keep_prob must be in (0, 1]')
        if self.keep_prob < 1.0:
            self.dedup = False
        self.nov_factor = float(novelty_reg_factor)
        self.dropout_seed = self.seed if dropout_seed is None else int(dropout_seed)
        d = self.dev
        # ---- resident tables
        acr = np.zeros((self.V, plan.acr_ld), dtype=np.float32)
        acr[:, :plan.acr_dim] = np.asarray(content_article_embeddings_matrix, dtype=np.float32)
        self.acr = torch.from_numpy(acr).to(d)
        self.created_at = torch.from_numpy(np.asarray(articles_metadata['created_at_ts'], dtype=np.int64)).to(d)
        self.meta = [torch.from_numpy(np.asarray(articles_metadata[n], dtype=np.int64)).to(d) for n in plan.meta_names]
        # ---- parameters (flat fp32 buffers; same offsets for grads / Adam slots)
        n = layout.total
        self.params = torch.zeros(n, device=d)
        # gradients and the 4 loss accumulators share ONE buffer, so that data parallel needs a single collective per step
        self._grads_ext = torch.zeros(n + 4, device=d)
        self.grads = self._grads_ext[:n]
        self.adam_m = torch.zeros(n, device=d)
        self.adam_v = torch.zeros(n, device=d)
        self.params_lo = torch.zeros(n, device=d)      # w - tf32_trunc(w): B_lo plane of the 3xTF32 forward GEMMs
        self.global_step = 0
        self.loss_dev = self._grads_ext[n:]               # [xe, l2 regulariser, novelty regulariser, -]: total = [0] + [1] - [2]
        self._loss_hosts = [torch.zeros(4).pin_memory() for _ in range(2)]   # two in flight: submit(n+1) before result(n)
        self._loss_slot = 0
        self.loss_host = torch.zeros(4).pin_memory()      # eval_step's own: an evaluation never overwrites an unread step
        self._bufs: Dict[str, torch.Tensor] = {}
        self._pinned: Dict[str, torch.Tensor] = {}
        self._side = None
        self._prep_flip = 0
        self._slot_events: Dict[str, torch.cuda.Event] = {}       # prepare() slot -> end of the last step that read it
        self._pin_events: Dict[str, torch.cuda.Event] = {}        # staging slot -> its last H2D copy
        self.use_aux_stream = True
        self._views: dict = {}
        self.last: Dict[str, torch.Tensor] = {}
        self.ops = ops
        self._ctx = ops.context(self.dev.index)     # fail loudly here if the library / device is unusable
        self._lib = self._ctx.lib
        # step workspaces: sized for the worst case (every position valid) when that fits the budget, else grown.  Default
        # budget: a quarter of the device (20 GB on an 80 GB H100), so that a worst-case workspace plus the superseded ones
        # a regrowth keeps alive leave room for weights, Adam slots and the caching allocator
        budget = os.environ.get('NAR_WS_BUDGET_GB')
        self._ws_budget = (int(float(budget) * (1 << 30)) if budget else
                           torch.cuda.get_device_properties(self.dev).total_memory // 4)
        self._L_cap = 0
        self._ws: Optional[torch.Tensor] = None
        self._prep_ws: Dict[str, torch.Tensor] = {}
        self._old = []                                # superseded workspaces, kept until the steps using them are done
        self.dstate = None                            # DeviceClickedItemsState when the recent-clicks state lives in HBM
        self._handle = C.c_void_p()
        self._cfg = self._make_cfg()
        check(self._lib.nar_engine_create(self._ctx.handle, C.byref(self._cfg), C.byref(self._handle)), 'nar_engine_create')
        self._cfg_key = self._dynamic_key()

    def __del__(self):
        try:
            if getattr(self, '_handle', None):
                torch.cuda.synchronize(self.dev)
                self._lib.nar_engine_destroy(self._handle)
                self._handle = None
        except Exception:  # noqa: BLE001
            pass

    # ------------------------------------------------------------------ C-side configuration
    def _dynamic_key(self):
        return (self.use_aux_stream, self.world, self.rank, self.lr, self.fwd_prec, self.bwd_prec, self.dedup,
                self.params.data_ptr(), self.params_lo.data_ptr(), self.K, self.n_from_buffer, self.keep_prob, self.nov_factor)

    def _make_cfg(self) -> ModelCfg:
        lay, pl = self.layout, self.plan
        c = ModelCfg()
        c.num_items, c.C, c.Hp, c.Fp, c.ctx_col0 = self.V, self.C, self.Hp, pl.Fp, pl.ctx_col0
        c.layers, c.rnn_cell, c.ranking = self.layers, {'ugrnn': 0, 'gru': 1, 'lstm': 2}[self.rnn_cell], 0 if self.ranking == 'mlp' else 1
        c.fwd_precision, c.bwd_precision = self.fwd_prec, self.bwd_prec
        c.dedup, c.use_aux_stream = int(self.dedup), int(self.use_aux_stream)
        c.keep_prob, c.novelty_reg_factor = self.keep_prob, self.nov_factor
        c.dropout_seed = self.dropout_seed & 0xFFFFFFFFFFFFFFFF
        c.K, c.n_from_buffer, c.buf_len, c.n_norm = self.K, self.n_from_buffer, self.buf_len, self.n_norm
        c.inv_temperature, c.reg_l2, c.lr = 1.0 / self.tau, self.reg, self.lr
        c.beta1, c.beta2, c.eps = 0.9, 0.999, 1e-8
        c.sampler_seed = self.seed & 0xFFFFFFFFFFFFFFFF
        c.world, c.rank = self.world, self.rank
        c.params, c.params_lo, c.grads = self.params.data_ptr(), self.params_lo.data_ptr(), self.grads.data_ptr()
        c.adam_m, c.adam_v = self.adam_m.data_ptr(), self.adam_v.data_ptr()
        c.n_params, c.reg_end = lay.total, lay.reg_end
        off = lambda k: lay.by_key[k].offset      # noqa: E731
        c.off_W1, c.off_b1, c.off_W2, c.off_b2 = off('W1'), off('b1'), off('W2'), off('b2')
        c.off_W3, c.off_b3, c.off_W4, c.off_b4 = off('W3'), off('b3'), off('W4'), off('b4')
        c.off_gamma, c.off_beta = off('gamma'), off('beta')
        for i in range(4):
            c.off_M[i], c.off_c[i], c.ld_M[i] = off('M%d' % (i + 1)), off('c%d' % (i + 1)), lay.by_key['M%d' % (i + 1)].ld
        for i in range(self.layers):
            c.off_Wx[i], c.off_Wh[i], c.off_rb[i] = off('rnn%d/Wx' % i), off('rnn%d/Wh' % i), off('rnn%d/b' % i)
            if self.rnn_cell == 'gru':
                c.off_Whc[i] = off('rnn%d/Whc' % i)
        c.plan = self._plan_c_static()
        return c

    def _sync_cfg(self):
        """Push attribute changes (tests flip use_aux_stream / world / rank / precisions on a live engine)."""
        key = self._dynamic_key()
        if key != self._cfg_key:
            if self.dedup != bool(self._cfg.dedup):
                self._ws = None; self._prep_ws = {}; self._L_cap = 0          # different carve
            self._cfg = self._make_cfg()
            check(self._lib.nar_engine_update_cfg(self._handle, C.byref(self._cfg)), 'nar_engine_update_cfg')
            self._cfg_key = key

    def _refresh(self):
        """Weights were written from outside the engine: rebuild what the C side derives from them (bf16x3 planes)."""
        if getattr(self, '_handle', None):
            self._sync_cfg()
            check(self._lib.nar_engine_refresh(self._handle, C.c_void_p(torch.cuda.current_stream().cuda_stream)), 'nar_engine_refresh')

    # ------------------------------------------------------------------ parameters
    def view(self, key: str, buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        b = self.params if buf is None else buf
        ck = (key, b.data_ptr())
        v = self._views.get(ck)
        if v is None:
            t = self.layout.by_key[key]
            v = b[t.offset:t.offset + t.size].view(t.rows, t.ld)
            self._views[ck] = v
        return v

    def set_params(self, logical: Dict[str, np.ndarray]):
        flat = self.layout.to_internal(logical)
        self.params.copy_(torch.from_numpy(flat))
        self.adam_m.zero_(); self.adam_v.zero_(); self.grads.zero_()
        ops.tf32_lo(self.params, self.layout.total, self.params_lo)
        self._refresh()
        self.global_step = 0

    def get_params(self) -> Dict[str, np.ndarray]:
        return self.layout.to_logical(self.params.detach().cpu().numpy())

    def get_grads(self) -> Dict[str, np.ndarray]:
        return self.layout.to_logical(self.grads.detach().cpu().numpy())

    def state_dict(self) -> dict:
        return {'params': self.layout.to_logical(self.params.cpu().numpy()),
                'adam_m': self.layout.to_logical(self.adam_m.cpu().numpy()),
                'adam_v': self.layout.to_logical(self.adam_v.cpu().numpy()),
                'global_step': self.global_step}

    def load_logical_state(self, params, adam_m, adam_v, global_step: int):
        """Set weights + Adam slots from logical (TF-shaped) dicts, e.g. to start a parity step from a given state."""
        self.load_state_dict({'params': params, 'adam_m': adam_m, 'adam_v': adam_v, 'global_step': global_step})

    def load_state_dict(self, sd: dict):
        self.params.copy_(torch.from_numpy(self.layout.to_internal(sd['params'])))
        self.adam_m.copy_(torch.from_numpy(self.layout.to_internal(sd['adam_m'])))
        self.adam_v.copy_(torch.from_numpy(self.layout.to_internal(sd['adam_v'])))
        self.global_step = int(sd['global_step'])
        ops.tf32_lo(self.params, self.layout.total, self.params_lo)
        self._refresh()

    # ------------------------------------------------------------------ buffers
    def _buf(self, name: str, rows: int, cols: int, dtype=torch.float32, cap_rows: int = 0) -> torch.Tensor:
        """Named device buffer, grown by 1.25x; ``cap_rows`` = the most rows it can ever need: allocated once at that size
        when given (a reallocation inside the training loop is a device-wide sync)."""
        need = max(1, rows) * cols
        t = self._bufs.get(name)
        if t is None or t.numel() < need or t.dtype != dtype:
            cap = max(int(need * 1.25) + 1024, max(1, cap_rows) * cols)
            t = torch.empty(cap, device=self.dev, dtype=dtype)
            self._bufs[name] = t
        return t[:max(1, rows) * cols].view(max(1, rows), cols)

    def _pin(self, name: str, nbytes: int) -> torch.Tensor:
        t = self._pinned.get(name)
        if t is None or t.numel() < nbytes:
            t = torch.empty(int(nbytes * 1.25) + 4096, dtype=torch.uint8).pin_memory()
            self._pinned[name] = t
        return t

    def _ws_bytes(self, Bg, B, T, L_cap, train=True):
        pb, wb = C.c_int64(0), C.c_int64(0)
        check(self._lib.nar_engine_workspace_bytes(self._handle, Bg, B, T, L_cap, 1 if train else 0, C.byref(pb), C.byref(wb)),
              'nar_engine_workspace_bytes')
        return int(pb.value), int(wb.value)

    def _ensure_capacity(self, Bg: int, B: int, T: int, L: int, slot: str):
        """Workspaces for a step with L valid positions.  Sized once for the worst case (all B*T positions valid) when
        that fits the workspace budget (G1 at its per-GPU batch: 8 GB, within the 20 GB default on an 80 GB H100); beyond
        that (stress shapes) sized for 1.25x the largest L seen - a regrowth keeps the superseded buffers alive until
        the steps that use them are done.  Allocated on the current (main) stream's pool."""
        self._sync_cfg()
        cap = self._L_cap
        if cap < max(L, 1) or self._ws is None:
            worst = B * T
            _, wb = self._ws_bytes(Bg, B, T, worst, True)
            # (1.5x head-room: a regrowth is a multi-GB cudaMalloc, i.e. a stall of several ms in the middle of the loop)
            cap = worst if wb <= self._ws_budget else max(self._L_cap, min(worst, int(L * 1.5) + 64))
            if cap != self._L_cap:
                self._old.append((self._ws, dict(self._prep_ws)))
                self._old = self._old[-3:]
                self._ws, self._prep_ws = None, {}
            self._L_cap = cap
        pb, wb = self._ws_bytes(Bg, B, T, cap, True)
        if self._ws is None or self._ws.numel() < wb:
            self._ws = torch.empty(wb, dtype=torch.uint8, device=self.dev)
        p = self._prep_ws.get(slot)
        if p is None or p.numel() < pb:
            # torch.empty, NOT zeros: a fill kernel would be queued on the CURRENT (main) stream behind the running step
            # and land after the side-stream prepare has written its results (found as an illegal address in the 2-GPU
            # bench: the pool kernel's key arrays were wiped under it).  Everything in here is written before it is read.
            p = torch.empty(pb, dtype=torch.uint8, device=self.dev)
            self._prep_ws[slot] = p
        return cap, p, self._ws

    # ------------------------------------------------------------------ device-resident ClickedItemsState (SURVEY 8f #1)
    def attach_device_state(self, host_state):
        """Move the recent-clicks buffer / recent popularity into HBM (device_state.py, csrc/state.cu): from now on
        ``stage(..., buffer=None, pop_norm=None)`` uploads neither (0.34 MB per G1 step) and ``advance_device_state``
        folds a staged batch in on the device - no host pass, no per-step upload.  ``detach_device_state`` writes the
        state back into the host object (checkpoints, evaluation hooks)."""
        from .device_state import DeviceClickedItemsState
        self.dstate = DeviceClickedItemsState(host_state, device=self.dev.index)
        self._dstate_host = host_state
        # its buffers were initialised on the current stream: the side stream must not touch them earlier
        self._dstate_ready = torch.cuda.Event()
        self._dstate_ready.record()
        return self.dstate

    def detach_device_state(self):
        if self.dstate is not None:
            self.dstate.to_host(self._dstate_host)
            self.dstate = None

    def advance_device_state(self, st: dict, stream: Optional[torch.cuda.Stream] = None):
        """ItemsStateUpdaterHook.after_run on the device: fold the clicks of the batch staged in ``st`` into the state
        (depends on the batch's ids / timestamps only, so it may run on the side stream right behind the batch's copy)."""
        if self.dstate is None:
            raise NarError('no device state attached')
        t = st['t']
        self.dstate.update(t['all_items'], t['event_ts'], has_clicks=st['has_clicks'], stream=stream)

    # ------------------------------------------------------------------ staging (host -> HBM, one copy)
    def stage(self, features: Dict[str, np.ndarray], labels: Dict[str, np.ndarray], buffer: Optional[np.ndarray],
              pop_norm: Optional[np.ndarray], slot: str = 'stage', stream: Optional[torch.cuda.Stream] = None) -> dict:
        """Pack the step inputs into one pinned buffer and issue one async H2D copy.
        ``features``/``labels`` hold the GLOBAL batch (all data-parallel ranks see the same arrays).  ``buffer`` /
        ``pop_norm`` None: the device-resident state is read instead (attach_device_state)."""
        item_clicked = np.ascontiguousarray(features['item_clicked'], dtype=np.int64)
        Bg, T = item_clicked.shape
        use_dstate = buffer is None
        if use_dstate:
            if self.dstate is None:
                raise NarError('stage(buffer=None) needs attach_device_state()')
        else:
            buffer = np.asarray(buffer)
            if buffer.size != self.buf_len:
                raise ValueError('recent-clicks buffer has %d entries, engine was built for %d' % (buffer.size, self.buf_len))
        # this rank's sessions + compact valid positions (session-major; flat index into the GLOBAL [Bg*T] arrays)
        sh = shard_sessions(np.asarray(features['session_size']), T, self.world, self.rank, balance=self.dp_balance)
        s0, per, lens, L, L_global = sh['s0'], sh['per'], sh['lens'], sh['L'], sh['L_global']
        sess_off, pos_idx = sh['sess_off'], sh['pos_idx']
        all_items = np.concatenate([item_clicked, np.asarray(labels['label_last_item'], dtype=np.int64).reshape(Bg, 1)], axis=1)
        ev = np.ascontiguousarray(features['event_timestamp'], dtype=np.int64)
        parts = [('all_items', all_items, np.int64), ('event_ts', ev, np.int64),
                 ('item_clicked', item_clicked, np.int64),
                 ('label_next', np.ascontiguousarray(labels['label_next_item'], dtype=np.int64), np.int64),
                 ('max_ts', np.asarray([ev.max() if ev.size else 0], dtype=np.int64), np.int64)]
        if not use_dstate:
            parts.append(('buffer', np.ascontiguousarray(buffer, dtype=np.int64), np.int64))
        for name in self.plan.ctx_int_names:
            parts.append(('ci/' + name, np.ascontiguousarray(features[name], dtype=np.int64), np.int64))
        if not use_dstate:
            parts.append(('pop_norm', np.ascontiguousarray(pop_norm, dtype=np.float32), np.float32))
        for name in self.plan.ctx_float_names:
            parts.append(('cf/' + name, np.ascontiguousarray(features[name], dtype=np.float32), np.float32))
        parts.append(('pos_idx', pos_idx if pos_idx.size else np.zeros(1, np.int32), np.int32))
        parts.append(('sess_off', sess_off, np.int32))
        offs, off = {}, 0
        for name, arr, dt in parts:
            off = round_up(off, 16)
            offs[name] = (off, arr.size, dt, arr.shape)
            off += arr.size * np.dtype(dt).itemsize
        total = round_up(off, 16)
        # pos_idx and (balanced shards: `per` varies) sess_off are the only parts whose size varies step to step
        worst = total + 4 * (Bg * T - pos_idx.size) + 4 * (Bg - per) + 64
        pin = self._pin(slot, worst)
        busy = self._pin_events.get(slot)
        if busy is not None:
            busy.synchronize()                # the previous H2D copy out of this pinned slot (issued >= 2 steps ago) is done
        pin_np = pin.numpy()
        for name, arr, dt in parts:
            o, nel, _, _ = offs[name]
            pin_np[o:o + nel * np.dtype(dt).itemsize].view(dt)[:] = arr.reshape(-1)
        dev = self._buf(slot, total, 1, torch.uint8, cap_rows=worst).view(-1)
        copy_stream = stream if stream is not None else torch.cuda.current_stream()
        with torch.cuda.stream(copy_stream):
            dev[:total].copy_(pin[:total], non_blocking=True)
        copied = torch.cuda.Event()
        copied.record(copy_stream)
        self._pin_events[slot] = copied
        self._last_copied = copied
        tens = {}
        for name, (o, nel, dt, shp) in offs.items():
            tens[name] = dev[o:o + nel * np.dtype(dt).itemsize].view(_NP2T[dt]).view(*shp) if nel > 0 else \
                torch.zeros(shp, dtype=_NP2T[dt], device=self.dev)
        return {'t': tens, 'Bg': Bg, 'B': per, 'T': T, 'L': L, 'L_global': L_global, 's0': s0,
                'h2d_bytes': total, 'lens': lens, 'slot': slot, 'dstate': use_dstate, 'has_clicks': bool(all_items.any()),
                'copied': copied}

    # ------------------------------------------------------------------ feature plan (static part)
    def _plan_c_static(self) -> FeaturePlanC:
        p = FeaturePlanC()
        pl = self.plan
        p.n_segments = len(pl.segments)
        p.row_ld = pl.Fp
        for i, s in enumerate(pl.segments):
            sg = p.seg[i]
            sg.kind, sg.col, sg.width, sg.card, sg.src = s.kind, s.int_col, s.width, s.card, s.src
            sg.ld, sg.table, sg.grad = 0, None, None
            if s.kind == SEG_ACR:
                sg.ld, sg.table = pl.acr_ld, self.acr.data_ptr()
            elif s.kind in (SEG_ITEM_EMB, SEG_CTX_EMBED, SEG_META_EMBED):
                pt = self.layout.by_key[s.param]
                sg.ld = pt.ld
                sg.table = self.params.data_ptr() + 4 * pt.offset
                sg.grad = self.grads.data_ptr() + 4 * pt.offset
        for i, m in enumerate(self.meta):
            p.meta[i] = m.data_ptr()
        p.created_at_ts = self.created_at.data_ptr()
        p.gamma = self.view('gamma').data_ptr()
        p.beta = self.view('beta').data_ptr()
        p.log_base_recency, p.log_base_novelty = self.lb_rec, self.lb_nov
        set_plan_columns(p, pl)
        return p

    def feature_plan_c(self, st: dict) -> FeaturePlanC:
        """Per-step plan for callers that launch the gather kernel themselves (micro-benchmarks): the static part + this
        step's staged input pointers + the statistics written by prepare()."""
        p = FeaturePlanC.from_buffer_copy(bytes(self._cfg.plan))
        io = st['prep']['io']
        p.ctx_int, p.ctx_float, p.pop_norm = io.ctx_int, io.ctx_float, io.pop_norm
        p.stats = self.buffer(st, 'stats').data_ptr()
        return p

    # ------------------------------------------------------------------ the step
    def _staged_io(self, st: dict) -> StepIO:
        """A StepIO holding the inputs staged in ``st``: dims, ids, timestamps, labels, the recent-clicks state and the
        context features.  Train, evaluate and predict all start from it."""
        t = st['t']
        io = StepIO()
        io.B, io.Bg, io.T, io.sess0, io.L, io.L_global = st['B'], st['Bg'], st['T'], st['s0'], st['L'], st['L_global']
        io.all_items, io.event_ts = t['all_items'].data_ptr(), t['event_ts'].data_ptr()
        io.item_clicked, io.label_next = t['item_clicked'].data_ptr(), t['label_next'].data_ptr()
        if st['dstate']:
            # the state as of NOW: every update of an earlier batch has been queued (stream order does the rest)
            buf_t, pop_t = self.dstate.buffer_ids(), self.dstate.articles_recent_pop_norm()
            st['_hold_state'] = (buf_t, pop_t)
        else:
            buf_t, pop_t = t['buffer'], t['pop_norm']
        io.buffer, io.max_ts, io.pop_norm = buf_t.data_ptr(), t['max_ts'].data_ptr(), pop_t.data_ptr()
        for i, n in enumerate(self.plan.ctx_int_names):
            io.ctx_int[i] = t['ci/' + n].data_ptr()
        for i, n in enumerate(self.plan.ctx_float_names):
            io.ctx_float[i] = t['cf/' + n].data_ptr()
        io.pos_idx, io.sess_off = t['pos_idx'].data_ptr(), t['sess_off'].data_ptr()
        return io

    def _make_io(self, st: dict, slot: str, sampler_step: int) -> StepIO:
        cap, prep_ws, ws = self._ensure_capacity(st['Bg'], st['B'], st['T'], st['L'], slot)
        io = self._staged_io(st)
        io.L_cap = cap
        io.global_step = self.global_step
        io.sampler_step = int(sampler_step) & 0xFFFFFFFF
        io.train = 1                        # the carve of a training step is a superset: evaluation reuses the same offsets
        io.prep_ws, io.prep_ws_bytes = prep_ws.data_ptr(), prep_ws.numel()
        io.ws, io.ws_bytes = ws.data_ptr(), ws.numel()
        io.loss = self.loss_dev.data_ptr()
        st['_hold'] = (prep_ws, ws)         # keep the buffers this io points into alive with the staged batch
        return io

    def prepare(self, st: dict, step_id: int, stream: Optional[torch.cuda.Stream] = None) -> dict:
        """Everything of a step that does not depend on the weights: negatives (nar_model.py:265-276), the row
        lists, the recency / novelty statistics and (dedup) the base rows.  May run one step AHEAD on a side stream
        (``stream``) while the previous step's GEMMs occupy the SMs - the reference's tf.data prefetch(1) gives the same
        look-ahead (datasets.py:142).  Results live in per-slot workspaces and are handed over through a CUDA event."""
        if stream is not None:
            self._prep_flip ^= 1
        slot = ('/ahead%d' % self._prep_flip) if stream is not None else ''
        cur = torch.cuda.current_stream()
        run_on = stream if stream is not None else cur
        io = self._make_io(st, slot, step_id)
        # two result slots alternate: the step that consumed this slot two prepare() calls ago may still be running (its
        # gather backward reads the row lists at the very end), so the side stream waits for that step's end first
        last_use = self._slot_events.get(slot) if stream is not None else None
        if last_use is not None:
            run_on.wait_event(last_use)
        check(self._lib.nar_engine_prepare(self._handle, C.byref(io), C.c_void_p(run_on.cuda_stream)), 'nar_engine_prepare')
        ev = None
        if stream is not None:
            ev = torch.cuda.Event()
            ev.record(run_on)
        st['prep'] = {'io': io, 'event': ev, 'step_id': step_id, 'slot': slot}
        return st

    _INT_BUFFERS = {'neg': torch.int64, 'row_item': torch.int64, 'base_item': torch.int64, 'neg_uidx': torch.int32,
                    'row_pos': torch.int32, 'base_pos': torch.int32}

    def buffer(self, st: dict, name: str) -> torch.Tensor:
        """Device view of a named intermediate of the step staged in ``st`` (see nar_engine_buffer)."""
        io = st['prep']['io']
        ptr, rows, ld = C.c_void_p(), C.c_int64(0), C.c_int64(0)
        check(self._lib.nar_engine_buffer(self._handle, C.byref(io), name.encode(), C.byref(ptr), C.byref(rows), C.byref(ld)),
              'nar_engine_buffer(%s)' % name)
        dt = self._INT_BUFFERS.get(name, torch.float32)
        esz = torch.empty((), dtype=dt).element_size()
        for owner in st['_hold']:
            o = ptr.value - owner.data_ptr()
            if 0 <= o < owner.numel():
                n = rows.value * ld.value
                return owner[o:o + n * esz].view(dt).view(rows.value, ld.value)
        raise NarError('buffer %s is outside the step workspaces' % name)

    def step(self, st: dict, train: bool = True, keep: bool = False) -> dict:
        """Run one step on staged inputs (ONE C call).  Returns device tensors (loss parts, logits, negatives)."""
        step_id = self.global_step + 1
        prep = st.get('prep')
        if prep is None or prep['step_id'] != step_id:
            prep = self.prepare(st, step_id)['prep']          # inline, on the current stream
        self._sync_cfg()
        cur = torch.cuda.current_stream()
        if prep['event'] is not None:
            cur.wait_event(prep['event'])
        io = prep['io']
        io.train = 1 if train else 0
        io.global_step = self.global_step
        B, T, L, K = st['B'], st['T'], st['L'], self.K
        check(self._lib.nar_engine_step(self._handle, C.byref(io), C.c_void_p(cur.cuda_stream)), 'nar_engine_step')
        io.train = 1
        neg = self.buffer(st, 'neg').view(-1)[st['s0'] * T * K:(st['s0'] + B) * T * K].view(B, T, K)
        out = {'negatives': neg, 'L': L, 'loss': self.loss_dev, 'logits': self.buffer(st, 'logits') if L > 0 else None}
        if keep and L > 0:
            self.last = self._collect(st, train)
        if prep.get('slot'):                                  # ran-ahead results: mark when this step is done with them
            ev = torch.cuda.Event()
            ev.record()
            self._slot_events[prep['slot']] = ev
        return out

    def _collect(self, st: dict, train: bool = True) -> Dict[str, torch.Tensor]:
        """Intermediates for the parity tests.  In dedup mode the full [R, Fp] feature matrix the reference builds is
        reassembled from the base rows (clicked / positive rows, unique-negative item halves + the position's context)."""
        L, K, T = st['L'], self.K, st['T']
        n_cand = K + 1
        b = lambda n: self.buffer(st, n)      # noqa: E731
        X = b('X')
        H1 = b('H1')
        if self.dedup:
            # the candidate rows of H1 are stored transposed (H1cT [C, ldr]) behind the clicked rows
            H1 = torch.cat([H1[:L], b('H1cT')[:, :L * n_cand].t()], dim=0)
            c0 = self.plan.ctx_col0
            pos = st['t']['pos_idx'][:L].long()
            uidx = b('neg_uidx')[pos].long()                                  # [L, K]
            xin, xpos, xu = X[:L], X[L:2 * L], X[2 * L:]
            xneg = torch.cat([xu[uidx][..., :c0], xin[:, None, c0:].expand(L, K, X.shape[1] - c0)], dim=2)
            X = torch.cat([xin, torch.cat([xpos[:, None, :], xneg], dim=1).reshape(L * n_cand, -1)], dim=0)
        # with dropout the RNN OUTPUT the reference exposes is the dropped one (DropoutWrapper); the state is HO<i>
        ho = 'HOd%d' if (self.keep_prob < 1.0 and train) else 'HO%d'
        extra = {n: b(n) for n in ('Z1', 'Z2', 'Z3')} if self.ranking == 'mlp' else {}
        return dict(X=X.clone(), H1=H1, E=b('E'), **extra, HO=[b(ho % i) for i in range(self.layers)], F1=b('F1'), PR=b('PR'),
                    logits=b('logits'), row_pos=b('row_pos').view(-1), row_item=b('row_item').view(-1),
                    stats=b('stats').view(-1).clone(),
                    neg=b('neg').view(-1)[st['s0'] * T * K:(st['s0'] + st['B']) * T * K].view(st['B'], T, K))

    def apply_gradients(self, st: Optional[dict] = None):
        """NCCL sum-allreduce of the flat gradient buffer + loss accumulators (data parallel: ONE collective per step), then
        TF-Adam (one C call)."""
        if self.world > 1:
            torch.distributed.all_reduce(self._grads_ext, group=self.pg)
            self._loss_reduced = True
        io = st['prep']['io'] if st is not None and st.get('prep') else StepIO()
        io.global_step = self.global_step
        self._sync_cfg()
        check(self._lib.nar_engine_apply(self._handle, C.byref(io), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
              'nar_engine_apply')
        self.global_step += 1

    @property
    def launches(self) -> int:
        """Kernels launched by the C engine so far."""
        return int(self._lib.nar_engine_launch_count(self._handle))

    # ---- pipelined interface: submit step n, overlap staging + prepare of step n+1 (side stream), then result(n)
    def side_stream(self) -> torch.cuda.Stream:
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        return self._side

    def stage_ahead(self, features, labels, buffer, pop_norm, slot: str, after: Optional[torch.cuda.Event] = None,
                    prev: Optional[dict] = None) -> dict:
        """Stage the NEXT step while the current one runs: the host packs the batch into the slot's pinned buffer; the
        H2D copy and the weight-independent front (sampler, row lists, statistics) run on the side stream next to the
        current step's GEMMs.  ``buffer`` / ``pop_norm`` None: the device-resident state is read, and on the side stream
        it first absorbs the PREVIOUS batch (``prev`` = its staged dict; what the hook's after_run does on the host in
        the reference)."""
        side = self.side_stream()
        if getattr(self, '_dstate_ready', None) is not None:
            side.wait_event(self._dstate_ready)
            self._dstate_ready = None
        if after is not None:
            side.wait_event(after)            # the step that last read this slot's buffers (two slots alternate) is done
        if prev is not None:
            side.wait_event(prev['copied'])
            self.advance_device_state(prev, stream=side)
        st = self.stage(features, labels, buffer, pop_norm, slot=slot, stream=side)
        return self.prepare(st, self.global_step + 1, stream=side)

    def submit(self, st: dict, keep: bool = False) -> dict:
        """Queue one training step; nothing here waits for the GPU.  ``result(out)`` later waits for THIS step only
        (event), so the caller may queue step n+1 before reading the loss of step n - no bubble between steps."""
        out = self.step(st, train=True, keep=keep)
        if st['L'] > 0 or self.world > 1:
            self.apply_gradients(st)                  # (the loss accumulators ride along with the gradients)
        self._loss_slot ^= 1
        host = self._loss_hosts[self._loss_slot]
        host.copy_(self.loss_dev, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        out['stage'], out['loss_host'], out['done'] = st, host, done
        return out

    def result(self, out: dict) -> dict:
        out['done'].synchronize()
        return _read_loss(out, out['loss_host'])

    # ---- evaluation (ModeKeys.EVAL): forward + ranking of the 1+K candidates + HR@n / MRR@n accumulators
    def share_params(self, other: 'NarEngine'):
        """Use ``other``'s weights (same ParamLayout) without a copy: what Estimator.evaluate does when it restores the
        training graph's variables into the evaluation graph (nar_trainer_gcom.py:523)."""
        if other.layout.total != self.layout.total:
            raise ValueError('parameter layouts differ')
        self.params, self.params_lo = other.params, other.params_lo
        self.global_step = other.global_step
        self._views = {}
        self._sync_cfg()
        self._refresh()

    def eval_step(self, features, labels, buffer, pop_norm, top_n: int, metrics: Optional[torch.Tensor] = None,
                  step_id: Optional[int] = None, keep: bool = False, before_sync=None) -> dict:
        """One evaluation batch: negatives with this engine's (eval) sampling hparams, forward, loss, then
        rank_items_by_predicted_prob (nar_model.py:777-795) and the streaming HR@n / MRR@n sums (:835-885).
        ``metrics`` [3] float64 device accumulator {hits, sum of reciprocal ranks, valid labels} (counts stay exact).
        ``before_sync``: called once the batch is queued, before the host waits for its loss (host work to overlap)."""
        st = self.stage(features, labels, buffer, pop_norm, slot='eval')
        if step_id is not None:
            self.prepare(st, step_id)
            st['prep']['step_id'] = self.global_step + 1          # step() checks the id it would use itself
        out = self.step(st, train=False, keep=keep)
        L, n_cand = st['L'], self.K + 1
        if metrics is None:
            metrics = torch.zeros(3, device=self.dev, dtype=torch.float64)
        assert metrics.dtype == torch.float64
        out['metrics'] = metrics
        if L > 0:
            pred_ids = self._buf('pred_ids', L, n_cand, torch.int64, cap_rows=st['B'] * st['T'])
            pred_probs = self._buf('pred_probs', L, n_cand, cap_rows=st['B'] * st['T'])
            ops.rank_candidates(out['logits'], self.buffer(st, 'row_item').view(-1)[L:], L, n_cand, int(top_n), pred_ids,
                                pred_probs, metrics)
            out['predicted_item_ids'], out['predicted_item_probs'] = pred_ids, pred_probs
        if self.world > 1:
            torch.distributed.all_reduce(self.loss_dev, group=self.pg)
        self.loss_host.copy_(self.loss_dev, non_blocking=True)
        if before_sync is not None:
            before_sync()
        torch.cuda.current_stream().synchronize()
        out['stage'] = st
        return _read_loss(out, self.loss_host)

    # ---- recommendation (ModeKeys.PREDICT): score a candidate set for query positions, keep the top n
    MAX_TOP_N = 4096

    def resolve_candidates(self, candidates, buffer) -> np.ndarray:
        """``None``: the sorted distinct nonzero ids of the recent-clicks buffer (the pool training negatives come from);
        ``'catalog'``: every id 1 .. V-1; otherwise an int array of distinct ids in [1, V).  Raises ValueError."""
        if candidates is None:
            b = np.asarray(buffer, dtype=np.int64).reshape(-1)
            return np.unique(b[b != 0])
        if isinstance(candidates, str):
            if candidates != 'catalog':
                raise ValueError("candidates must be None, 'catalog' or an array of article ids, not %r" % candidates)
            return np.arange(1, self.V, dtype=np.int64)
        c = np.asarray(candidates)
        if c.ndim != 1 or c.size == 0 or not np.issubdtype(c.dtype, np.integer):
            raise ValueError('candidates must be a non-empty 1-D integer array of article ids')
        c = c.astype(np.int64)
        if c.min() < 1 or c.max() >= self.V:
            raise ValueError('candidate ids must be in [1, %d)' % self.V)
        if np.unique(c).size != c.size:
            raise ValueError('candidate ids must be distinct')
        return c

    def recommend(self, features, buffer, pop_norm, top_n: int, candidates=None, positions: str = 'last',
                  exclude_session_clicks: bool = True, ws_budget: Optional[int] = None) -> dict:
        """Top-``top_n`` next articles out of ``candidates`` (see resolve_candidates) for the valid positions t <
        session_size - 1 of the batch ``features`` (``positions='last'``: one query per session at its last valid
        position; ``'all'``: every valid position, session-major).  A candidate is scored like a sampled negative of the
        query position (nar_model.py:356-364, :374-405, :444-515); ``exclude_session_clicks`` never returns the query's own
        clicks item_clicked[b, 0..t].  Reads the weights and the given state only (one C call, csrc/engine.cu).
        ``ws_budget``: workspace bytes (default: the engine's budget); smaller budgets run more, smaller blocks with
        bit-identical results.  -> numpy dict: query_session [Q], query_position [Q], predicted_item_ids /
        predicted_item_scores / predicted_item_probs [Q, top_n], candidates [N]."""
        if self.world > 1:
            raise NotImplementedError('recommend runs on one process; data-parallel prediction is not implemented')
        if positions not in ('last', 'all'):
            raise ValueError("positions must be 'last' or 'all', not %r" % (positions,))
        if buffer is None or pop_norm is None:
            raise ValueError('recommend needs the host recent-clicks buffer and popularity')
        cand = self.resolve_candidates(candidates, buffer)
        N = int(cand.size)
        if isinstance(top_n, (bool, np.bool_)) or not isinstance(top_n, (int, np.integer)):
            raise ValueError('top_n must be an integer')
        top_n = int(top_n)
        if not 1 <= top_n <= min(N, self.MAX_TOP_N):
            raise ValueError('top_n=%d outside [1, min(N=%d, %d)]' % (top_n, N, self.MAX_TOP_N))
        item_clicked = np.asarray(features['item_clicked'])
        Bg, T = item_clicked.shape
        labels = {'label_next_item': np.zeros((Bg, T), dtype=np.int64), 'label_last_item': np.zeros(Bg, dtype=np.int64)}
        st = self.stage(features, labels, buffer, pop_norm, slot='predict')
        L, lens = st['L'], st['lens']
        ends = np.cumsum(lens)
        if positions == 'last':
            q_rows = (ends - 1)[lens > 0].astype(np.int64)
            q_sess = np.flatnonzero(lens > 0).astype(np.int64)
            q_t = (lens[lens > 0] - 1).astype(np.int64)
        else:
            q_rows = np.arange(L, dtype=np.int64)
            q_sess = np.repeat(np.arange(Bg, dtype=np.int64), lens)
            q_t = np.arange(L, dtype=np.int64) - np.repeat(ends - lens, lens)
        Q = int(q_rows.size)
        out = {'query_session': q_sess, 'query_position': q_t, 'candidates': cand,
               'predicted_item_ids': np.zeros((Q, top_n), np.int64), 'predicted_item_scores': np.zeros((Q, top_n), np.float32),
               'predicted_item_probs': np.zeros((Q, top_n), np.float32)}
        if Q == 0:
            return out
        gather_q = positions == 'last'
        budget = int(self._ws_budget if ws_budget is None else ws_budget)
        wb, qb, nb = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        check(self._lib.nar_engine_recommend_workspace_bytes(self._handle, L, Q, N, int(gather_q), budget, C.byref(wb),
                                                             C.byref(qb), C.byref(nb)), 'nar_engine_recommend_workspace_bytes')
        self._sync_cfg()
        d = self.dev
        ws = self._buf('rec_ws', int(wb.value), 1, torch.uint8).view(-1)
        q_pos = torch.from_numpy(q_sess * T + q_t).to(torch.int32).to(d)
        q_rows_t = torch.from_numpy(q_rows).to(d) if gather_q else None
        cand_t = torch.from_numpy(cand).to(d)
        ids = torch.empty(Q, top_n, dtype=torch.int64, device=d)
        scores = torch.empty(Q, top_n, dtype=torch.float32, device=d)
        probs = torch.empty(Q, top_n, dtype=torch.float32, device=d)
        io = self._staged_io(st)
        io.L_cap, io.global_step, io.train = L, self.global_step, 0
        io.ws, io.ws_bytes = ws.data_ptr(), ws.numel()
        cur = torch.cuda.current_stream()
        check(self._lib.nar_engine_recommend(self._handle, C.byref(io), C.c_void_p(0 if q_rows_t is None else q_rows_t.data_ptr()),
                                             C.c_void_p(q_pos.data_ptr()), Q, C.c_void_p(cand_t.data_ptr()), N, top_n,
                                             int(bool(exclude_session_clicks)), int(qb.value), int(nb.value),
                                             C.c_void_p(ids.data_ptr()), C.c_void_p(scores.data_ptr()),
                                             C.c_void_p(probs.data_ptr()), C.c_void_p(cur.cuda_stream)), 'nar_engine_recommend')
        out['predicted_item_ids'] = ids.cpu().numpy()
        out['predicted_item_scores'] = scores.cpu().numpy()
        out['predicted_item_probs'] = probs.cpu().numpy()
        out['q_block'], out['n_block'] = int(qb.value), int(nb.value)
        return out

    # ---- unsampled evaluation (DESIGN.md section 13): rank each label against every candidate the sampler could draw
    MAX_RANK_SESSION = 1023           # positions T of a batch: the session row of T + 1 ids is the kernel's exclusion list

    @staticmethod
    def unsampled_pool(item_clicked, label_last_item, buffer) -> np.ndarray:
        """The sorted distinct nonzero ids of the batch's clicks, its last labels and the recent-clicks buffer: every id
        the negative sampler of an EVAL step may draw from (nar_model.py:1220-1304, before the per-session exclusion)."""
        ids = np.concatenate([np.asarray(a, dtype=np.int64).reshape(-1) for a in (item_clicked, label_last_item, buffer)])
        return np.unique(ids[ids != 0])

    def rank_labels(self, st: dict, candidates, top_n: int, hist: Optional[torch.Tensor] = None,
                    ws_budget: Optional[int] = None) -> dict:
        """Rank the label of every valid position of the EVAL batch staged in ``st`` (eval_step's ``out['stage']``) against
        ``candidates`` (distinct ids in [1, V), any order; see unsampled_pool), each scored as recommend scores it.  The
        competitors of a query are the candidates other than its label outside its session's row [item_clicked[b] |
        label_last_item[b]]; rank = how many of them score above the label (ties go to the label).  ``hist`` [top_n + 2]
        int64 device accumulator (default: a new zero one): the count of each rank below top_n, the ranked queries and
        their competitors.  Reads the staged batch, the weights and the state it was staged with; writes nothing else.
        -> dict(rank [L] int32 device tensor, -1 for a label outside the candidates; hist; candidates (ascending);
        q_block, n_block)."""
        if self.world > 1:
            raise NotImplementedError('the unsampled evaluation runs on one process; data-parallel evaluation is not '
                                      'implemented')
        if isinstance(top_n, (bool, np.bool_)) or not isinstance(top_n, (int, np.integer)) or top_n < 1:
            raise ValueError('top_n must be a positive integer, not %r' % (top_n,))
        top_n = int(top_n)
        if st['T'] > self.MAX_RANK_SESSION:
            raise ValueError('the unsampled evaluation ranks sessions of at most %d positions, not %d'
                             % (self.MAX_RANK_SESSION, st['T']))
        L, d = st['L'], self.dev
        cand = np.sort(self.resolve_candidates(np.asarray(candidates), None)) if L > 0 else np.sort(np.asarray(candidates))
        N = int(cand.size)
        if hist is None:
            hist = torch.zeros(top_n + 2, dtype=torch.int64, device=d)
        if hist.dtype != torch.int64 or hist.numel() != top_n + 2 or hist.device != d:
            raise ValueError('hist must be an int64 tensor of top_n + 2 = %d entries on %s' % (top_n + 2, d))
        rank = torch.empty(max(L, 1), dtype=torch.int32, device=d)[:L]
        out = {'rank': rank, 'hist': hist, 'candidates': cand, 'q_block': 0, 'n_block': 0}
        if L == 0:
            return out
        budget = int(self._ws_budget if ws_budget is None else ws_budget)
        wb, qb, nb = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        check(self._lib.nar_engine_recommend_workspace_bytes(self._handle, L, L, N, 0, budget, C.byref(wb), C.byref(qb),
                                                             C.byref(nb)), 'nar_engine_recommend_workspace_bytes')
        self._sync_cfg()
        ws = self._buf('rec_ws', int(wb.value), 1, torch.uint8).view(-1)
        cand_t = torch.from_numpy(cand).to(d)
        io = self._staged_io(st)
        io.L_cap, io.global_step, io.train = L, self.global_step, 0
        io.ws, io.ws_bytes = ws.data_ptr(), ws.numel()
        check(self._lib.nar_engine_rank_labels(self._handle, C.byref(io), C.c_void_p(cand_t.data_ptr()), N, top_n,
                                               int(qb.value), int(nb.value), C.c_void_p(rank.data_ptr()),
                                               C.c_void_p(hist.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
              'nar_engine_rank_labels')
        out['q_block'], out['n_block'] = int(qb.value), int(nb.value)
        return out

    def train_step(self, features, labels, buffer, pop_norm, keep: bool = False, sync: bool = True) -> dict:
        """Stage, run and apply one training step; ``sync``: wait for it and read its loss (else ``result(out)`` does)."""
        out = self.submit(self.stage(features, labels, buffer, pop_norm), keep=keep)
        return self.result(out) if sync else out


def _read_loss(out: dict, host: torch.Tensor) -> dict:
    """The four loss keys of ``out`` from a host copy of the loss accumulators [xe, l2, novelty, -]."""
    out['xe_loss'], out['reg_loss'], out['nov_reg_loss'] = host[:3].tolist()
    out['total_loss'] = out['xe_loss'] + out['reg_loss'] - out['nov_reg_loss']
    return out
