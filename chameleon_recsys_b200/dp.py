"""Data-parallel host logic (numpy only; no CUDA needed, so it is testable with gloo on CPU).

The reference has no distribution at all (README.md:252: single worker on purpose).  The H100 build
shards the *sessions* of one global batch contiguously across ranks (chronological order per rank is
kept; boundaries balanced by valid positions, see shard_bounds) and keeps global-batch semantics
identical to one GPU (SURVEY.md section 8e):
  * every rank sees the ids of the whole global batch, so the candidate pool and the per-click draws
    (counter = global session index) are identical for any world size;
  * the loss normaliser sum(mask) is the GLOBAL count (known from session_size, no collective);
  * gradients are sum-allreduced (NCCL) - the only collective on the path;
  * the host ClickedItemsState update is a deterministic function of the global ids: every rank
    computes it redundantly.
"""
from __future__ import annotations

from typing import Dict

import numpy as np


def shard_bounds(lens_g: np.ndarray, world: int, balance: bool = True) -> np.ndarray:
    """Session boundaries [world+1] of the contiguous shards.  ``balance``: equal numbers of VALID POSITIONS per rank
    (the unit of work of a step: every GEMM row count is proportional to it) instead of equal numbers of sessions -
    with G1-shaped session lengths the fullest of 8 equal-count shards holds 7 % more positions than the mean, and a
    synchronous step is as slow as its fullest rank; balanced boundaries bring that to < 1 %.  Every rank computes the
    same boundaries from the global ``session_size`` (no collective); every rank keeps at least one session."""
    Bg = int(lens_g.shape[0])
    if Bg < world:
        raise ValueError('global batch %d smaller than world size %d' % (Bg, world))
    total = int(lens_g.sum())
    if not balance and Bg % world:
        raise ValueError('global batch %d not divisible by world size %d' % (Bg, world))
    if not balance or world == 1 or total == 0:
        return np.arange(world + 1, dtype=np.int64) * Bg // world
    cs = np.cumsum(lens_g, dtype=np.int64)                 # cs[i] = positions of sessions [0, i]
    bounds = np.zeros(world + 1, dtype=np.int64)
    bounds[world] = Bg
    for k in range(1, world):
        target = total * k / world
        i = int(np.searchsorted(cs, target, side='left'))   # first i with cs[i] >= target: boundary i or i + 1
        below = cs[i - 1] if i > 0 else 0
        b = i + 1 if (i < Bg and cs[i] - target <= target - below) else i
        bounds[k] = min(max(b, bounds[k - 1] + 1), Bg - (world - k))
    return bounds


def shard_sessions(session_size: np.ndarray, T: int, world: int, rank: int, balance: bool = True) -> Dict[str, np.ndarray]:
    """-> dict(s0, per, lens[per], L, L_global, sess_off[per+1] int32, pos_idx[L] int32 (flat b*T+t, global b)).
    Rank ``rank`` owns the sessions [s0, s0 + per) of the global batch (``shard_bounds``)."""
    lens_g = np.clip(np.asarray(session_size, dtype=np.int64) - 1, 0, T)      # seq_lengths, nar_model.py:227
    bounds = shard_bounds(lens_g, world, balance)
    s0, per = int(bounds[rank]), int(bounds[rank + 1] - bounds[rank])
    lens = lens_g[s0:s0 + per]
    sess_off = np.zeros(per + 1, dtype=np.int32)
    np.cumsum(lens, out=sess_off[1:])
    tt = np.arange(T, dtype=np.int64)[None, :]
    valid = tt < lens[:, None]                                                # tf.sequence_mask, nar_model.py:231
    bb = (np.arange(per, dtype=np.int64) + s0)[:, None]
    pos_idx = (bb * T + tt)[valid].astype(np.int32)
    return {'s0': s0, 'per': per, 'lens': lens, 'L': int(lens.sum()), 'L_global': int(lens_g.sum()),
            'sess_off': sess_off, 'pos_idx': pos_idx}
