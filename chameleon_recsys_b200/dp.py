"""Data-parallel host logic (numpy, plus torch.distributed for the prediction gather; no CUDA needed, so it is testable
with gloo on CPU).

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
Prediction (NarEngine.recommend) shards the same way with the queries as the unit of work (query_weights) and rebuilds
the one-process result on every rank with one all_gather (gather_query_rows).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np


def shard_bounds(lens_g: np.ndarray, world: int, balance: bool = True, weights: Optional[np.ndarray] = None) -> np.ndarray:
    """Session boundaries [world+1] of the contiguous shards.  ``balance``: equal numbers of VALID POSITIONS per rank
    (the unit of work of a step: every GEMM row count is proportional to it) instead of equal numbers of sessions -
    with G1-shaped session lengths the fullest of 8 equal-count shards holds 7 % more positions than the mean, and a
    synchronous step is as slow as its fullest rank; balanced boundaries bring that to < 1 %.  ``weights`` [Bg]: the
    work of each session when it is not its valid positions (a recommendation for the last position only: 1 for a
    session with a valid position, 0 without; see query_weights); None = ``lens_g``.  Every rank computes the same
    boundaries from the global ``session_size`` (no collective); every rank keeps at least one session."""
    Bg = int(lens_g.shape[0])
    if Bg < world:
        raise ValueError('global batch %d smaller than world size %d' % (Bg, world))
    w = lens_g if weights is None else np.asarray(weights, dtype=np.int64)
    if w.shape != (Bg,) or (w < 0).any():
        raise ValueError('weights must be %d non-negative integers' % Bg)
    total = int(w.sum())
    if not balance and Bg % world:
        raise ValueError('global batch %d not divisible by world size %d' % (Bg, world))
    if not balance or world == 1 or total == 0:
        return np.arange(world + 1, dtype=np.int64) * Bg // world
    cs = np.cumsum(w, dtype=np.int64)                      # cs[i] = weight of sessions [0, i]
    bounds = np.zeros(world + 1, dtype=np.int64)
    bounds[world] = Bg
    for k in range(1, world):
        target = total * k / world
        i = int(np.searchsorted(cs, target, side='left'))   # first i with cs[i] >= target: boundary i or i + 1
        below = cs[i - 1] if i > 0 else 0
        b = i + 1 if (i < Bg and cs[i] - target <= target - below) else i
        bounds[k] = min(max(b, bounds[k - 1] + 1), Bg - (world - k))
    return bounds


def session_lengths(session_size: np.ndarray, T: int) -> np.ndarray:
    """Valid positions of each session (seq_lengths, nar_model.py:227)."""
    return np.clip(np.asarray(session_size, dtype=np.int64) - 1, 0, T)


def shard_sessions(session_size: np.ndarray, T: int, world: int, rank: int, balance: bool = True,
                   weights: Optional[np.ndarray] = None) -> Dict[str, np.ndarray]:
    """-> dict(s0, per, lens[per], L, L_global, sess_off[per+1] int32, pos_idx[L] int32 (flat b*T+t, global b)).
    Rank ``rank`` owns the sessions [s0, s0 + per) of the global batch (``shard_bounds`` with ``weights``)."""
    lens_g = session_lengths(session_size, T)
    bounds = shard_bounds(lens_g, world, balance, weights)
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


# ---------------------------------------------------------------------------------------------- data-parallel prediction
def query_weights(lens_g: np.ndarray, positions: str) -> Optional[np.ndarray]:
    """Queries of each session in a recommend call: ``'last'``: 1 for a session with a valid position, 0 without;
    ``'all'``: its valid positions, which are the default weights of shard_bounds (None)."""
    return (np.asarray(lens_g) > 0).astype(np.int64) if positions == 'last' else None


def query_counts(lens_g: np.ndarray, bounds: np.ndarray, positions: str) -> np.ndarray:
    """[world] queries of each rank's shard ``bounds``: every rank knows them from the global batch, no collective."""
    w = query_weights(lens_g, positions)
    w = np.asarray(lens_g, dtype=np.int64) if w is None else w
    cs = np.concatenate([[0], np.cumsum(w, dtype=np.int64)])
    return cs[bounds[1:]] - cs[bounds[:-1]]


def gather_query_rows(parts: Sequence, counts: Sequence[int], group=None) -> List:
    """Every rank's query rows, concatenated in rank order, on every rank, with ONE all_gather.  ``parts``: this rank's
    tensors [counts[rank], ...] (4- or 8-byte dtypes, one device); ``counts``: every rank's row count (query_counts).
    The parts are packed bit for bit into one int32 buffer of max(counts) rows (zero rows on a rank without queries),
    gathered and unpacked -> one tensor [sum(counts), ...] per part.  Every rank of ``group`` calls it with the same
    ``counts`` and the same part shapes beyond the first dimension and dtypes."""
    import torch
    import torch.distributed as dist
    world, rank = len(counts), dist.get_rank(group)
    if world != dist.get_world_size(group):
        raise ValueError('counts has %d entries for a group of %d ranks' % (world, dist.get_world_size(group)))
    Q, Qmax = int(counts[rank]), int(max(counts))
    if any(int(p.shape[0]) != Q for p in parts):
        raise ValueError('every part must have counts[rank] = %d rows' % Q)
    cols = [int(np.prod(p.shape[1:], dtype=np.int64)) * p.element_size() // 4 for p in parts]
    packed = torch.zeros(max(Qmax, 1), sum(cols), dtype=torch.int32, device=parts[0].device)
    if Q:
        packed[:Q] = torch.cat([p.reshape(Q, -1).contiguous().view(torch.int32) for p in parts], dim=1)
    got = [torch.empty_like(packed) for _ in range(world)]
    dist.all_gather(got, packed, group=group)
    rows = torch.cat([g[:int(n)] for g, n in zip(got, counts)], dim=0)
    out, c0 = [], 0
    for p, c in zip(parts, cols):
        part = rows[:, c0:c0 + c].contiguous()
        out.append((part.view(p.dtype) if rows.shape[0] else part.new_empty(0, dtype=p.dtype)).reshape(rows.shape[0], *p.shape[1:]))
        c0 += c
    return out
