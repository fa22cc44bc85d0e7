"""Data-parallel prediction, host side (CPU, gloo): shard boundaries balanced by queries, and the one all_gather that
rebuilds the one-process recommendation arrays on every rank (dp.gather_query_rows)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chameleon_recsys_b200.dp import (query_counts, query_weights, session_lengths, shard_bounds,  # noqa: E402
                                      shard_sessions)


def _batches():
    """Session lengths: G1-like, with runs of sessions without a valid position, a single valid session, none."""
    rs = np.random.RandomState(7)
    out = []
    for Bg in (3, 5, 16, 64, 256):
        size = rs.geometric(0.3, size=Bg).clip(1, 21)            # session_size: 1 .. 21 clicks
        out.append(size)
        holes = size.copy()
        holes[rs.rand(Bg) < 0.6] = 1                            # most sessions have no valid position
        out.append(holes)
        one = np.ones(Bg, np.int64)
        one[rs.randint(Bg)] = 4
        out.append(one)
        out.append(np.ones(Bg, np.int64))
        front = np.ones(Bg, np.int64)
        front[:2] = 9                                           # every query in the first sessions
        out.append(front)
    return out


@pytest.mark.parametrize('positions', ['last', 'all'])
def test_query_shards_cover_the_batch(positions):
    T = 20
    for size in _batches():
        lens = session_lengths(size, T)
        w = query_weights(lens, positions)
        wq = lens if w is None else w
        for world in range(1, min(8, lens.size) + 1):
            b = shard_bounds(lens, world, weights=w)
            # contiguous, covering, every rank keeps at least one session
            assert b[0] == 0 and b[-1] == lens.size and (np.diff(b) >= 1).all(), (size, world, b)
            counts = query_counts(lens, b, positions)
            assert counts.sum() == wq.sum()
            assert all(int(wq[b[r]:b[r + 1]].sum()) == counts[r] for r in range(world))
            # the fullest shard exceeds the mean by at most the weight of one session (one query for 'last')
            if wq.sum() and lens.size >= 2 * world:
                assert counts.max() <= wq.sum() / world + wq.max(), (size, world, counts)
            # the engine's shards are these bounds
            for r in range(world):
                sh = shard_sessions(size, T, world, r, weights=w)
                assert (sh['s0'], sh['per']) == (b[r], b[r + 1] - b[r])


def test_default_weights_give_the_training_shards():
    """weights=None and weights=valid positions are today's bounds, bit for bit, for every batch and world size."""
    T = 20

    def old_bounds(lens_g, world):                            # the boundaries training has always used
        Bg, total = int(lens_g.shape[0]), int(lens_g.sum())
        if world == 1 or total == 0:
            return np.arange(world + 1, dtype=np.int64) * Bg // world
        cs = np.cumsum(lens_g, dtype=np.int64)
        bounds = np.zeros(world + 1, dtype=np.int64)
        bounds[world] = Bg
        for k in range(1, world):
            target = total * k / world
            i = int(np.searchsorted(cs, target, side='left'))
            below = cs[i - 1] if i > 0 else 0
            bb = i + 1 if (i < Bg and cs[i] - target <= target - below) else i
            bounds[k] = min(max(bb, bounds[k - 1] + 1), Bg - (world - k))
        return bounds

    for size in _batches():
        lens = session_lengths(size, T)
        for world in range(1, min(8, lens.size) + 1):
            want = old_bounds(lens, world)
            assert np.array_equal(shard_bounds(lens, world), want)
            assert np.array_equal(shard_bounds(lens, world, weights=lens), want)
            assert query_weights(lens, 'all') is None
            if lens.size % world == 0:
                assert np.array_equal(shard_bounds(lens, world, balance=False, weights=query_weights(lens, 'last')),
                                      np.arange(world + 1) * lens.size // world)


def test_weights_are_checked():
    lens = np.array([1, 2, 0, 3])
    with pytest.raises(ValueError):
        shard_bounds(lens, 2, weights=np.ones(3))
    with pytest.raises(ValueError):
        shard_bounds(lens, 2, weights=np.array([1, -1, 0, 0]))
    with pytest.raises(ValueError):
        shard_bounds(lens, 5)


def _gather_worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from chameleon_recsys_b200.dp import gather_query_rows
        torch.set_num_threads(1)
        rs = np.random.RandomState(3)
        top_n = 5
        for counts in ([4, 0, 3][:world], [0] * (world - 1) + [6], [1] * world, [7, 2, 5][:world]):
            Qg = sum(counts)
            # the one-process arrays, with NaN, -0.0, denormals and int64 ids above 2^32 to catch any lossy copy
            ids = rs.randint(1, 1 << 40, size=(Qg, top_n)).astype(np.int64)
            sc = rs.randn(Qg, top_n).astype(np.float32)
            pr = rs.rand(Qg, top_n).astype(np.float32)
            if Qg:
                sc[0, 0], sc[-1, -1], pr[0, -1] = np.nan, -0.0, np.float32(1e-45)
            q0 = sum(counts[:rank])
            parts = [torch.from_numpy(a[q0:q0 + counts[rank]].copy()) for a in (ids, sc, pr)]
            got = gather_query_rows(parts, counts)
            for g, want in zip(got, (ids, sc, pr)):
                g = g.numpy()
                assert g.dtype == want.dtype and g.shape == want.shape, (counts, g.shape, want.shape)
                assert g.tobytes() == want.tobytes(), counts
        ret[rank] = 1
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3])
def test_gather_rebuilds_the_one_process_arrays(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + (os.getpid() % 2000) + 7 * world
    mp.spawn(_gather_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {r: 1 for r in range(world)}
