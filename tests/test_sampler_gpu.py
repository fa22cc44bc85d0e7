"""The negative sampler (csrc/sampler.cu) against oracle/sampler_ref.py, bit for bit.

Every case runs nar_sample_negatives_uidx and compares all four of its outputs with the oracle:
- ``out`` [B, T1-1, K] with ``sampler_ref.sample_negatives`` on the slice [sess0, sess0+B), the pool built from every
  session (data parallel);
- ``n_unique`` with the number of distinct ids in ``sampler_ref.build_pool``, and ``unique_items[:n_unique]`` with those
  ids sorted (both read from the workspace through the pointers the call returns);
- ``out_uidx``: K*20 (the padding slot) where a negative is 0, else the index of the negative in the unique table.
The plain entry point (ops.sample_negatives -> nar_sample_negatives) runs on the same inputs and must give the same
``out``.  Outputs start from a sentinel and carry guard space past their end that must keep it.

The cases choose the nonzero clicks and buffer samples so that the pool holds 1, 2, 1023, 1024, 1025, 2048, 2049, 8192,
8193 and 16380 entries: both sort paths of the pool kernel (the 1024-key register network and the shared-memory network
above 1024 keys), and click-kernel sorts of 1 to 16384 keys.  K spans 1 .. 819 (K*20 = 16380, the largest
pool that fits), buffers hold zeros between their samples and heavy duplicates, sessions hold padding before their last
click, repeated items and their own label, seeds use the high half of the Philox key and steps reach 2^32 - 1.  The
oracle's per-click work is kept to a few hundred clicks per case; the pool itself is full size.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import sampler_ref

NAR_ERR_INVALID, NAR_ERR_UNSUPPORTED, NAR_ERR_WORKSPACE = -1, -2, -4
SENT64 = 0x5A5A5A5A5A5A5A5A
SENT32 = 0x5A5A5A5A
GUARD = 64
FACTOR = sampler_ref.FIRST_SAMPLING_MULTIPLYING_FACTOR


# ------------------------------------------------------------------------------------------------ inputs and reference
def _ids(rs, shape, n_nz, V):
    """ids in [1, V) of the given shape with exactly n_nz nonzero entries; the zeros fall anywhere (between buffer
    samples, before a session's last click)"""
    a = rs.randint(1, V, size=shape).astype(np.int64)
    flat = a.reshape(-1)
    flat[rs.permutation(flat.size)[:flat.size - n_nz]] = 0
    return a


def _expected_tables(allc, buf, K, nfb, seed, step):
    """the pool of the oracle, its sorted unique ids (the table the kernels index) and a function that maps negatives to
    their out_uidx"""
    pool = sampler_ref.build_pool(allc, buf, K, nfb, seed, step)
    uniq = np.unique(pool)

    def uidx(neg):
        return np.where(neg == 0, K * FACTOR, np.searchsorted(uniq, neg)).astype(np.int32)
    return pool, uniq, uidx


def test_uidx_derivation_matches_build_pool():
    """CPU: the unique table and out_uidx the GPU tests expect, derived from sampler_ref.build_pool, against a plain
    restatement: the table is the sorted set of pool ids, every nonzero oracle negative is in it at its uidx, and the
    padding negative maps to the slot past the table's capacity."""
    rs = np.random.RandomState(3)
    for K, V, nfb in ((5, 40, 7), (50, 3000, 100), (1, 6, 0)):
        allc = _ids(rs, (9, 6), 40, V)
        buf = _ids(rs, (300,), 120, V)
        seed, step = 0xDEADBEEF12345678, 7
        pool, uniq, uidx = _expected_tables(allc, buf, K, nfb, seed, step)
        assert uniq.tolist() == sorted(set(pool.tolist()))
        assert pool.size == min(int((allc != 0).sum()) + min(int((buf != 0).sum()), nfb), K * FACTOR)
        neg = sampler_ref.sample_negatives(allc[2:6], buf, K, nfb, seed, step, session_offset=2,
                                           all_clicked_items_global=allc)
        u = uidx(neg)
        nz = neg != 0
        assert (u[~nz] == K * FACTOR).all()
        assert (u[nz] < uniq.size).all() and np.array_equal(uniq[u[nz]], neg[nz])
        for b in range(4):                                   # ListDiff: no negative is an item of its own session
            assert not np.isin(neg[b][neg[b] != 0], allc[2 + b]).any()


# ------------------------------------------------------------------------------------------------ GPU calls
def _lib_ctx():
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import load
    return load(), ops.context(), ops


def _ws(ops, torch, Bg, T1, buf_len, K):
    return torch.zeros(ops.sample_negatives_workspace(Bg, T1, buf_len, K) + GUARD, dtype=torch.uint8, device='cuda')


def _call_uidx(torch, allc_d, Bg, T1, sess0, B, buf_d, buf_len, K, nfb, seed, step, out, ou, ws, ws_bytes):
    lib, ctx, ops = _lib_ctx()
    ui, nu = C.c_void_p(), C.c_void_p()
    rc = lib.nar_sample_negatives_uidx(ctx.handle, ops._p(allc_d), Bg, T1, sess0, B, ops._p(buf_d), buf_len, K, nfb,
                                       C.c_uint64(seed), C.c_uint32(step), ops._p(out), ops._p(ou), C.byref(ui),
                                       C.byref(nu), ops._p(ws), ws_bytes, ops._stream())
    return rc, ui.value, nu.value


def _run_case(allc, buf, K, nfb, seed, step, sess0, B, n_pool=None):
    torch = pytest.importorskip('torch')
    _, _, ops = _lib_ctx()
    Bg, T1 = allc.shape
    pool, uniq, uidx = _expected_tables(allc, buf, K, nfb, seed, step)
    if n_pool is not None:
        assert pool.size == n_pool, (pool.size, n_pool)          # the case reaches the pool size it is meant to
    ref = sampler_ref.sample_negatives(allc[sess0:sess0 + B], buf, K, nfb, seed, step, session_offset=sess0,
                                       all_clicked_items_global=allc)
    n_out = B * (T1 - 1) * K
    allc_d = torch.from_numpy(np.ascontiguousarray(allc)).cuda()
    buf_d = torch.from_numpy(np.ascontiguousarray(buf)).cuda()
    out = torch.full((n_out + GUARD,), SENT64, dtype=torch.int64, device='cuda')
    ou = torch.full((n_out + GUARD,), SENT32, dtype=torch.int32, device='cuda')
    ws = _ws(ops, torch, Bg, T1, buf.size, K)
    ws_bytes = ws.numel() - GUARD
    rc, ui, nu = _call_uidx(torch, allc_d, Bg, T1, sess0, B, buf_d, buf.size, K, nfb, seed, step, out, ou, ws, ws_bytes)
    assert rc == 0
    out2 = torch.full((n_out + GUARD,), SENT64, dtype=torch.int64, device='cuda')
    ws2 = _ws(ops, torch, Bg, T1, buf.size, K)
    ops.sample_negatives(allc_d, sess0, B, buf_d, K, nfb, seed, step, out2, ws2[:ws2.numel() - GUARD])
    torch.cuda.synchronize()
    base = ws.data_ptr()
    assert 0 <= ui - base and ui - base + 8 * K * FACTOR <= ws_bytes and (ui - base) % 8 == 0
    assert 0 <= nu - base and nu - base + 4 <= ws_bytes and (nu - base) % 4 == 0
    n_unique = int(ws[nu - base:nu - base + 4].view(torch.int32).item())
    assert n_unique == uniq.size, (n_unique, uniq.size)
    got_u = ws[ui - base:ui - base + 8 * n_unique].view(torch.int64).cpu().numpy()
    assert np.array_equal(got_u, uniq)
    got = out[:n_out].cpu().numpy().reshape(B, T1 - 1, K)
    got_idx = ou[:n_out].cpu().numpy().reshape(B, T1 - 1, K)
    assert np.array_equal(got, ref), np.argwhere(got != ref)[:8]
    assert np.array_equal(got_idx, uidx(ref)), np.argwhere(got_idx != uidx(ref))[:8]
    assert np.array_equal(out2[:n_out].cpu().numpy().reshape(B, T1 - 1, K), ref)
    for t in (out, ou, out2):
        s = SENT64 if t.dtype == torch.int64 else SENT32
        assert bool((t[n_out:] == s).all()), 'write past the end of an output'
    for b in range(B):                                           # ListDiff, stated directly
        assert not np.isin(got[b][got[b] != 0], allc[sess0 + b]).any()
    return got


# ------------------------------------------------------------------------------------------------ pool size / K
# id, K, Bg, T1, nonzero clicks, buffer length, nonzero buffer entries, n_from_buffer, V, sess0, B, pool size
POOL_CASES = [
    ('pool1_batch_only', 1, 4, 3, 1, 64, 5, 0, 50, 0, 4, 1),
    ('pool2_click_and_sample', 1, 4, 3, 1, 64, 3, 1, 50, 0, 4, 2),
    ('pool1023_K52', 52, 50, 21, 1000, 400, 50, 23, 40000, 10, 8, 1023),
    ('pool1024_K52', 52, 50, 21, 1000, 400, 24, 24, 40000, 0, 8, 1024),        # n_from_buffer = count
    ('pool1025_K52', 52, 50, 21, 1000, 400, 26, 25, 40000, 49, 1, 1025),        # count - 1, last session
    ('pool1000_K50_capped', 50, 256, 21, 4000, 2000, 1500, 1000, 40000, 128, 6, 1000),
    ('pool1020_K51_capped', 51, 64, 21, 1300, 100, 60, 60, 40000, 30, 6, 1020),
    ('pool2000_K100_capped', 100, 160, 21, 3000, 500, 300, 250, 40000, 80, 4, 2000),
    ('pool2048_K409', 409, 100, 21, 2000, 3000, 100, 48, 46000, 50, 2, 2048),
    ('pool2049_K410_no_buffer', 410, 100, 21, 2049, 3000, 900, 0, 46000, 99, 1, 2049),
    ('pool8192_K410', 410, 400, 21, 8000, 3000, 192, 192, 46000, 200, 1, 8192),
    ('pool8193_K500_nfb_above', 500, 400, 21, 8100, 3000, 93, 200, 46000, 0, 1, 8193),
    ('pool16380_K819_capped', 819, 600, 31, 17000, 20000, 12000, 5000, 360000, 300, 1, 16380),
    ('pool16380_K819_stress', 819, 512, 41, 16000, 20000, 380, 380, 360000, 511, 1, 16380),
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_sampler_pool_sizes(case):
    _, K, Bg, T1, n_nz, buf_len, n_buf, nfb, V, sess0, B, n_pool = case
    rs = np.random.RandomState(K * 1000 + n_nz)
    allc = _ids(rs, (Bg, T1), n_nz, V)
    buf = _ids(rs, (buf_len,), n_buf, V)
    _run_case(allc, buf, K, nfb, 0x1234 + K, 11 + n_pool, sess0, B, n_pool=n_pool)


# ------------------------------------------------------------------------------------------------ content edges
@pytest.mark.gpu
@pytest.mark.parametrize('K,V', [(5, 4), (50, 30), (500, 300)])
def test_sampler_fewer_distinct_items_than_K(K, V):
    """n_unique < K: the tail of every output row is the zero id and the padding slot; heavy duplicates in the batch
    and the buffer"""
    rs = np.random.RandomState(K)
    allc = _ids(rs, (40, 11), 300, V)
    buf = _ids(rs, (800,), 700, V)
    got = _run_case(allc, buf, K, 400, 99, 5, 7, 12)
    assert (got[..., V - 1:] == 0).all()


@pytest.mark.gpu
def test_sampler_one_item_pool():
    """every click and buffer entry is the same id: the table has one entry and every session excludes it"""
    allc = np.zeros((6, 5), np.int64)
    allc[:, :3] = 7
    allc[2, 1] = 0
    buf = np.array([7, 0, 7, 7, 0, 0, 7] * 10, np.int64)
    got = _run_case(allc, buf, 5, 30, 1, 1, 0, 6, n_pool=6 * 3 - 1 + 30)
    assert (got == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('B', [3, 0])
def test_sampler_empty_pool(B):
    """an all-zero batch and buffer: n_pool = n_unique = 0, every negative 0 / the padding slot"""
    allc = np.zeros((5, 4), np.int64)
    buf = np.zeros(100, np.int64)
    got = _run_case(allc, buf, 5, 50, 3, 3, 1, B, n_pool=0)
    assert (got == 0).all()


@pytest.mark.gpu
def test_sampler_session_holds_every_pool_item():
    """Adressa's T1 = 31: session 3 clicks every id of the vocabulary (so all its negatives are 0), the other sessions
    click a few ids, some of them twice, with padding between clicks; each label is excluded at every position"""
    rs = np.random.RandomState(5)
    Bg, T1 = 12, 31
    allc = np.zeros((Bg, T1), np.int64)
    for b in range(Bg):
        n = rs.randint(2, 6)
        allc[b, rs.choice(T1 - 1, n, replace=False)] = rs.randint(1, 9, size=n)
        allc[b, T1 - 1] = rs.randint(1, 9)                      # the label: in the pool, excluded from the session
    allc[3, :8] = np.arange(1, 9)
    buf = rs.randint(0, 9, size=200).astype(np.int64)
    got = _run_case(allc, buf, 5, 60, 0xDEADBEEF12345678, 77, 1, 6)
    assert (got[2] == 0).all()
    assert (got != 0).any()
    for b in range(6):
        assert not np.isin(allc[1 + b, T1 - 1], got[b]).any()


@pytest.mark.gpu
@pytest.mark.parametrize('T1', [2, 31])
@pytest.mark.parametrize('seed,step', [(0xDEADBEEF12345678, 3), (0x00000001FFFFFFFF, 0xFFFFFFFF), (42, 0)],
                         ids=['seed_hi', 'seed_hi_last_step', 'seed_lo_step0'])
@pytest.mark.parametrize('where', ['first', 'middle', 'last', 'none'])
def test_sampler_rng_and_slices(T1, seed, step, where):
    """seeds with the high key word set, the last 32-bit step, and data-parallel slices at session 0, in the middle, at
    Bg-1 and empty (B = 0: only the pool runs, its table must still be right)"""
    Bg, K = 90, 51
    rs = np.random.RandomState(T1 + step % 1000)
    allc = _ids(rs, (Bg, T1), Bg * T1 * 3 // 4, 2000)
    buf = _ids(rs, (1500,), 700, 2000)
    sess0, B = {'first': (0, 5), 'middle': (44, 5), 'last': (Bg - 1, 1), 'none': (30, 0)}[where]
    if T1 == 2:
        B = min(B * 20, Bg - sess0)
    _run_case(allc, buf, K, 300, seed, step, sess0, B)


@pytest.mark.gpu
@pytest.mark.parametrize('nfb_delta', [None, -1, 0, 1, 500])
def test_sampler_n_from_buffer(nfb_delta):
    """n_from_buffer 0, the buffer's nonzero count minus one, the count, and above it; the buffer's zeros are
    interleaved with its samples"""
    rs = np.random.RandomState(8)
    allc = _ids(rs, (30, 11), 200, 5000)
    buf = _ids(rs, (2000,), 611, 5000)
    nfb = 0 if nfb_delta is None else 611 + nfb_delta
    _run_case(allc, buf, 100, nfb, 2024, 9, 10, 8, n_pool=200 + min(nfb, 611))


# ------------------------------------------------------------------------------------------------ argument checks
def _reject(over):
    torch = pytest.importorskip('torch')
    _, _, ops = _lib_ctx()
    a = dict(Bg=6, T1=5, sess0=0, B=6, buf_len=50, K=5, nfb=10)
    a.update(over)
    rs = np.random.RandomState(1)
    allc_d = torch.from_numpy(_ids(rs, (6, 5), 20, 100)).cuda()
    buf_d = torch.from_numpy(_ids(rs, (50,), 20, 100)).cuda()
    n_out = 6 * 5 * max(a['K'], 1) * 2
    out = torch.full((n_out,), SENT64, dtype=torch.int64, device='cuda')
    ou = torch.full((n_out,), SENT32, dtype=torch.int32, device='cuda')
    need = ops.sample_negatives_workspace(a['Bg'], max(a['T1'], 2), max(a['buf_len'], 0), max(a['K'], 1))
    ws = torch.zeros(need + GUARD, dtype=torch.uint8, device='cuda')
    ws_bytes = need - 1 if over.get('short') else need
    rc, _, _ = _call_uidx(torch, allc_d, a['Bg'], a['T1'], a['sess0'], a['B'], buf_d, a['buf_len'], a['K'], a['nfb'], 1, 1,
                          out, ou, ws, ws_bytes)
    torch.cuda.synchronize()
    assert bool((out == SENT64).all()) and bool((ou == SENT32).all()), 'a rejected call wrote its outputs'
    return rc


@pytest.mark.gpu
@pytest.mark.parametrize('over,rc', [
    (dict(T1=1), NAR_ERR_INVALID),
    (dict(K=0), NAR_ERR_INVALID),
    (dict(K=-3), NAR_ERR_INVALID),
    (dict(sess0=1), NAR_ERR_INVALID),                           # sess0 + B > Bg
    (dict(sess0=0, B=7), NAR_ERR_INVALID),
    (dict(nfb=-1), NAR_ERR_INVALID),
    (dict(K=820), NAR_ERR_UNSUPPORTED),                         # K*20 > 16384
    (dict(short=True), NAR_ERR_WORKSPACE),                      # one byte short of nar_sample_negatives_workspace
], ids=['T1_1', 'K_0', 'K_neg', 'slice_past_Bg', 'B_past_Bg', 'n_from_buffer_neg', 'K_820', 'workspace_short'])
def test_sampler_rejects(over, rc):
    assert _reject(over) == rc


@pytest.mark.gpu
def test_sampler_rejects_negative_buf_len():
    """a negative buffer length is rejected before any launch, by the sampler and by its workspace query"""
    from chameleon_recsys_b200._lib import load
    n = C.c_int64(0)
    assert load().nar_sample_negatives_workspace(6, 5, -1, 5, C.byref(n)) == NAR_ERR_INVALID
    assert _reject(dict(buf_len=-8)) == NAR_ERR_INVALID
