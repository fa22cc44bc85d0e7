"""The CAR layer-1 combine kernels against a plain numpy fp32 reference, bit for bit.

nar_car_combine (H1c [L*(1+K), C]), nar_car_combine_t (the same rows stored transposed, H1cT [C, ldr]) and
nar_car_combine_grid (H1 [Q*Nc, C] for every query x candidate pair) each round exactly once per element: one fp32 add
PI[u] + PC[l] (none for a positive row, which is PP[l]), then the activation.  The build has no fast-math, so the
reference below is that add in numpy float32 followed by ``where(x > 0, x, float32(0.2) * x)``, and the kernels must give
its bits, signed zeros and subnormals included.  test_reference_is_fp64_rounded_once shows the reference equals the
fp64 sum and product rounded once to fp32.

The operands are built to catch indexing and tail errors: pos_idx is a permutation with gaps (not the identity), neg_uidx
holds repeated ids and the padding slot U-1, and the values hold +-0, exact cancellations PI = -PC, negative subnormals
and magnitudes near 1e30.  Outputs start from a signalling-NaN sentinel and carry guard rows (and, for H1cT, the padding
columns past L*(1+K)) that must keep it.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip('torch')

NAR_ERR_INVALID, NAR_ERR_UNSUPPORTED = -1, -2
ACT_NONE, ACT_LEAKY = 0, 1
SENT_BITS = 0x7FA5A5A5
GUARD_ROWS = 2


# ------------------------------------------------------------------------------------------------ operands / reference
def _values(rs, rows, C_):
    """normal values with special columns: +0, -0, negative subnormals, +-1e30-scale, and a column that the cancellation
    pattern below makes PI = -PC"""
    v = rs.standard_normal((rows, C_)).astype(np.float32)
    col = np.arange(C_) % 8
    v[:, col == 0] = np.float32(0.0)
    v[:, col == 1] = np.float32(-0.0)
    v[:, col == 2] = -np.float32(rs.randint(1, 1 << 22, size=(rows, int((col == 2).sum())))) * np.float32(2.0 ** -149)
    v[:, col == 3] = (rs.standard_normal((rows, int((col == 3).sum()))) * 1e30).astype(np.float32)
    v[:, col == 4] = np.float32(1.5) * np.float32(rs.randint(-3, 4, size=(rows, int((col == 4).sum()))))
    return v


def _operands(L, K, C_, U, seed):
    rs = np.random.RandomState(seed)
    P = L + max(3, L // 4)                                       # neg_uidx rows; pos_idx skips some of them
    pos_idx = rs.permutation(P)[:L].astype(np.int32)
    neg = rs.randint(0, U, size=(P, K)).astype(np.int32)
    neg[:, 0] = U - 1                                            # the padding slot
    if K > 2:
        neg[:, 2] = neg[:, 1]                                    # repeated ids within a row
    PP = _values(rs, L, C_)
    PC = _values(rs, L, C_)
    PI = _values(rs, U, C_)
    col = np.arange(C_) % 8
    PI[:, col == 4] = -PI[:, col == 4]                           # col 4 of PC and PI share a small grid: PI = -PC often
    PI[::2, col == 1] = np.float32(0.0)                          # -0 + +0 = +0 on even rows, -0 + -0 = -0 on odd
    PI[U - 1, :] = -PC[0, :]                                     # the padding row cancels position 0's context exactly
    PI[0, col == 2] = np.float32(2.0 ** -149) * 3
    return pos_idx, neg, PP, PC, PI


def _leaky(x):
    return np.where(x > 0, x, np.float32(0.2) * x).astype(np.float32)


def _act(x, act):
    return _leaky(x) if act == ACT_LEAKY else x


def _ref_rows(pos_idx, neg, PP, PC, PI, K, act):
    """H1c [L*(1+K), C] in numpy float32"""
    L, C_ = PP.shape
    u = neg[pos_idx]                                             # [L, K]
    with np.errstate(over='ignore'):
        x = PI[u] + PC[:, None, :]                               # [L, K, C]: one fp32 add
    out = np.empty((L, K + 1, C_), np.float32)
    out[:, 0] = _act(PP, act)
    out[:, 1:] = _act(x, act)
    return out.reshape(L * (K + 1), C_)


def test_reference_is_fp64_rounded_once():
    """CPU: the numpy float32 add of the reference equals the exact (fp64) sum rounded once to fp32, and its leaky_relu
    equals the exact product 0.2f * x rounded once, on the test operands themselves (specials included): each reference
    step is the correctly rounded result, as the kernels' fp32 instructions are"""
    pos_idx, neg, PP, PC, PI = _operands(37, 5, 1028, 23, seed=4)
    u = neg[pos_idx]
    x32 = PI[u] + PC[:, None, :]
    x64 = PI[u].astype(np.float64) + PC[:, None, :].astype(np.float64)
    assert np.array_equal(x32.view(np.int32), x64.astype(np.float32).view(np.int32))
    y32 = _leaky(x32)                                            # the kernel applies leaky_relu to the rounded sum
    x = x32.astype(np.float64)
    y64 = np.where(x > 0, x, np.float64(np.float32(0.2)) * x).astype(np.float32)
    assert np.array_equal(y32.view(np.int32), y64.view(np.int32))
    # the operands reach the edges the docstring names
    assert (np.signbit(x32) & (x32 == 0)).any() and (~np.signbit(x32) & (x32 == 0)).any()
    assert ((x32 < 0) & (np.abs(x32) < np.finfo(np.float32).tiny)).any()
    assert (np.abs(x32) > 1e29).any()


# ------------------------------------------------------------------------------------------------ GPU helpers
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sentinel(n):
    return torch.full((n,), SENT_BITS, dtype=torch.int32, device='cuda').view(torch.float32)


def _bits(t):
    return t.view(torch.int32).cpu().numpy()


def _assert_bits(got, ref):
    g, r = got.view(np.int32), ref.view(np.int32)
    bad = np.argwhere(g != r)
    assert bad.size == 0, (bad[:5], g[tuple(bad[0])] if bad.size else None)


def _lib():
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import load
    return load(), ops


# ------------------------------------------------------------------------------------------------ nar_car_combine
KS = [1, 3, 4, 5, 50, 100, 500]
CS = [4, 12, 1020, 1024, 1028]
LS = [1, 37, 462]


def _combine_shapes():
    """every K x C pair; L cycles through 1, 37 and 462 (the largest that keeps the output under 24M floats)"""
    out = []
    for i, K in enumerate(KS):
        for j, C_ in enumerate(CS):
            k = (i + j) % 3
            while k > 0 and LS[k] * (K + 1) * C_ > 24_000_000:
                k -= 1
            out.append((LS[k], K, C_))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('L,K,C_', _combine_shapes())
def test_combine(L, K, C_):
    """K below 4 and not a multiple of 4 run the remainder loop; C = 1028 needs a second column pass past 256*4"""
    lib, ops = _lib()
    U = 2 * K + 7
    pos_idx, neg, PP, PC, PI = _operands(L, K, C_, U, seed=L * 131 + K * 7 + C_)
    ref = _ref_rows(pos_idx, neg, PP, PC, PI, K, ACT_LEAKY)
    R = L * (K + 1)
    H = _sentinel((R + GUARD_ROWS) * C_)
    d = [_dev(a) for a in (PP, PC, PI, pos_idx, neg)]
    assert lib.nar_car_combine(*[ops._p(t) for t in d], L, K, C_, ACT_LEAKY, ops._p(H), ops._stream()) == 0
    got = _bits(H)
    _assert_bits(got[:R * C_].reshape(R, C_), ref)
    assert (got[R * C_:] == SENT_BITS).all(), 'write past the last row'


# ------------------------------------------------------------------------------------------------ nar_car_combine_t
def _combine_t_shapes():
    """L*(1+K) at every residue mod 32 (and so mod 4): 37*(K+1) runs through all of them for K+1 = 2..33; C ragged inside
    its 128-wide tile; plus G1 (462 positions x 51 candidates) and a two-pass C"""
    out = [(37, k1 - 1, 4 * (1 + (k1 * 13) % 45)) for k1 in range(2, 34)]
    out += [(1, 500, 132), (462, 50, 1024), (462, 50, 1028), (37, 100, 1020)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('L,K,C_', _combine_t_shapes())
def test_combine_t(L, K, C_):
    lib, ops = _lib()
    U = K + 5
    pos_idx, neg, PP, PC, PI = _operands(L, K, C_, U, seed=L * 17 + K * 3 + C_)
    ref = _ref_rows(pos_idx, neg, PP, PC, PI, K, ACT_LEAKY)
    R = L * (K + 1)
    ldr = (R + 3) // 4 * 4 + 8                                   # padding columns past R
    H = _sentinel((C_ + GUARD_ROWS) * ldr)
    d = [_dev(a) for a in (PP, PC, PI, pos_idx, neg)]
    assert lib.nar_car_combine_t(*[ops._p(t) for t in d], L, K, C_, ACT_LEAKY, ops._p(H), ldr, ops._stream()) == 0
    got = _bits(H)
    main = got[:C_ * ldr].reshape(C_, ldr)
    _assert_bits(np.ascontiguousarray(main[:, :R].T), ref)
    assert (main[:, R:] == SENT_BITS).all(), 'padding columns past L*(1+K) were written'
    assert (got[C_ * ldr:] == SENT_BITS).all(), 'write past the last row'


# ------------------------------------------------------------------------------------------------ nar_car_combine_grid
@pytest.mark.gpu
@pytest.mark.parametrize('act', [ACT_NONE, ACT_LEAKY], ids=['none', 'leaky'])
@pytest.mark.parametrize('C_', [4, 1028])
@pytest.mark.parametrize('Q', [1, 7])
@pytest.mark.parametrize('Nc', [1, 15, 16, 17, 4097])
def test_combine_grid(Nc, Q, C_, act):
    """16-row candidate blocks: one partial block, one full, one and a bit, and 257 blocks ending in a single row"""
    lib, ops = _lib()
    rs = np.random.RandomState(Nc * 11 + Q * 3 + C_ + act)
    PC = _values(rs, Q, C_)
    PI = _values(rs, Nc, C_)
    col = np.arange(C_) % 8
    PI[:, col == 4] = -PI[:, col == 4]
    PI[Nc // 2] = -PC[Q - 1]                                    # one candidate row cancels the last query exactly
    with np.errstate(over='ignore'):
        ref = _act(PI[None, :, :] + PC[:, None, :], act).reshape(Q * Nc, C_)
    H = _sentinel((Q * Nc + GUARD_ROWS) * C_)
    assert lib.nar_car_combine_grid(ops._p(_dev(PC)), ops._p(_dev(PI)), Q, Nc, C_, act, ops._p(H),
                                    ops._stream()) == 0
    got = _bits(H)
    _assert_bits(got[:Q * Nc * C_].reshape(Q * Nc, C_), ref)
    assert (got[Q * Nc * C_:] == SENT_BITS).all(), 'write past the last row'


# ------------------------------------------------------------------------------------------------ argument checks
def _small():
    L, K, C_, U = 3, 2, 8, 5
    pos_idx, neg, PP, PC, PI = _operands(L, K, C_, U, seed=1)
    return [_dev(a) for a in (PP, PC, PI, pos_idx, neg)]


@pytest.mark.gpu
@pytest.mark.parametrize('K,C_', [(2, 6), (0, 8), (-1, 8), (8193, 8)], ids=['C_not_x4', 'K_0', 'K_neg', 'K_8193'])
def test_combine_rejects(K, C_):
    lib, ops = _lib()
    d = _small()
    H = _sentinel(4096)
    assert lib.nar_car_combine(*[ops._p(t) for t in d], 3, K, C_, ACT_LEAKY, ops._p(H), ops._stream()) == NAR_ERR_INVALID
    ldr = 3 * (max(K, 1) + 1) + 4
    ldr += (-ldr) % 4
    H2 = _sentinel(8 * ldr + 64)
    assert lib.nar_car_combine_t(*[ops._p(t) for t in d], 3, K, C_, ACT_LEAKY, ops._p(H2), ldr,
                                 ops._stream()) == NAR_ERR_INVALID
    torch.cuda.synchronize()
    assert (_bits(H) == SENT_BITS).all() and (_bits(H2) == SENT_BITS).all()


@pytest.mark.gpu
@pytest.mark.parametrize('ldr,shift', [(8, 0), (4, 0), (14, 0), (16, 1)], ids=['short_by_1', 'short_by_5', 'not_x4', 'H1cT_misaligned'])
def test_combine_t_rejects(ldr, shift):
    """L*(1+K) = 9 rows: an ldr shorter than that or not a multiple of 4, or an H1cT that is not 16-byte aligned"""
    lib, ops = _lib()
    d = _small()
    H = _sentinel(8 * 16 + 64)
    assert lib.nar_car_combine_t(*[ops._p(t) for t in d], 3, 2, 8, ACT_LEAKY, C.c_void_p(H.data_ptr() + 4 * shift), ldr,
                                 ops._stream()) == NAR_ERR_INVALID
    torch.cuda.synchronize()
    assert (_bits(H) == SENT_BITS).all()


@pytest.mark.gpu
@pytest.mark.parametrize('which', ['C_not_x4', 'C_0', 'PC', 'PI', 'H1', 'Q_blocks'])
def test_combine_grid_rejects(which):
    """C not a multiple of 4, misaligned PC / PI / H1: NAR_ERR_INVALID; Q * ceil(Nc/16) above 2^31-1: NAR_ERR_UNSUPPORTED
    (checked before the launch: the buffers here are far smaller than that grid)"""
    lib, ops = _lib()
    PC = torch.zeros(64, device='cuda')
    PI = torch.zeros(64, device='cuda')
    H = _sentinel(256)
    Q, Nc, C_ = 2, 3, 8
    p = {'PC': PC.data_ptr(), 'PI': PI.data_ptr(), 'H1': H.data_ptr()}
    rc_want = NAR_ERR_INVALID
    if which in p:
        p[which] += 4
    elif which == 'C_not_x4':
        C_ = 6
    elif which == 'C_0':
        C_ = 0
    else:
        Q, Nc, rc_want = 1 << 31, 16, NAR_ERR_UNSUPPORTED
    assert lib.nar_car_combine_grid(C.c_void_p(p['PC']), C.c_void_p(p['PI']), Q, Nc, C_, ACT_LEAKY, C.c_void_p(p['H1']),
                                    ops._stream()) == rc_want
    torch.cuda.synchronize()
    assert (_bits(H) == SENT_BITS).all()
