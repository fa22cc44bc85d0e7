"""The CAR layer-1 backward formed in the layer-2 dgrad epilogue (nar_gemm_epilogue.car_*) against the plain path: the
dgrad with leaky' read from the H1c that nar_car_combine writes, then the per-position / per-id sums of its rows in
fp64.  dPP, and dPI where every id is drawn once, must be the same bits (leaky' recomputed from PP / PC + PI); dPC and
dPI of sampler-like draws (popular ids, the padding slot drawn several times) agree to fp32 summation error."""
import pytest
import torch

from chameleon_recsys_b200 import ops
from chameleon_recsys_b200._lib import NarError, check, load

pytestmark = pytest.mark.gpu


def _draws(L, K, U, unique, g):
    """pos_idx [L] (positions of a [P, K] neg_uidx, not in order) and neg_uidx.  unique: every id of [0, L*K) exactly once
    (U = L*K + 1).  Otherwise a click's K ids are distinct, drawn with Zipf-like popularity from [0, U-1), and every
    fifth click ends in a run of the padding slot U-1."""
    P = L + 7
    pos_idx = torch.randperm(P, device='cuda', generator=g)[:L].to(torch.int32)
    neg = torch.full((P, K), U - 1, dtype=torch.int32, device='cuda')
    if unique:
        neg[pos_idx.long()] = torch.randperm(L * K, device='cuda', generator=g).view(L, K).to(torch.int32)
    else:
        w = 1.0 / torch.arange(1, U, device='cuda', dtype=torch.float64)
        ids = torch.multinomial(w.expand(L, U - 1), K, replacement=False, generator=g).to(torch.int32)
        pad = torch.arange(L, device='cuda') % 5 == 0
        ids[pad, K - 1 - K // 4:] = U - 1
        neg[pos_idx.long()] = ids
    return pos_idx, neg


def _operands(L, K, Cin, Cout, U, unique, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    pos_idx, neg = _draws(L, K, U, unique, g)
    PP = torch.randn(L, Cin, device='cuda', generator=g)
    PC = torch.randn(L, Cin, device='cuda', generator=g)
    PI = torch.randn(U, Cin, device='cuda', generator=g)
    PP[:, ::7] = 0.0                                                   # pre exactly 0 (both zeros) on the positives
    PP[::2, ::7] = -0.0
    if unique:                                                         # ... and PC + PI == 0 exactly on negatives
        u = neg[pos_idx.long()].long()                                 # [L, K], each id once
        PI[u[:, ::3], 5::11] = -PC[:, None, 5::11]
    dEc = torch.randn(L * (K + 1), Cout, device='cuda', generator=g)
    W2 = torch.randn(Cin, Cout, device='cuda', generator=g) / 32
    return pos_idx, neg, PP, PC, PI, dEc, W2


def _plain(L, K, Cin, Cout, pos_idx, neg, PP, PC, PI, dEc, W2, precision=1):
    Rc = L * (K + 1)
    H1c = torch.empty(Rc, Cin, device='cuda')
    check(load().nar_car_combine(ops._p(PP), ops._p(PC), ops._p(PI), ops._p(pos_idx), ops._p(neg), L, K, Cin, ops.ACT_LEAKY,
                                 ops._p(H1c), ops._stream()), 'nar_car_combine')
    dH1 = torch.empty(Rc, Cin, device='cuda')
    ops.gemm(dEc, W2, dH1, Rc, Cin, Cout, precision=precision, dact=ops.ACT_LEAKY, aux=H1c)
    return dH1.view(L, K + 1, Cin)


def _fused(L, K, Cin, Cout, U, pos_idx, neg, PP, PC, PI, dEc, W2, precision=1):
    dPP = torch.full((L, Cin), float('nan'), device='cuda')
    dPC = torch.zeros(L, Cin, device='cuda')
    dPI = torch.zeros(U, Cin, device='cuda')
    ops.gemm(dEc, W2, None, L * (K + 1), Cin, Cout, precision=precision, dact=ops.ACT_LEAKY,
             car=dict(pp=PP, pc=PC, pi=PI, pos_idx=pos_idx, neg_uidx=neg, dpp=dPP, dpc=dPC, dpi=dPI, k=K))
    torch.cuda.synchronize()
    return dPP, dPC, dPI


def _sums(rows, L, K, U, u):
    """fp64 dPC / dPI from the plain dgrad's rows, and the sums of |terms| that bound fp32 summation error"""
    neg_rows = rows[:, 1:, :].double()                                 # [L, K, C]
    dPC, aPC = neg_rows.sum(1), neg_rows.abs().sum(1)
    flat = neg_rows.reshape(L * K, -1)
    dPI = torch.zeros(U, flat.shape[1], dtype=torch.float64, device='cuda').index_add_(0, u.reshape(-1), flat)
    aPI = torch.zeros_like(dPI).index_add_(0, u.reshape(-1), flat.abs())
    cnt = torch.bincount(u.reshape(-1), minlength=U).double()[:, None]
    return dPC, aPC, float(K), dPI, aPI, cnt


def _close(got, ref, abs_sum, n_terms):
    # |fl(sum) - sum| <= (n - 1) * 2^-24 * sum |terms| for any order of fp32 additions (+1: the add onto the zeroed buffer)
    tol = (torch.as_tensor(n_terms, dtype=torch.float64) + 1) * 2.0 ** -24 * abs_sum + 1e-30
    err = (got.double() - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())


@pytest.mark.parametrize('L,K,Cin,Cout,precision', [(462, 50, 1024, 1024, 1), (233, 100, 1024, 1024, 1),  # G1 / Adressa
                                                    (37, 50, 1000, 1024, 1),        # N not a multiple of 128
                                                    (5, 127, 256, 96, 1),           # 128 rows per position
                                                    (37, 50, 1000, 1024, 3)])       # 3xTF32 backward
def test_unique_draws_are_bit_identical(L, K, Cin, Cout, precision):
    U = L * K + 1
    args = _operands(L, K, Cin, Cout, U, True, seed=L + K)
    rows = _plain(L, K, Cin, Cout, *args, precision=precision)
    dPP, dPC, dPI = _fused(L, K, Cin, Cout, U, *args, precision=precision)
    pos_idx, neg = args[0], args[1]
    u = neg[pos_idx.long()].long()
    assert torch.equal(dPP, rows[:, 0, :])
    assert torch.equal(dPI[u.reshape(-1)], rows[:, 1:, :].reshape(L * K, Cin))
    assert not bool(dPI[U - 1].any())                                  # the padding slot was never drawn
    ref, a, n, _, _, _ = _sums(rows, L, K, U, u)
    _close(dPC, ref, a, n)


@pytest.mark.parametrize('L,K,Cin', [(462, 50, 1024), (233, 100, 1024), (61, 50, 1000), (3, 1, 128)])
def test_sampler_like_draws(L, K, Cin):
    """Rc = L * (1 + K) is not a multiple of 128 in every case, and positions straddle M tiles."""
    Cout = 1024
    U = K * 20 + 1
    args = _operands(L, K, Cin, Cout, U, False, seed=3 * L + K)
    rows = _plain(L, K, Cin, Cout, *args)
    dPP, dPC, dPI = _fused(L, K, Cin, Cout, U, *args)
    pos_idx, neg = args[0], args[1]
    u = neg[pos_idx.long()].long()
    if K > 1:                                                          # popular ids are drawn by several positions
        assert int(torch.bincount(u[:, :K // 2].reshape(-1), minlength=U).max()) > 1
    assert bool((u == U - 1).any())
    assert torch.equal(dPP, rows[:, 0, :])
    rPC, aPC, n, rPI, aPI, cnt = _sums(rows, L, K, U, u)
    _close(dPC, rPC, aPC, n)
    _close(dPI, rPI, aPI, cnt)


def test_dpp_and_dpc_are_reproducible():
    L, K, Cin, Cout = 462, 50, 1024, 1024
    U = K * 20 + 1
    args = _operands(L, K, Cin, Cout, U, False, seed=11)
    a = _fused(L, K, Cin, Cout, U, *args)
    b = _fused(L, K, Cin, Cout, U, *args)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_rejects_what_it_does_not_implement():
    L, K, Cin, Cout = 4, 10, 128, 128
    U = K * 20 + 1
    pos_idx, neg, PP, PC, PI, dEc, W2 = _operands(L, K, Cin, Cout, U, False, seed=1)
    Rc = L * (K + 1)
    car = dict(pp=PP, pc=PC, pi=PI, pos_idx=pos_idx, neg_uidx=neg, dpp=torch.empty_like(PP), dpc=torch.zeros_like(PC),
               dpi=torch.zeros_like(PI), k=K)
    D = torch.empty(Rc, Cin, device='cuda')
    for kw in (dict(D=D), dict(precision=3, b_lo=W2), dict(precision=4), dict(split_k=2, accumulate=True),
               dict(bias=torch.zeros(Cin, device='cuda')), dict(aux=D), dict(M=Rc - 1), dict(car=dict(car, k=K + 1))):
        call = dict(D=None, M=Rc, precision=1, car=car)
        call.update(kw)
        with pytest.raises(NarError):
            ops.gemm(dEc, W2, call.pop('D'), call.pop('M'), Cin, Cout, dact=ops.ACT_LEAKY, **call)
