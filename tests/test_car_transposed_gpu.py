"""The candidate rows of CAR layer 1 stored transposed (H1cT [C, ldr]) and the two layer-2 GEMMs that read them:
nar_car_combine_t against the transpose of nar_car_combine (same bits, unwritten padding columns untouched), the
forward with an MN-major A against the K-major forward (same bits at bf16x3 and at 3xTF32 with a B_lo plane), and the
weight gradient computed as dW^T = dY^T * X with D stored transposed (nar_gemm_tf32_dt) against fp64 and against the
MN-major x MN-major weight gradient it replaces."""
import pytest
import torch

from chameleon_recsys_b200 import ops
from chameleon_recsys_b200._lib import NarError, check, load

pytestmark = pytest.mark.gpu

BAR = 3e-3            # single-pass TF32 against fp64: max |D - ref| / max |ref|


def _ld(n):
    return (n + 3) // 4 * 4


def _combine_inputs(L, K, C, U, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    P = L + 3
    pos_idx = torch.randperm(P, device='cuda', generator=g)[:L].to(torch.int32)
    neg = torch.randint(0, U, (P, K), device='cuda', generator=g, dtype=torch.int32)
    PP = torch.randn(L, C, device='cuda', generator=g)
    PC = torch.randn(L, C, device='cuda', generator=g)
    PI = torch.randn(U, C, device='cuda', generator=g)
    PP[:, ::7] = 0.0                                           # signed zeros through leaky_relu
    PP[::2, ::7] = -0.0
    return pos_idx, neg, PP, PC, PI


def _combine(L, K, C, pos_idx, neg, PP, PC, PI):
    H1c = torch.empty(L * (K + 1), C, device='cuda')
    check(load().nar_car_combine(ops._p(PP), ops._p(PC), ops._p(PI), ops._p(pos_idx), ops._p(neg), L, K, C, ops.ACT_LEAKY,
                                 ops._p(H1c), ops._stream()), 'nar_car_combine')
    return H1c


def _combine_t(L, K, C, ldr, pos_idx, neg, PP, PC, PI, fill=float('nan')):
    H1cT = torch.full((C, ldr), fill, device='cuda')
    check(load().nar_car_combine_t(ops._p(PP), ops._p(PC), ops._p(PI), ops._p(pos_idx), ops._p(neg), L, K, C, ops.ACT_LEAKY,
                                   ops._p(H1cT), ldr, ops._stream()), 'nar_car_combine_t')
    return H1cT


@pytest.mark.parametrize('L,K,C,U,pad', [(462, 50, 1024, 1001, 22), (3, 2, 12, 5, 0), (5, 6, 200, 9, 13), (37, 9, 136, 40, 4)])
def test_combine_t_is_the_transpose(L, K, C, U, pad):
    """G1's 462 positions x 51 candidates (ldr rounded up to 32 rows, as the engine carves it), and tiny shapes with a
    ragged last 32-row block, a column tail inside a 128-wide block, and padding columns past L*(1+K)."""
    Rc = L * (K + 1)
    ldr = _ld(Rc + pad)
    ins = _combine_inputs(L, K, C, U, seed=L * 31 + K)
    ref = _combine(L, K, C, *ins)
    got = _combine_t(L, K, C, ldr, *ins)
    torch.cuda.synchronize()
    assert torch.equal(got[:, :Rc].t().contiguous().view(torch.int32), ref.view(torch.int32))
    assert bool(torch.isnan(got[:, Rc:]).all()), 'columns past L*(1+K) were written'


def test_combine_t_rejects_bad_strides():
    L, K, C = 4, 3, 16
    pos_idx, neg, PP, PC, PI = _combine_inputs(L, K, C, 7, seed=1)
    for ldr in (L * (K + 1) - 4, L * (K + 1) + 2):              # too short; not a multiple of 4
        H1cT = torch.empty(C, _ld(ldr) + 4, device='cuda')
        with pytest.raises(NarError):
            check(load().nar_car_combine_t(ops._p(PP), ops._p(PC), ops._p(PI), ops._p(pos_idx), ops._p(neg), L, K, C,
                                           ops.ACT_LEAKY, ops._p(H1cT), ldr, ops._stream()), 'nar_car_combine_t')


@pytest.mark.parametrize('precision', [4, 3])
@pytest.mark.parametrize('M,N,K', [(23562, 1024, 1024), (35, 200, 72), (300, 128, 1000)])
def test_forward_mn_major_a_same_bits(precision, M, N, K):
    """Y = tanh(A W + b) with A read MN-major from A^T [K, ldr] equals the K-major forward bit for bit: the same fragment
    values enter the same MMAs in the same order (bf16x3 splits A in registers; 3xTF32 with the weights' B_lo plane)."""
    g = torch.Generator(device='cuda').manual_seed(M + N + K + precision)
    A = torch.randn(M, K, device='cuda', generator=g)
    ldr = _ld(M) + 4
    AT = torch.zeros(K, ldr, device='cuda')
    AT[:, :M] = A.t()
    W = torch.randn(K, N, device='cuda', generator=g) / 32
    b = torch.randn(N, device='cuda', generator=g) * 0.1
    Y0 = torch.full((M, N), float('nan'), device='cuda')
    Y1 = torch.full((M, N), float('nan'), device='cuda')
    if precision == 4:
        plane = ops.pack_bf16x3(W, K, N)
        kw = dict(ldb=0, b_bf16=plane, ld_bf16=plane.stride(0))
        Bop = None
    else:
        Wlo = torch.empty_like(W)
        ops.tf32_lo(W, W.numel(), Wlo)
        kw = dict(b_kmajor=False, b_lo=Wlo)
        Bop = W
    ops.gemm(A, Bop, Y0, M, N, K, a_kmajor=True, bias=b, act=ops.ACT_TANH, precision=precision, **kw)
    ops.gemm(AT, Bop, Y1, M, N, K, a_kmajor=False, lda=ldr, bias=b, act=ops.ACT_TANH, precision=precision, **kw)
    torch.cuda.synchronize()
    assert not torch.isnan(Y0).any()
    assert torch.equal(Y1.view(torch.int32), Y0.view(torch.int32))


def _wgrad_t(X, XT, ldr, dY, n_in, n_out, rows, ldd, fill, precision=1):
    """dW [n_in, ldd] = fill + X^T dY, as dW^T = dY^T X with D stored transposed"""
    D = torch.full((n_in, ldd), fill, device='cuda')
    ops.gemm(dY, XT, D, n_out, n_in, rows, a_kmajor=False, b_kmajor=True, ldb=ldr, accumulate=True, split_k=0,
             precision=precision, trans_d=True)
    return D


@pytest.mark.parametrize('n_in,n_out,rows', [(1024, 1024, 23562), (130, 198, 1000), (64, 32, 100)])
def test_wgrad_transposed_d(n_in, n_out, rows):
    """CAR layer 2's weight gradient at G1 (64 tiles, split-K to one wave) and ragged blocks whose output columns end
    inside a 4-wide store: against fp64 at the TF32 bar, and against the MN-major x MN-major weight gradient within the
    fp32 error of two summation orders of the same TF32 products."""
    g = torch.Generator(device='cuda').manual_seed(n_in * 7 + n_out + rows)
    ldx, ldy, ldd, ldr = _ld(n_in), _ld(n_out), _ld(n_out) + 4, _ld(rows) + 4
    X = torch.zeros(rows, ldx, device='cuda')
    X[:, :n_in] = torch.randn(rows, n_in, device='cuda', generator=g)
    dY = torch.zeros(rows, ldy, device='cuda')
    dY[:, :n_out] = torch.randn(rows, n_out, device='cuda', generator=g)
    XT = torch.zeros(n_in, ldr, device='cuda')
    XT[:, :rows] = X[:, :n_in].t()
    got = _wgrad_t(X, XT, ldr, dY, n_in, n_out, rows, ldd, 1.0)
    old = torch.full((n_in, ldd), 1.0, device='cuda')
    ops.gemm(X, dY, old, n_in, n_out, rows, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=0, precision=1)
    torch.cuda.synchronize()
    Xd, dYd = X[:, :n_in].double(), dY[:, :n_out].double()
    ref = Xd.t() @ dYd
    abs_sum = Xd.abs().t() @ dYd.abs()
    assert bool((got[:, n_out:] == 1.0).all()), 'columns past n_out were written'
    g_, o_ = got[:, :n_out].double() - 1.0, old[:, :n_out].double() - 1.0
    rel = float((g_ - ref).abs().max() / ref.abs().max())
    assert rel < BAR, rel
    # each result is within ~(rows + 2) * 2^-24 * (sum |terms| + the 1.0 it lands on) of the exact sum of its (identical)
    # TF32 products; 2x for a rounding mode other than round-to-nearest in the tensor cores' accumulation
    assert bool(((g_ - o_).abs() <= 4 * (rows + 2) * 2.0 ** -24 * (abs_sum + 1.0)).all())


def test_wgrad_transposed_d_3xtf32():
    """the 3xTF32 form (B split in-kernel) against fp64 at ~fp32 accuracy"""
    n_in, n_out, rows = 256, 192, 2000
    g = torch.Generator(device='cuda').manual_seed(5)
    X = torch.randn(rows, n_in, device='cuda', generator=g)
    dY = torch.randn(rows, n_out, device='cuda', generator=g)
    XT = X.t().contiguous()
    got = _wgrad_t(X, XT, rows, dY, n_in, n_out, rows, n_out, 0.0, precision=3)
    torch.cuda.synchronize()
    Xd, dYd = X.double(), dY.double()
    ref = Xd.t() @ dYd
    assert float((got.double() - ref).abs().max() / ref.abs().max()) < 2e-5


def test_transposed_d_rejects_other_forms():
    """nar_gemm_tf32_dt takes A MN-major, B K-major and no epilogue beyond accumulate"""
    A = torch.randn(64, 64, device='cuda')
    B = torch.randn(64, 64, device='cuda')
    D = torch.zeros(64, 64, device='cuda')
    bias = torch.zeros(64, device='cuda')
    for kw in (dict(a_kmajor=True, b_kmajor=True), dict(a_kmajor=False, b_kmajor=False), dict(a_kmajor=False, bias=bias),
               dict(a_kmajor=False, act=ops.ACT_TANH)):
        with pytest.raises(NarError):
            ops.gemm(A, B, D, 64, 64, 64, precision=1, trans_d=True, **kw)
