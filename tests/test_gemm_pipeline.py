"""The wgmma GEMM keeps one k-tile's MMAs in flight while the next k-tile is staged, with STAGES - 1 k-tiles of TMA
ahead (STAGES = 4 with a transpose / split pass of B, 3 with a B_lo plane or without that pass - two CTAs per SM) and
double-buffered A fragments / transposed B tiles.  These cases walk the
k-tile counts around those depths for every operand major and precision, ragged M / N tails, split-K splits whose last
split is one or two k-tiles, the fused epilogues, and run-to-run bit identity; results against fp64.

Error bars (max |D - ref| / max |ref|): single-pass TF32 3e-3, 3xTF32 2e-5, bf16x3 1e-4."""
import pytest
import torch

from chameleon_recsys_b200 import ops

pytestmark = pytest.mark.gpu

BAR = {0: 3e-3, 1: 2e-5, 2: 2e-5, 4: 1e-4}
PRECISION = {0: 1, 1: 3, 2: 3, 4: 4}
# 1, 2, STAGES - 1, STAGES, STAGES + 1, 2 STAGES + 1 for STAGES = 4 and STAGES = 3, and 37
K_TILES = (1, 2, 3, 4, 5, 7, 9, 37)
MAJORS = [(True, True), (True, False), (False, True), (False, False)]


def _ld(n):
    return (n + 3) // 4 * 4


def run_gemm(mode, M, N, K, a_k=True, b_k=True, epi='none', split=1, seed=0):
    """D = epilogue(A B^T) through ops.gemm with the given operand majors; returns (D[:, :N], fp64 reference, D)."""
    g = torch.Generator(device='cuda').manual_seed(seed * 1000003 + M * 7 + N * 3 + K)
    A = torch.zeros(M if a_k else K, _ld(K if a_k else M), device='cuda')
    A[:, :(K if a_k else M)] = torch.randn(A.shape[0], K if a_k else M, device='cuda', generator=g)
    if epi == 'bias_tanh':
        A /= 30
    Al = (A[:, :K] if a_k else A[:, :M].t()).double()                  # [M, K]
    kw = dict(precision=PRECISION[mode])
    if mode == 4:
        W = torch.randn(K, _ld(N), device='cuda', generator=g)           # [in, out], packed into the bf16x3 plane
        plane = ops.pack_bf16x3(W, K, N)
        B, ldb, b_k = None, 0, True
        Bl = W[:, :N].t().double()
        kw.update(b_bf16=plane, ld_bf16=plane.stride(0))
    else:
        B = torch.zeros(N if b_k else K, _ld(K if b_k else N), device='cuda')
        B[:, :(K if b_k else N)] = torch.randn(B.shape[0], K if b_k else N, device='cuda', generator=g)
        ldb = B.stride(0)
        Bl = (B[:, :K] if b_k else B[:, :N].t()).double()               # [N, K]
        if mode == 2:
            Blo = torch.empty_like(B)
            ops.tf32_lo(B, B.numel(), Blo)
            kw['b_lo'] = Blo
    ref = Al @ Bl.t()
    D = torch.full((M, _ld(N)), 7.0, device='cuda')
    if epi == 'bias_leaky':
        bias = torch.randn(_ld(N), device='cuda', generator=g)
        ref = torch.nn.functional.leaky_relu(ref + bias[:N].double(), 0.2)
        kw.update(bias=bias, act=ops.ACT_LEAKY)
    elif epi == 'bias_tanh':
        bias = torch.randn(_ld(N), device='cuda', generator=g) * 0.1
        ref = torch.tanh(ref + bias[:N].double())
        kw.update(bias=bias, act=ops.ACT_TANH)
    elif epi == 'dact_leaky':
        aux = torch.randn(M, _ld(N), device='cuda', generator=g)           # a separate tensor, not D
        ref = ref * torch.where(aux[:, :N] > 0, 1.0, 0.2).double()
        kw.update(dact=ops.ACT_LEAKY, aux=aux)
    elif epi == 'accumulate':
        D.fill_(1.0)
        ref = ref + 1.0
        kw.update(accumulate=True, split_k=split)
    else:
        assert epi == 'none', epi
    ops.gemm(A, B, D, M, N, K, a_kmajor=a_k, b_kmajor=b_k, lda=A.stride(0), ldb=ldb, **kw)
    torch.cuda.synchronize()
    return D[:, :N], ref, D


def check(mode, got, ref, D, N, pad):
    assert not torch.isnan(got).any()
    rel = float((got.double() - ref).abs().max() / ref.abs().max())
    assert rel < BAR[mode], rel
    if D.shape[1] > N:
        assert bool((D[:, N:] == pad).all()), 'columns past N were written'


@pytest.mark.parametrize('n_kt', K_TILES)
@pytest.mark.parametrize('a_k,b_k', MAJORS)
@pytest.mark.parametrize('mode', [0, 1, 2])
def test_k_tile_counts_tf32(mode, a_k, b_k, n_kt):
    M, N, K = 129, 200, 32 * n_kt
    got, ref, D = run_gemm(mode, M, N, K, a_k, b_k)
    check(mode, got, ref, D, N, 7.0)


@pytest.mark.parametrize('n_kt', K_TILES)
def test_k_tile_counts_bf16x3(n_kt):
    M, N, K = 129, 200, 32 * n_kt
    got, ref, D = run_gemm(4, M, N, K)
    check(4, got, ref, D, N, 7.0)


@pytest.mark.parametrize('mode,M,N,K', [(0, 257, 130, 100), (1, 300, 61, 300), (2, 131, 255, 1000), (4, 383, 129, 72),
                                        (4, 130, 1000, 1180)])
def test_ragged_tails(mode, M, N, K):
    """M and N off the 128 grid, K off the 32 grid (the last k-tile is partly out of range: TMA fills zeros)."""
    for a_k, b_k in (MAJORS if mode != 4 else [(True, True)]):
        got, ref, D = run_gemm(mode, M, N, K, a_k, b_k)
        check(mode, got, ref, D, N, 7.0)


def _split_sizes(k_tiles, split):
    per = -(-k_tiles // split)                 # the library's split policy: ceil, then no empty splits
    n = -(-k_tiles // per)
    return [min(per, k_tiles - i * per) for i in range(n)]


@pytest.mark.parametrize('mode,a_k,b_k', [(0, False, False), (0, True, True), (1, False, False), (2, True, False)])
@pytest.mark.parametrize('k_tiles,split,last', [(13, 4, 1), (10, 3, 2), (5, 2, 2), (6, 6, 1), (9, 1, 9)])
def test_split_k_accumulate(mode, a_k, b_k, k_tiles, split, last):
    assert _split_sizes(k_tiles, split)[-1] == last
    M, N = 200, 129
    got, ref, D = run_gemm(mode, M, N, 32 * k_tiles, a_k, b_k, epi='accumulate', split=split)
    check(mode, got, ref, D, N, 1.0)


@pytest.mark.parametrize('mode,epi', [(0, 'bias_leaky'), (0, 'bias_tanh'), (0, 'dact_leaky'), (1, 'bias_leaky'),
                                      (1, 'dact_leaky'), (2, 'bias_tanh'), (2, 'dact_leaky'), (4, 'bias_leaky'),
                                      (4, 'bias_tanh')])
def test_epilogues(mode, epi):
    for a_k, b_k in (MAJORS if mode != 4 else [(True, True)]):
        got, ref, D = run_gemm(mode, 129, 200, 32 * 9 + 12, a_k, b_k, epi=epi)
        check(mode, got, ref, D, 200, 7.0)


@pytest.mark.parametrize('mode,a_k,b_k', [(4, True, True), (0, True, True), (0, True, False), (1, False, True),
                                          (2, False, False)])
def test_bitwise_repeatable(mode, a_k, b_k):
    """One non-split GEMM twice on the same inputs: the same bits (each accumulator's MMA order is fixed)."""
    _, _, D1 = run_gemm(mode, 1000, 1024, 1024, a_k, b_k, epi='bias_tanh')
    _, _, D2 = run_gemm(mode, 1000, 1024, 1024, a_k, b_k, epi='bias_tanh')
    assert torch.equal(D1.view(torch.int32), D2.view(torch.int32))
