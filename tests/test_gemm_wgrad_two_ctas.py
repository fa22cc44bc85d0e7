"""Single-pass TF32 with an MN-major B (the weight gradients dW = X^T dY, and forwards that read W [in, out]) transposes
each B tile in place inside its own pipeline stage and runs two CTAs per SM; accumulating launches with split_k=0 let
the library pick the split from the CTA slots the SMs hold.  These cases run that automatic split at the shapes the
training step launches (CAR layer 2 and the scorer's first layer at 23 600 rows, an RNN-sized block, an accumulating
dgrad) and an in-place-transposed B whose N tail ends inside a 32-wide box; results against fp64 at the single-pass
TF32 bar (max |D - ref| / max |ref| < 3e-3)."""
import pytest
import torch

from chameleon_recsys_b200 import ops

pytestmark = pytest.mark.gpu

BAR = 3e-3


def run(M, N, K, a_k, b_k, accumulate, width, fill, seed=0):
    """D[:, :N] (+)= A B^T with precision=1 and split_k=0, D `width` columns wide and filled with `fill`; returns
    (D, fp64 reference of D[:, :N])."""
    g = torch.Generator(device='cuda').manual_seed(seed * 1000003 + M * 7 + N * 3 + K)

    def operand(mn, kmajor):        # [mn, K] K-major or [K, mn] MN-major, rows padded to a multiple of 4 floats
        rows, cols = (mn, K) if kmajor else (K, mn)
        X = torch.zeros(rows, (cols + 3) // 4 * 4, device='cuda')
        X[:, :cols] = torch.randn(rows, cols, device='cuda', generator=g)
        return X, (X[:, :K] if kmajor else X[:, :mn].t()).double()
    A, Al = operand(M, a_k)
    B, Bl = operand(N, b_k)
    ref = Al @ Bl.t() + (fill if accumulate else 0.0)
    D = torch.full((M, width), fill, device='cuda')
    ops.gemm(A, B, D, M, N, K, a_kmajor=a_k, b_kmajor=b_k, accumulate=accumulate, split_k=0, precision=1)
    torch.cuda.synchronize()
    return D, ref


def check(D, ref, N, fill):
    got = D[:, :N]
    assert not torch.isnan(got).any()
    rel = float((got.double() - ref).abs().max() / ref.abs().max())
    assert rel < BAR, rel
    if D.shape[1] > N:
        assert bool((D[:, N:] == fill).all()), 'columns past N were written'


@pytest.mark.parametrize('M,N,K', [(1024, 1024, 23600), (1024, 128, 23600), (255, 510, 484)])
def test_wgrad_auto_split(M, N, K):
    """dW = X^T dY with both operands MN-major, accumulated onto 1.0: CAR layer 2 (64 tiles), the scorer's first layer
    (8 tiles), and a ragged RNN-sized block."""
    D, ref = run(M, N, K, a_k=False, b_k=False, accumulate=True, width=(N + 3) // 4 * 4, fill=1.0)
    check(D, ref, N, 1.0)


def test_dgrad_accumulate_auto_split():
    """dX += dY W^T with K-major operands, as the GRU and context-block dgrads accumulate: 8 x 8 tiles, 32 k-tiles."""
    D, ref = run(1000, 1024, 1024, a_k=True, b_k=True, accumulate=True, width=1024, fill=1.0)
    check(D, ref, 1024, 1.0)


@pytest.mark.parametrize('a_k', [True, False])
@pytest.mark.parametrize('accumulate', [False, True])
def test_in_place_transpose_ragged_n(a_k, accumulate):
    """N = 200 ends 8 columns into B's box [192, 224) of the second n-tile: the box's out-of-range rows come from TMA
    as zeros and are transposed with the rest; D's columns 200..255 keep their fill."""
    M, N, K = 300, 200, 32 * 11 + 5
    fill = 1.0 if accumulate else 7.0
    D, ref = run(M, N, K, a_k=a_k, b_k=False, accumulate=accumulate, width=256, fill=fill)
    check(D, ref, N, fill)
