"""The scorer product folded into its first Dense layer's GEMMs gives the same bits as the separate product kernels.

Forward: Z1 = leaky(PD M1 + c1) with PD = Ec * PR[row / n_cand] formed as the bf16x3 GEMM loads Ec (a_scale); weight
gradient: dM1 = PD^T dZ1 with the same scale on the MN-major A; dgrad: dEc = (dZ1 M1^T) * PR * tanh'(Ec) and
dPR = sum over the position's rows of (dZ1 M1^T) * Ec in the epilogue of position-aligned M tiles (pred).  Each is
compared with ==, not a tolerance, against nar_mul_pred / nar_mul_pred_bwd around the plain GEMM; then whole training
steps with NAR_FUSED_SCORER_PRODUCT on and off."""
import pytest
import torch

from chameleon_recsys_b200 import ops
from chameleon_recsys_b200._lib import NarError

pytestmark = pytest.mark.gpu

C, H = 1024, 128
N_CAND = [1, 11, 51, 101, 128, 129]


def _positions(n_cand):
    """G1-sized candidate row counts (~24K rows, the last M tile partial)."""
    return max(1, 23600 // n_cand) + 1


def _operands(n_cand, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed * 7919 + n_cand)
    L = _positions(n_cand)
    R = L * n_cand
    Ec = torch.tanh(torch.randn(R, C, device='cuda', generator=g))
    PR = torch.tanh(torch.randn(L, C, device='cuda', generator=g))
    M1 = torch.randn(C, H, device='cuda', generator=g) / 32
    c1 = torch.randn(H, device='cuda', generator=g) * 0.1
    dZ1 = torch.randn(R, H, device='cuda', generator=g) * 1e-3
    return L, R, Ec, PR, M1, c1, dZ1


@pytest.mark.parametrize('n_cand', N_CAND)
def test_scaled_forward_is_bit_identical(n_cand):
    L, R, Ec, PR, M1, c1, _ = _operands(n_cand)
    plane = ops.pack_bf16x3(M1, C, H)
    PD = torch.empty_like(Ec)
    ops.mul_pred(Ec, PR, L, n_cand, C, PD)
    ref = torch.empty(R, H, device='cuda')
    ops.gemm(PD, None, ref, R, H, C, ldb=0, bias=c1, act=ops.ACT_LEAKY, precision=4, b_bf16=plane, ld_bf16=plane.stride(0))
    got = torch.full((R, H), float('nan'), device='cuda')
    ops.gemm(Ec, None, got, R, H, C, ldb=0, bias=c1, act=ops.ACT_LEAKY, precision=4, b_bf16=plane, ld_bf16=plane.stride(0),
             a_scale=PR, a_scale_group=n_cand)
    torch.cuda.synchronize()
    assert torch.equal(got, ref)


@pytest.mark.parametrize('n_cand', N_CAND)
def test_scaled_wgrad_is_bit_identical(n_cand):
    L, R, Ec, PR, _, _, dZ1 = _operands(n_cand)
    PD = torch.empty_like(Ec)
    ops.mul_pred(Ec, PR, L, n_cand, C, PD)
    ref = torch.zeros(C, H, device='cuda')
    ops.gemm(PD, dZ1, ref, C, H, R, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=1, precision=1)
    got = torch.zeros(C, H, device='cuda')
    ops.gemm(Ec, dZ1, got, C, H, R, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=1, precision=1,
             a_scale=PR, a_scale_group=n_cand)
    torch.cuda.synchronize()
    assert torch.equal(got, ref)


@pytest.mark.parametrize('n_cand', N_CAND)
def test_product_backward_epilogue_is_bit_identical(n_cand):
    L, R, Ec, PR, M1, _, dZ1 = _operands(n_cand)
    got_dE = torch.full((R, C), float('nan'), device='cuda')
    got_dPR = torch.full((L, C), float('nan'), device='cuda')

    def fused():
        ops.gemm(dZ1, M1, got_dE, R, C, H, precision=1, dact=ops.ACT_TANH, aux=Ec, pred=PR, d_pred=got_dPR, pred_group=n_cand)
    if n_cand > 128:
        with pytest.raises(NarError):
            fused()
        return
    fused()
    dPD = torch.empty(R, C, device='cuda')
    ops.gemm(dZ1, M1, dPD, R, C, H, precision=1)
    ref_dE = torch.empty(R, C, device='cuda')
    ref_dPR = torch.empty(L, C, device='cuda')
    ops.mul_pred_bwd(dPD, Ec, PR, L, n_cand, C, ref_dE, ref_dPR, cand_act=ops.ACT_TANH)
    torch.cuda.synchronize()
    assert torch.equal(got_dE, ref_dE)
    assert torch.equal(got_dPR, ref_dPR)


def test_invalid_combinations_are_rejected():
    _, _, Ec, PR, M1, c1, dZ1 = _operands(11)
    R = Ec.shape[0]
    plane = ops.pack_bf16x3(M1, C, H)
    Z = torch.empty(R, H, device='cuda')
    dE = torch.empty(R, C, device='cuda')
    dPR = torch.empty_like(PR)
    W = torch.zeros(C, H, device='cuda')
    bad = [
        # a_scale: 3xTF32, single-pass TF32 with a K-major operand, group 0, with pred
        lambda: ops.gemm(Ec, M1.t().contiguous(), Z, R, H, C, precision=3, a_scale=PR, a_scale_group=11),
        lambda: ops.gemm(Ec, M1, Z, R, H, C, b_kmajor=False, precision=1, a_scale=PR, a_scale_group=11),
        lambda: ops.gemm(Ec, dZ1, W, C, H, R, a_kmajor=False, b_kmajor=True, accumulate=True, precision=1, a_scale=PR,
                         a_scale_group=11),
        lambda: ops.gemm(Ec, None, Z, R, H, C, ldb=0, precision=4, b_bf16=plane, ld_bf16=plane.stride(0), a_scale=PR,
                         a_scale_group=0),
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, aux=Ec, a_scale=PR, a_scale_group=11, pred=PR, d_pred=dPR,
                         pred_group=11),
        # pred: bf16x3 / 3xTF32, split-K, accumulate, bias, no aux, rows not whole positions, no d_pred
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=3, aux=Ec, pred=PR, d_pred=dPR, pred_group=11),
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, aux=Ec, pred=PR, d_pred=dPR, pred_group=11, split_k=2,
                         accumulate=True),
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, aux=Ec, pred=PR, d_pred=dPR, pred_group=11, bias=c1),
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, pred=PR, d_pred=dPR, pred_group=11),
        lambda: ops.gemm(dZ1, M1, dE, R - 1, C, H, precision=1, aux=Ec, pred=PR, d_pred=dPR, pred_group=11),
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, aux=Ec, pred=PR, pred_group=11),
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, aux=Ec, pred=PR, d_pred=dPR, pred_group=0),
    ]
    for fn in bad:
        with pytest.raises(NarError, match=r'-1'):
            fn()


def _step(pb, batch, logical, fused, monkeypatch):
    from tools import gpu_step_check as g
    monkeypatch.setenv('NAR_FUSED_SCORER_PRODUCT', '1' if fused else '0')    # read when the engine is created
    eng = g.make_engine(pb)
    eng.set_params(logical)
    st = eng.stage(*batch)
    eng.step(st, train=True, keep=True)
    torch.cuda.synchronize()
    return eng.last['logits'].clone(), eng.loss_dev.clone(), eng.buffer(st, 'dE').clone(), eng.grads.clone()


@pytest.mark.parametrize('name,hp', [('g1', {}), ('tiny', {}), ('adressa', dict(batch_size=128))])
def test_step_matches_unfused(name, hp, monkeypatch):
    """One training step from the same parameters and batch with the switch on and off: logits and dE equal.  The loss
    is an fp32 atomicAdd over the positions, whose order varies from run to run: equal up to that reordering
    (L positions * 2^-24 relative).  The gradient buffer within twice what two runs of the unfused path differ by (the
    split-K red.add order varies from run to run; exactly equal when those two agree)."""
    import numpy as np
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem(name, profile='B', **hp)
    warm_state(pb, 5)
    f, l = pb.input_fn().get_next()
    batch = (f, l, pb.clicked_items_state.get_recent_clicks_buffer().copy(),
             pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32))
    logical = pb.layout.init_logical(3)
    off_a = _step(pb, batch, logical, False, monkeypatch)
    off_b = _step(pb, batch, logical, False, monkeypatch)
    on = _step(pb, batch, logical, True, monkeypatch)
    assert torch.equal(on[0], off_a[0])                                   # logits
    assert torch.equal(on[2], off_a[2])                                   # dE
    L = on[0].shape[0]
    assert float((on[1] - off_a[1]).abs().max()) <= L * 2.0 ** -24 * float(off_a[1].abs().max())
    spread = float((off_a[3] - off_b[3]).abs().max())
    assert float((on[3] - off_a[3]).abs().max()) <= 2 * spread


def test_product_backward_partial_column_tile():
    """C = 1000: the last column tile holds 104 of 128 columns; dEc's columns past C keep their fill."""
    n_cand, L, Cs = 51, 40, 1000
    g = torch.Generator(device='cuda').manual_seed(5)
    R = L * n_cand
    Ec = torch.tanh(torch.randn(R, Cs, device='cuda', generator=g))
    PR = torch.tanh(torch.randn(L, Cs, device='cuda', generator=g))
    M1 = torch.randn(Cs, H, device='cuda', generator=g) / 32
    dZ1 = torch.randn(R, H, device='cuda', generator=g) * 1e-3
    got_dE = torch.full((R, 1024), 7.0, device='cuda')
    got_dPR = torch.full((L, Cs), 7.0, device='cuda')          # row stride of pred and d_pred: one ld_pred
    ops.gemm(dZ1, M1, got_dE, R, Cs, H, precision=1, dact=ops.ACT_TANH, aux=Ec, pred=PR, d_pred=got_dPR, pred_group=n_cand)
    dPD = torch.empty(R, Cs, device='cuda')
    ops.gemm(dZ1, M1, dPD, R, Cs, H, precision=1)
    ref_dE = torch.empty(R, Cs, device='cuda')
    ref_dPR = torch.empty(L, Cs, device='cuda')
    ops.mul_pred_bwd(dPD, Ec, PR, L, n_cand, Cs, ref_dE, ref_dPR, cand_act=ops.ACT_TANH)
    torch.cuda.synchronize()
    assert torch.equal(got_dE[:, :Cs], ref_dE) and torch.equal(got_dPR, ref_dPR)
    assert bool((got_dE[:, Cs:] == 7.0).all())
