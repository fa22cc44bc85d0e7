"""The scorer product-backward dgrad's epilogue (nar_gemm_epilogue.pred) with its optional column sums (d_bias).

dEc and dPR are compared with ==, not a tolerance, against nar_mul_pred_bwd around the plain TF32 dgrad, at position
lengths that fill a chunk of the epilogue with several positions (1, 11, 51) or split one position over several chunks
(101, 128), with full, partial (1000) and not 4-aligned (998) last column tiles, and last M tiles holding fewer
positions than the others.  The column sums against fp64 within the bar of test_colsum_add; then one G1 training step,
whose layer-2 bias gradient the epilogue now sums, against the same step through nar_mul_pred_bwd and nar_colsum_add."""
import math

import numpy as np
import pytest
import torch

from chameleon_recsys_b200 import ops
from chameleon_recsys_b200._lib import NarError

pytestmark = pytest.mark.gpu

H = 128
U = 2.0 ** -24


def _colsum_bar(rows, mag):
    """test_colsum_add's bound on an fp32 column sum of `rows` terms onto a prefill: (ceil(rows/64) + 17) u mag.  The
    epilogue's sums are shallower: at most 16 terms per thread, a 3-level tree over the warps and one red.add per M tile
    of at least 65 rows (one position when n_cand > 64)."""
    return (math.ceil(rows / 64) + 17) * U * mag


@pytest.mark.parametrize('N', [1024, 1000, 998])
@pytest.mark.parametrize('n_cand', [1, 11, 51, 101, 128])
def test_wide_epilogue_matches_mul_pred_bwd(n_cand, N):
    P = 128 // n_cand                                            # positions per M tile
    L = 23600 // n_cand + 1
    if P > 1:
        assert L % P != 0                                        # the last M tile holds fewer positions
    R, ld = L * n_cand, 1000 if N == 998 else N                  # N = 998: rows of 1000, the last column group partial
    g = torch.Generator(device='cuda').manual_seed(31 * n_cand + N)
    Ec = torch.tanh(torch.randn(R, ld, device='cuda', generator=g))
    PR = torch.tanh(torch.randn(L, ld, device='cuda', generator=g))
    M1 = torch.randn(ld, H, device='cuda', generator=g) / 32
    dZ1 = torch.randn(R, H, device='cuda', generator=g) * 1e-3
    pre = torch.rand(N + 4, device='cuda', generator=g) * 4 - 2
    got_dE = torch.full((R, 1024), 7.0, device='cuda')
    got_dPR = torch.full((L, ld), 7.0, device='cuda')
    got_b = pre.clone()
    ops.gemm(dZ1, M1, got_dE, R, N, H, precision=1, dact=ops.ACT_TANH, aux=Ec[:, :N], pred=PR[:, :N], d_pred=got_dPR,
             pred_group=n_cand, d_bias=got_b)
    dPD = torch.empty(R, ld, device='cuda')
    ops.gemm(dZ1, M1, dPD, R, ld, H, precision=1)
    ref_dE = torch.empty(R, ld, device='cuda')
    ref_dPR = torch.empty(L, ld, device='cuda')
    ops.mul_pred_bwd(dPD, Ec, PR, L, n_cand, ld, ref_dE, ref_dPR, cand_act=ops.ACT_TANH)
    cs = pre.clone()
    ops.colsum_add(got_dE, R, N, 1024, cs)
    torch.cuda.synchronize()
    assert torch.equal(got_dE[:, :N], ref_dE[:, :N]) and torch.equal(got_dPR[:, :N], ref_dPR[:, :N])
    assert bool((got_dE[:, N:] == 7.0).all()) and bool((got_dPR[:, N:] == 7.0).all())
    assert torch.equal(got_b[N:], pre[N:])                       # columns past N untouched
    d64 = ref_dE[:, :N].double()
    mag = pre[:N].double().abs() + d64.abs().sum(0)
    bar = _colsum_bar(R, mag)
    err = (got_b[:N].double() - (pre[:N].double() + d64.sum(0))).abs()
    assert bool((err <= bar).all()), float((err / bar).max())
    assert bool(((got_b[:N] - cs[:N]).double().abs() <= 2 * bar).all())


def test_column_sum_rejected_outside_product_backward():
    g = torch.Generator(device='cuda').manual_seed(3)
    R, C = 11 * 40, 256
    Ec = torch.tanh(torch.randn(R, C, device='cuda', generator=g))
    PR = torch.tanh(torch.randn(40, C, device='cuda', generator=g))
    M1 = torch.randn(C, H, device='cuda', generator=g) / 32
    dZ1 = torch.randn(R, H, device='cuda', generator=g)
    plane = ops.pack_bf16x3(M1, C, H)
    dE, Z, W = torch.empty(R, C, device='cuda'), torch.empty(R, H, device='cuda'), torch.zeros(C, H, device='cuda')
    W2, EcT = torch.randn(C, C, device='cuda', generator=g) / 32, Ec.t().contiguous()
    PP, PI = torch.randn(40, C, device='cuda', generator=g), torch.randn(101, C, device='cuda', generator=g)
    car = dict(pp=PP, pc=PP.clone(), pi=PI, pos_idx=torch.arange(40, dtype=torch.int32, device='cuda'),
               neg_uidx=torch.randint(0, 101, (40, 10), dtype=torch.int32, device='cuda', generator=g),
               dpp=torch.zeros_like(PP), dpc=torch.zeros_like(PP), dpi=torch.zeros_like(PI), k=10)
    b = torch.zeros(C, device='cuda')
    bad = [
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, d_bias=b),                                   # plain dgrad
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=1, dact=ops.ACT_TANH, aux=Ec, d_bias=b),          # + dact
        lambda: ops.gemm(dZ1, M1, dE, R, C, H, precision=3, dact=ops.ACT_TANH, aux=Ec, d_bias=b),          # 3xTF32
        lambda: ops.gemm(Ec, None, Z, R, H, C, ldb=0, precision=4, b_bf16=plane, ld_bf16=plane.stride(0),
                         a_scale=PR, a_scale_group=11, d_bias=b),                                          # scaled forward
        lambda: ops.gemm(Ec, dZ1, W, C, H, R, a_kmajor=False, b_kmajor=False, accumulate=True, precision=1,
                         a_scale=PR, a_scale_group=11, d_bias=b),                                          # scaled wgrad
        lambda: ops.gemm(dZ1, EcT, W, H, C, R, a_kmajor=False, b_kmajor=True, accumulate=True, precision=1,
                         trans_d=True, d_bias=b),                                                          # D transposed
        lambda: ops.gemm(dE, W2, None, R, C, C, precision=1, dact=ops.ACT_LEAKY, car=car, d_bias=b),      # CAR backward
    ]
    for fn in bad:
        with pytest.raises(NarError, match=r'-1'):
            fn()
    torch.cuda.synchronize()
    assert bool((b == 0).all())


def _step(pb, batch, logical, fused, monkeypatch):
    from tools import gpu_step_check as gsc
    monkeypatch.setenv('NAR_FUSED_SCORER_PRODUCT', '1' if fused else '0')    # read when the engine is created
    eng = gsc.make_engine(pb)
    eng.set_params(logical)
    st = eng.stage(*batch)
    eng.step(st, train=True, keep=True)
    torch.cuda.synchronize()
    return eng.buffer(st, 'dE').clone(), eng.buffer(st, 'dPR').clone(), eng.grads.clone()


def test_g1_step_bias_sum_in_epilogue(monkeypatch):
    """One G1 training step from identical parameters and batch: the epilogue's path (b2 summed in the dgrad, no
    nar_colsum_add over the candidate rows) against nar_mul_pred_bwd + nar_colsum_add (switch 0, run three times).  dE
    (all rows) and dPR are equal; b2 is within the fp32 summation bar of the fp64 column sums of dE, the clicked rows'
    sum included; every other gradient block differs from the reference by at most twice what the reference runs differ
    by among themselves (split-K red.add order varies from run to run; blocks that do not vary must be equal)."""
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('g1', profile='B')
    warm_state(pb, 5)
    f, lab = pb.input_fn().get_next()
    batch = (f, lab, pb.clicked_items_state.get_recent_clicks_buffer().copy(),
             pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32))
    logical = pb.layout.init_logical(3)
    refs = [_step(pb, batch, logical, False, monkeypatch) for _ in range(3)]
    ref_a = refs[0]
    on = _step(pb, batch, logical, True, monkeypatch)
    assert torch.equal(on[0], ref_a[0])                          # dE: clicked and candidate rows
    assert torch.equal(on[1], ref_a[1])                          # dPR
    dE = on[0].double()
    b2 = pb.layout.by_key['b2']
    C = b2.ld
    got = on[2][b2.offset:b2.offset + C].double()
    want, mag = dE.sum(0), dE.abs().sum(0)
    bar = _colsum_bar(dE.shape[0], mag)
    assert bool(((got - want).abs() <= bar).all())
    assert bool(((got - ref_a[2][b2.offset:b2.offset + C].double()).abs() <= 2 * bar).all())
    for t in pb.layout.tensors:
        if t.key == 'b2' or t.into is not None:                  # `into`: storage of another block
            continue
        s = slice(t.offset, t.offset + t.size)
        spread = max(float((x[2][s] - y[2][s]).abs().max()) for i, x in enumerate(refs) for y in refs[i + 1:])
        diff = float((on[2][s] - ref_a[2][s]).abs().max())
        assert diff <= 2 * spread, (t.key, diff, spread)
