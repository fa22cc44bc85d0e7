"""Stand-alone GEMM micro-benchmark (CUDA events, L2 flush between iterations).
   python tools/gemm_bench.py [quick]      -> prints one JSON line per shape.

Two groups of cases: operand-major / precision variants at 24000 x 1024 x 1024, and the training step's own GEMMs at
the shapes bench.py's roofline times (R = 23 600 candidate rows, C = 1024): CAR layer 2 forward (bf16x3, bias + tanh),
dgrad (single-pass TF32, leaky derivative from a separate aux, and with the CAR layer-1 gradients formed in its epilogue
instead of a stored dH1) and split-K wgrad (single-pass TF32, both operands
MN-major, split chosen by the library), and the scorer's first layer
(C -> 128) forward / dgrad / wgrad, also with the scorer product (51 candidates per position) as separate kernels
(mul_pred + forward, dgrad + mul_pred_bwd) against folded into the GEMMs (A scaled by PR, product backward epilogue),
and that epilogue with and without the layer-2 bias column sums next to the nar_colsum_add pass they replace (with the
rate of its least HBM traffic, one read of Ec and one write of dEc).
CAR layer 2 also in the form the step runs with the candidate rows stored transposed (H1cT [C, ldr]): the forward with
an MN-major A, and the weight gradient as dW^T = dE^T H1 (A = dE MN-major, B = H1cT K-major, D stored transposed).  Each step case also reports the share of the data-sheet peak of the tensor path it
issues on (bf16 for bf16x3, counting its 3 MMAs per product; TF32 otherwise) and the rate at which TMA fills shared
memory with operand tiles."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from chameleon_recsys_b200 import ops  # noqa: E402

BF16_PEAK, TF32_PEAK = 989.0, 495.0      # dense TFLOP/s, H100 SXM data sheet (700 W)
STEP_R, C = 23600, 1024


def bench(fn, iters=10, flush=None):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def variant_cases(dev):
    """(name, fn, flops, output) at 24000 x 1024 x 1024: every operand major and precision the kernel has."""
    M, N, K = 24000, 1024, 1024
    X = torch.randn(M, K, device=dev)
    W = torch.randn(K, N, device=dev) / 32
    Y = torch.empty(M, N, device=dev)
    dY = torch.randn(M, N, device=dev)
    dW = torch.zeros(K, N, device=dev)
    bias = torch.zeros(N, device=dev)
    X2 = torch.randn(M, K, device=dev)
    Wlo = torch.empty_like(W)
    ops.tf32_lo(W, W.numel(), Wlo)
    Wt = W.t().contiguous()
    Wtlo = torch.empty_like(Wt)
    ops.tf32_lo(Wt, Wt.numel(), Wtlo)
    Wplane = ops.pack_bf16x3(W, K, N)
    f = 2.0 * M * N * K
    return [
        ('fwd  bf16x3 A:K fp32 split in registers, B: packed bf16 plane', lambda: ops.gemm(X, None, Y, M, N, K, a_kmajor=True, b_kmajor=True, ldb=0, bias=bias, act=2, precision=4, b_bf16=Wplane, ld_bf16=Wplane.stride(0)), f, Y),
        ('fwd  3x  A:K  B:K(W^T) +B_lo', lambda: ops.gemm(X, Wt, Y, M, N, K, a_kmajor=True, b_kmajor=True, bias=bias, act=2, precision=3, b_lo=Wtlo), f, Y),
        ('fwd  3x  A:K  B:K(W^T) in-kernel split', lambda: ops.gemm(X, Wt, Y, M, N, K, a_kmajor=True, b_kmajor=True, bias=bias, act=2, precision=3), f, Y),
        ('fwd  1x  A:K  B:K(W^T)', lambda: ops.gemm(X, Wt, Y, M, N, K, a_kmajor=True, b_kmajor=True, bias=bias, act=2, precision=1), f, Y),
        ('fwd  3x  A:K  B:MN +B_lo', lambda: ops.gemm(X, W, Y, M, N, K, a_kmajor=True, b_kmajor=False, bias=bias, act=2, precision=3, b_lo=Wlo), f, Y),
        ('fwd  3x  A:K  B:MN', lambda: ops.gemm(X, W, Y, M, N, K, a_kmajor=True, b_kmajor=False, bias=bias, act=2, precision=3), f, Y),
        ('fwd  1x  A:K  B:MN', lambda: ops.gemm(X, W, Y, M, N, K, a_kmajor=True, b_kmajor=False, bias=bias, act=2, precision=1), f, Y),
        ('dgrad 1x A:K  B:K ', lambda: ops.gemm(dY, W, Y, M, K, N, a_kmajor=True, b_kmajor=True, precision=1), f, Y),
        ('dgrad 1x +dact aux sep', lambda: ops.gemm(dY, W, Y, M, K, N, a_kmajor=True, b_kmajor=True, precision=1, dact=1, aux=X), f, Y),
        ('dgrad 1x +dact in place', lambda: ops.gemm(dY, W, X2, M, K, N, a_kmajor=True, b_kmajor=True, precision=1, dact=1, aux=X2), f, X2),
        ('wgrad 1x A:MN B:MN', lambda: ops.gemm(X, dY, dW, K, N, M, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=0, precision=1), f, dW),
    ]


def step_cases(dev):
    """(name, fn, [M, N, K], output, precision) of the training step's CAR layer-2 and scorer layer-1 GEMMs, operands as
    engine.cu passes them: forward A = activations (K-major) with the bf16x3 plane of W [in, out]; dgrad A = dY, B = W
    read K-major; wgrad A = X and B = dY both MN-major (dY transposed in place in shared memory, two CTAs per SM),
    split-K chosen by the library to fill one wave of the SMs' CTA slots (64 x 4 CTAs for layer 2, 8 x 33 for the
    scorer on 132 SMs), red.add into dW."""
    R = STEP_R
    H1 = torch.randn(R, C, device=dev)
    ldr = (R + 31) // 32 * 32
    H1T = torch.zeros(C, ldr, device=dev)
    H1T[:, :R] = H1.t()
    E = torch.empty(R, C, device=dev)
    dE = torch.randn(R, C, device=dev)
    dH1 = torch.empty(R, C, device=dev)
    W2 = torch.randn(C, C, device=dev) / 32
    b2 = torch.randn(C, device=dev) * 0.1
    dW2 = torch.zeros(C, C, device=dev)
    W2plane = ops.pack_bf16x3(W2, C, C)
    PD = torch.randn(R, C, device=dev)
    Z1 = torch.empty(R, 128, device=dev)
    dZ1 = torch.randn(R, 128, device=dev)
    dPD = torch.empty(R, C, device=dev)
    M0 = torch.randn(C, 128, device=dev) / 32
    c0 = torch.randn(128, device=dev) * 0.1
    dM0 = torch.zeros(C, 128, device=dev)
    M0plane = ops.pack_bf16x3(M0, C, 128)
    # the scorer product PD = Ec * PR[position] at G1's 51 candidates per position: separate kernels vs folded into M1
    n_cand = 51
    L = R // n_cand
    Rp = L * n_cand
    Ec = torch.tanh(H1[:Rp])
    PR = torch.tanh(torch.randn(L, C, device=dev))
    dEc = torch.empty(Rp, C, device=dev)
    dPR = torch.empty(L, C, device=dev)
    db2 = torch.zeros(C, device=dev)

    def mul_pred_fwd():
        ops.mul_pred(Ec, PR, L, n_cand, C, PD)
        ops.gemm(PD, None, Z1, Rp, 128, C, ldb=0, bias=c0, act=ops.ACT_LEAKY, precision=4, b_bf16=M0plane, ld_bf16=M0plane.stride(0))

    # CAR layer 1 per unique id at G1 (462 positions x 51 candidate rows, 1001 table slots): the layer-2 dgrad with its
    # gradients of PP / PC / PI formed in the epilogue (dPI | dPC zeroed first, as the step does)
    Lg, Kg = 462, 50
    Rg, Ug = Lg * (Kg + 1), Kg * 20 + 1
    PP, PC = torch.randn(Lg, C, device=dev), torch.randn(Lg, C, device=dev)
    PI = torch.randn(Ug, C, device=dev)
    pos_idx = torch.arange(Lg, dtype=torch.int32, device=dev)
    neg_uidx = torch.multinomial(1.0 / torch.arange(1, Ug, device=dev, dtype=torch.float64).expand(Lg, Ug - 1), Kg).to(torch.int32)
    DB = torch.empty(Lg + Ug + Lg, C, device=dev)                     # dPP | dPI | dPC, as in the step's DB
    car = dict(pp=PP, pc=PC, pi=PI, pos_idx=pos_idx, neg_uidx=neg_uidx, dpp=DB[:Lg], dpi=DB[Lg:Lg + Ug], dpc=DB[Lg + Ug:], k=Kg)

    def car_dgrad():
        DB[Lg:].zero_()
        ops.gemm(dE[:Rg], W2, None, Rg, C, C, precision=1, dact=ops.ACT_LEAKY, car=car)

    def dgrad_mul_pred_bwd():
        ops.gemm(dZ1, M0, dPD, Rp, C, 128, precision=1)
        ops.mul_pred_bwd(dPD, Ec, PR, L, n_cand, C, dEc, dPR, cand_act=ops.ACT_TANH)
    return [
        ('step L2 fwd   bf16x3 +bias tanh', lambda: ops.gemm(H1, None, E, R, C, C, ldb=0, bias=b2, act=ops.ACT_TANH, precision=4, b_bf16=W2plane, ld_bf16=W2plane.stride(0)), [R, C, C], E, 4),
        ('step L2 fwd   bf16x3 A:MN (H1cT) +bias tanh', lambda: ops.gemm(H1T, None, E, R, C, C, a_kmajor=False, lda=ldr, ldb=0, bias=b2, act=ops.ACT_TANH, precision=4, b_bf16=W2plane, ld_bf16=W2plane.stride(0)), [R, C, C], E, 4),
        ('step L2 dgrad 1x +dact leaky aux sep', lambda: ops.gemm(dE, W2, dH1, R, C, C, precision=1, dact=ops.ACT_LEAKY, aux=H1), [R, C, C], dH1, 1),
        ('step L2 dgrad 1x CAR layer-1 backward epilogue (G1 462 x 51 rows)', car_dgrad, [Rg, C, C], DB, 1),
        ('step L2 wgrad 1x split-K', lambda: ops.gemm(H1, dE, dW2, C, C, R, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=0, precision=1), [C, C, R], dW2, 1),
        ('step L2 wgrad 1x split-K dW^T = dE^T H1cT^T, D transposed', lambda: ops.gemm(dE, H1T, dW2, C, C, R, a_kmajor=False, b_kmajor=True, ldb=ldr, accumulate=True, split_k=0, precision=1, trans_d=True), [C, C, R], dW2, 1),
        ('step M1 fwd   bf16x3 +bias leaky', lambda: ops.gemm(PD, None, Z1, R, 128, C, ldb=0, bias=c0, act=ops.ACT_LEAKY, precision=4, b_bf16=M0plane, ld_bf16=M0plane.stride(0)), [R, 128, C], Z1, 4),
        ('step M1 dgrad 1x', lambda: ops.gemm(dZ1, M0, dPD, R, C, 128, precision=1), [R, C, 128], dPD, 1),
        ('step M1 wgrad 1x split-K', lambda: ops.gemm(PD, dZ1, dM0, C, 128, R, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=0, precision=1), [C, 128, R], dM0, 1),
        ('step M1 mul_pred + fwd bf16x3', mul_pred_fwd, [Rp, 128, C], Z1, 4),
        ('step M1 fwd bf16x3 A scaled by PR', lambda: ops.gemm(Ec, None, Z1, Rp, 128, C, ldb=0, bias=c0, act=ops.ACT_LEAKY, precision=4, b_bf16=M0plane, ld_bf16=M0plane.stride(0), a_scale=PR, a_scale_group=n_cand), [Rp, 128, C], Z1, 4),
        ('step M1 dgrad 1x + mul_pred_bwd', dgrad_mul_pred_bwd, [Rp, C, 128], dEc, 1),
        ('step M1 dgrad 1x product backward epilogue', lambda: ops.gemm(dZ1, M0, dEc, Rp, C, 128, precision=1, dact=ops.ACT_TANH, aux=Ec, pred=PR, d_pred=dPR, pred_group=n_cand), [Rp, C, 128], dEc, 1),
        ('step M1 dgrad 1x product backward epilogue + layer-2 bias column sums', lambda: ops.gemm(dZ1, M0, dEc, Rp, C, 128, precision=1, dact=ops.ACT_TANH, aux=Ec, pred=PR, d_pred=dPR, pred_group=n_cand, d_bias=db2), [Rp, C, 128], dEc, 1),
        ('step colsum_add of dEc (layer-2 bias, candidate rows)', lambda: ops.colsum_add(dEc, Rp, C, C, db2), [Rp, C, 0], db2, 0),
        ('step M1 wgrad 1x split-K A scaled by PR', lambda: ops.gemm(Ec, dZ1, dM0, C, 128, Rp, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=0, precision=1, a_scale=PR, a_scale_group=n_cand), [C, 128, Rp], dM0, 1),
    ]


def step_rates(shape, precision, us):
    """algorithmic TFLOP/s, share of the issuing tensor path's peak, and the shared-memory fill rate: TMA brings one
    32 KB pair of operand tiles (A 128 x 32 fp32 + B 128 x 32 fp32, or B's 128 x 64 bf16 plane tile) per 128 x 128
    output tile and 32-wide k-tile"""
    M, N, K = shape
    flops = 2.0 * M * N * K
    tflops = flops / (us * 1e-6) / 1e12
    share = 3 * tflops / BF16_PEAK if precision == 4 else tflops / TF32_PEAK
    tiles = -(-M // 128) * -(-N // 128) * -(-K // 32)
    return {'tflops': tflops, 'share_of_peak': share, 'peak': 'bf16 %.0f (3 MMAs per product)' % BF16_PEAK if precision == 4
            else 'tf32 %.0f' % TF32_PEAK, 'smem_ingest_GBps': tiles * 32768 / (us * 1e-6) / 1e9}


def main():
    quick = len(sys.argv) > 1 and sys.argv[1] == 'quick'
    iters = 2 if quick else 10
    dev = 'cuda'
    torch.manual_seed(0)
    flush = None if quick else torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    only = os.environ.get('NAR_GEMM_BENCH_ONLY')           # substring filter
    for name, fn, flops, _ in variant_cases(dev):
        if only and only not in name:
            continue
        ms = bench(fn, iters, flush)
        print(json.dumps({'case': name, 'shape': [24000, 1024, 1024], 'us': ms * 1e3, 'tflops': flops / (ms * 1e-3) / 1e12}), flush=True)
    for name, fn, shape, _, prec in step_cases(dev):
        if only and only not in name:
            continue
        ms = bench(fn, iters, flush)
        M, N, K = shape
        if K == 0:                    # not a GEMM: one read of [M, N] fp32
            out = {'case': name, 'shape': [M, N], 'us': ms * 1e3, 'hbm_GBps': M * N * 4 / (ms * 1e-3) / 1e9}
        else:
            out = {'case': name, 'shape': shape, 'us': ms * 1e3, **step_rates(shape, prec, ms * 1e3)}
        if 'product backward' in name:            # the least HBM traffic: Ec read once, dEc written once
            out['ec_dec_GBps'] = 2 * M * N * 4 / (ms * 1e-3) / 1e9
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
