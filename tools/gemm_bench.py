"""Stand-alone GEMM / gather micro-benchmark (CUDA events, L2 flush between iterations).
   python tools/gemm_bench.py [quick]      -> prints one JSON line per shape."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from chameleon_recsys_b200 import ops  # noqa: E402


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


def main():
    quick = len(sys.argv) > 1 and sys.argv[1] == 'quick'
    iters = 2 if quick else 10
    dev = 'cuda'
    flush = None if quick else torch.empty(256 << 20, dtype=torch.uint8, device=dev)
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
    only = os.environ.get('NAR_GEMM_BENCH_ONLY')           # substring filter
    cases = [
        ('fwd  bf16x3 A:K fp32 split in registers, B: packed bf16 plane', lambda: ops.gemm(X, None, Y, M, N, K, a_kmajor=True, b_kmajor=True, ldb=0, bias=bias, act=2, precision=4, b_bf16=Wplane, ld_bf16=Wplane.stride(0)), 2.0 * M * N * K),
        ('fwd  3x  A:K  B:K(W^T) +B_lo', lambda: ops.gemm(X, Wt, Y, M, N, K, a_kmajor=True, b_kmajor=True, bias=bias, act=2, precision=3, b_lo=Wtlo), 2.0 * M * N * K),
        ('fwd  3x  A:K  B:K(W^T) in-kernel split', lambda: ops.gemm(X, Wt, Y, M, N, K, a_kmajor=True, b_kmajor=True, bias=bias, act=2, precision=3), 2.0 * M * N * K),
        ('fwd  1x  A:K  B:K(W^T)', lambda: ops.gemm(X, Wt, Y, M, N, K, a_kmajor=True, b_kmajor=True, bias=bias, act=2, precision=1), 2.0 * M * N * K),
        ('fwd  3x  A:K  B:MN +B_lo', lambda: ops.gemm(X, W, Y, M, N, K, a_kmajor=True, b_kmajor=False, bias=bias, act=2, precision=3, b_lo=Wlo), 2.0 * M * N * K),
        ('fwd  3x  A:K  B:MN', lambda: ops.gemm(X, W, Y, M, N, K, a_kmajor=True, b_kmajor=False, bias=bias, act=2, precision=3), 2.0 * M * N * K),
        ('fwd  1x  A:K  B:MN', lambda: ops.gemm(X, W, Y, M, N, K, a_kmajor=True, b_kmajor=False, bias=bias, act=2, precision=1), 2.0 * M * N * K),
        ('dgrad 1x A:K  B:K ', lambda: ops.gemm(dY, W, Y, M, K, N, a_kmajor=True, b_kmajor=True, precision=1), 2.0 * M * N * K),
        ('dgrad 1x +dact aux sep', lambda: ops.gemm(dY, W, Y, M, K, N, a_kmajor=True, b_kmajor=True, precision=1, dact=1, aux=X), 2.0 * M * N * K),
        ('dgrad 1x +dact in place', lambda: ops.gemm(dY, W, X2, M, K, N, a_kmajor=True, b_kmajor=True, precision=1, dact=1, aux=X2), 2.0 * M * N * K),
        ('wgrad 1x A:MN B:MN', lambda: ops.gemm(X, dY, dW, K, N, M, a_kmajor=False, b_kmajor=False, accumulate=True, split_k=0, precision=1), 2.0 * M * N * K),
    ]
    for name, fn, flops in cases:
        if only and only not in name:
            continue
        ms = bench(fn, iters, flush)
        print(json.dumps({'case': name, 'shape': [M, N, K], 'us': ms * 1e3, 'tflops': flops / (ms * 1e-3) / 1e12}), flush=True)


if __name__ == '__main__':
    main()
