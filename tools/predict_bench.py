"""Recommendation throughput on one GPU: NarEngine.recommend on the G1 workload (46 033 articles, C = 1024), batch 256,
one query per session (positions='last'), recent-clicks state warmed with warm_state.  Candidate sets: the distinct ids
of the recent-clicks buffer, and the full catalog.

Per set it prints one JSON line: ms per batch (CUDA events around whole calls after warm-up, median of the repeats),
sessions/s, candidate pairs/s, model FLOP/s at 2*(C^2 + 128*C + 128*64 + 64*32) per pair, the achieved rate of the CAR
layer-2 GEMM (2*pairs*C^2 over its own time, timed standalone at the chunk shape the call used, bf16x3 like the engine),
the top-n kernel time on a [Q, N] logits matrix, and the GPU name and power limit.  Writes nothing.
Usage: python tools/predict_bench.py [--repeats 5] [--warm-batches 30] [--top-n 10]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chameleon_recsys_b200 import ops  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from tools.gpu_step_check import make_engine  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        limit = r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        limit = 'unavailable (%s)' % e
    return name, limit


def time_ms(fn, repeats, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), [round(t, 3) for t in ts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--warm-batches', type=int, default=30)
    ap.add_argument('--top-n', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('predict_bench needs a CUDA device')
    name, limit = gpu_info()
    pb = make_problem('g1', profile='B')
    warm_state(pb, args.warm_batches)
    eng = make_engine(pb)
    eng.set_params(pb.layout.init_logical(pb.hp.init_seed))
    feats, _ = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    Cd = eng.C
    flop_pair = 2 * (Cd * Cd + 128 * Cd + 128 * 64 + 64 * 32)
    W2 = eng.view('W2')
    plane = ops.pack_bf16x3(W2, Cd, Cd)
    for cands in (None, 'catalog'):
        last = {}

        def call():
            last['out'] = eng.recommend(feats, buf, pop, args.top_n, candidates=cands)
        ms, all_ms = time_ms(call, args.repeats)
        out = last['out']
        Q, N = out['predicted_item_ids'].shape[0], out['candidates'].size
        pairs = Q * N
        # layer-2 GEMM at the call's chunk shape (one chunk = q_block x n_block pairs), standalone
        P = out['q_block'] * out['n_block']
        A = torch.randn(P, Cd, device='cuda').tanh_()
        D = torch.empty(P, Cd, device='cuda')
        g_ms, _ = time_ms(lambda: ops.gemm(A, None, D, P, Cd, Cd, bias=eng.view('b2').view(-1), act=ops.ACT_TANH, precision=4,
                                           b_bf16=plane, ld_bf16=plane.shape[1]), args.repeats)
        del A, D
        # top-n over [Q, N] logits with the sessions' clicks excluded
        lg = torch.randn(Q, N, device='cuda')
        cid = torch.from_numpy(out['candidates']).cuda()
        ic = torch.from_numpy(np.ascontiguousarray(feats['item_clicked'], dtype=np.int64)).cuda()
        T = ic.shape[1]
        qp = torch.from_numpy((out['query_session'] * T + out['query_position']).astype(np.int32)).cuda()
        ids = torch.empty(Q, args.top_n, dtype=torch.int64, device='cuda')
        sc = torch.empty(Q, args.top_n, device='cuda')
        pr = torch.empty(Q, args.top_n, device='cuda')
        t_ms, _ = time_ms(lambda: ops.topn_candidates(lg, cid, Q, N, args.top_n, ids, sc, pr, ic, qp, T), args.repeats * 4)
        del lg
        print(json.dumps({
            'candidates': 'buffer' if cands is None else cands, 'Q': Q, 'N': N, 'top_n': args.top_n,
            'q_block': out['q_block'], 'n_block': out['n_block'], 'fwd_precision': eng.fwd_prec,
            'ms_per_batch': round(ms, 3), 'ms_repeats': all_ms, 'sessions_per_s': round(Q / ms * 1e3, 1),
            'pairs_per_s': round(pairs / ms * 1e3, 1), 'model_tflops': round(pairs * flop_pair / ms / 1e9, 1),
            'car2_gemm_ms_per_chunk': round(g_ms, 3), 'car2_gemm_tflops': round(2.0 * P * Cd * Cd / g_ms / 1e9, 1),
            'topn_ms': round(t_ms, 3), 'gpu': name, 'power_limit_max_sm_clock': limit}))
        sys.stdout.flush()


if __name__ == '__main__':
    main()
