"""Recommendation throughput on one GPU: NarEngine.recommend on the G1 workload (46 033 articles, C = 1024), batch 256,
one query per session (positions='last'), recent-clicks state warmed with warm_state.  Candidate sets: the distinct ids
of the recent-clicks buffer, and the full catalog.

Per set it prints one JSON line: ms per batch (CUDA events around whole calls after warm-up, median of the repeats),
sessions/s, candidate pairs/s, model FLOP/s at 2*(C^2 + 128*C + 128*64 + 64*32) per pair, the achieved rate of the CAR
layer-2 GEMM (2*pairs*C^2 over its own time, timed standalone at the chunk shape the call used, bf16x3 like the engine),
the top-n kernel time on a [Q, N] logits matrix, and the GPU name and power limit.  Writes nothing.
Usage: python tools/predict_bench.py [--repeats 5] [--warm-batches 30] [--top-n 10]

--dp: data-parallel prediction (DESIGN.md section 8), one rank per GPU, launched by torchrun over NCCL:
  torchrun --nproc-per-node N tools/predict_bench.py --dp
Per candidate set, rank 0 prints one JSON line: sessions/s of a one-process engine at batch 256 (the other GPUs idle) and
of the data-parallel engine at the global batch 256 * N, the scaling between them, and every rank's GPU name and power
limit.  Host clock around whole calls (each ends with the results on the host), median of the repeats.  Without
torchrun, or with one GPU, only the one-process rate is measured and the scaling is reported as not measured; ranks
sharing a GPU are refused, since their rate says nothing about N GPUs."""
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


def host_ms(fn, repeats, warmup=2):
    """Median wall time of whole calls that end with their results on the host (recommend copies them back)."""
    import time
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), [round(t, 3) for t in ts]


def dp_main(args):
    import torch.distributed as dist
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank, local = int(os.environ.get('RANK', '0')), int(os.environ.get('LOCAL_RANK', '0'))
    if world > torch.cuda.device_count():
        raise SystemExit('--dp runs one rank per GPU: %d ranks, %d GPUs' % (world, torch.cuda.device_count()))
    torch.cuda.set_device(local)
    pg = None
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
        pg = dist.group.WORLD
    per = 256
    pb = make_problem('g1', profile='B', batch_size=per * world)
    warm_state(pb, args.warm_batches)
    logical = pb.layout.init_logical(pb.hp.init_seed)
    feats, _ = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    one_feats = {k: np.asarray(v)[:per] for k, v in feats.items()}       # one GPU's share: the first 256 sessions
    gpus = [None] * world
    if world > 1:
        dist.all_gather_object(gpus, gpu_info())
    else:
        gpus = [gpu_info()]
    eng1 = None
    if rank == 0:
        eng1 = make_engine(pb)
        eng1.set_params(logical)
    engn = make_engine(pb, process_group=pg) if world > 1 else None
    if engn is not None:
        engn.set_params(logical)
    for cands in (None, 'catalog'):
        res = {'candidates': 'buffer' if cands is None else cands, 'batch_per_gpu': per, 'world': world, 'top_n': args.top_n,
               'gpus': [{'name': n, 'power_limit_max_sm_clock': lim} for n, lim in gpus]}
        if rank == 0:
            last = {}

            def one():
                last['out'] = eng1.recommend(one_feats, buf, pop, args.top_n, candidates=cands)
            ms1, all1 = host_ms(one, args.repeats)
            q1 = last['out']['query_session'].size
            res.update(world1_ms=round(ms1, 3), world1_ms_repeats=all1, world1_sessions_per_s=round(q1 / ms1 * 1e3, 1))
        if world > 1:
            dist.barrier()
            last = {}

            def dp():
                last['out'] = engn.recommend(feats, buf, pop, args.top_n, candidates=cands)
            msn, alln = host_ms(dp, args.repeats)
            qn = last['out']['query_session'].size
            res.update(worldN_ms=round(msn, 3), worldN_ms_repeats=alln, worldN_sessions_per_s=round(qn / msn * 1e3, 1))
            if rank == 0:
                res['scaling'] = round(res['worldN_sessions_per_s'] / res['world1_sessions_per_s'], 3)
        else:
            res['scaling'] = 'not measured (one GPU: data-parallel prediction needs one GPU per rank)'
        if rank == 0:
            print(json.dumps(res))
            sys.stdout.flush()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--warm-batches', type=int, default=30)
    ap.add_argument('--top-n', type=int, default=10)
    ap.add_argument('--dp', action='store_true', help='data-parallel mode (torchrun, one rank per GPU)')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('predict_bench needs a CUDA device')
    if args.dp:
        return dp_main(args)
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
