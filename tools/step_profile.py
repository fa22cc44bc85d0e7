"""Per-kernel profile of the device-resident training step that bench.py times (`value`): G1 workload, batch 256, inputs
staged in HBM, eng.step + eng.apply_gradients on the main stream and eng.prepare of the next batch on the side stream,
at most two steps queued ahead of the device.  The steps run under torch.profiler with CUDA activities; kernel times
come from the trace, grouped by kernel name, and for gemm_kernel by template arguments and grid.

Kernels of the engine's auxiliary and side streams run concurrently with the main stream, so the per-kernel sum is
larger than the step's wall time.

Writes OUT_DIR/step_profile.json (GPU name, power limit and max SM clock of the same run included) and prints a
table.  Usage: python tools/step_profile.py OUT_DIR [--steps 20] [--warmup 5]"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import make_batches  # noqa: E402
from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from tools.predict_bench import gpu_info  # noqa: E402


def kernel_key(name: str, grid) -> str:
    """'void nar::gemm::gemm_kernel<false, true, 0>(CUtensorMap_st, ...)' -> 'gemm_kernel<false, true, 0> grid [x, y, z]';
    any other kernel -> its name without namespace, template arguments and parameter list."""
    m = re.search(r'gemm_kernel<[^>]*>', name)
    if m:
        return '%s grid %s' % (m.group(0), list(grid) if grid else '?')
    base = re.sub(r'\(.*$', '', name.replace('(anonymous namespace)::', ''))
    base = re.sub(r'<.*$', '', base)
    return base.split('::')[-1].replace('void ', '').strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'the step profile needs a GPU'
    torch.cuda.set_device(0)

    # the problem bench.py run_ours builds: G1, profile B, G1 session lengths, 100 batches of state warm-up
    pb = make_problem('g1', profile='B', session_len='g1')
    warm_state(pb, 100)
    n_total = args.warmup + args.steps
    batches = make_batches(pb, n_total, pb.hp.batch_size)
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, pb.hp, pb.clicked_items_state, device=0)
    eng = est._ensure_spec(None, None).model.engine
    staged = [eng.stage(f, l, buf, pop, slot='prof%d' % i) for i, (f, l, buf, pop) in enumerate(batches)]
    torch.cuda.synchronize()
    side = eng.side_stream()
    done = {}

    def step(i):
        if (i - 2) in done:
            done.pop(i - 2).synchronize()
        eng.step(staged[i], train=True)
        eng.apply_gradients(staged[i])
        if i + 1 < len(staged):
            eng.prepare(staged[i + 1], eng.global_step + 1, stream=side)
        ev = torch.cuda.Event()
        ev.record()
        done[i] = ev

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        e0.record()
        for i in range(args.warmup, n_total):
            step(i)
        e1.record()
        torch.cuda.synchronize()
    ms_per_step = e0.elapsed_time(e1) / args.steps
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, 'trace.json')
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    groups = {}
    for ev in trace.get('traceEvents', []):
        if ev.get('cat') != 'kernel':
            continue
        key = kernel_key(ev['name'], ev.get('args', {}).get('grid'))
        g = groups.setdefault(key, [0, 0.0])
        g[0] += 1
        g[1] += float(ev.get('dur', 0.0))
    total = sum(g[1] for g in groups.values())
    rows = sorted(({'kernel': k, 'calls_per_step': n / args.steps, 'us_per_step': us / args.steps, 'share': us / total}
                   for k, (n, us) in groups.items()), key=lambda r: -r['us_per_step'])
    gemm = {}                                   # the step's row counts vary, and with them the grids: totals per template
    for r in rows:
        if r['kernel'].startswith('gemm_kernel<'):
            k = r['kernel'].split(' grid')[0]
            gemm[k] = gemm.get(k, 0.0) + r['us_per_step']
    name, limit = gpu_info()
    out = {'gpu': name, 'power_limit_max_sm_clock': limit, 'workload': 'g1, batch %d, K=%d, C=%d' % (
               pb.hp.batch_size, pb.hp.train_total_negative_samples, pb.hp.CAR_embedding_size),
           'steps': args.steps, 'warmup': args.warmup, 'ms_per_step_under_profiler': ms_per_step,
           'kernel_us_per_step_sum_all_streams': total / args.steps,
           'interactions_per_step': sum(st['L_global'] for st in staged[args.warmup:]) / args.steps,
           'gemm_us_per_step_by_template': dict(sorted(gemm.items(), key=lambda kv: -kv[1])), 'kernels': rows}
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, 'step_profile.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print('%s | %s | %.3f ms/step under the profiler, kernel sum %.1f us/step' % (name, limit, ms_per_step, total / args.steps))
    for k, us in out['gemm_us_per_step_by_template'].items():
        print('%9.1f us  %s, all grids' % (us, k))
    for r in rows:
        print('%9.1f us %5.1f%% %6.1f calls  %s' % (r['us_per_step'], 100 * r['share'], r['calls_per_step'], r['kernel']))


if __name__ == '__main__':
    main()
