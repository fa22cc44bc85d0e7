"""Cost of the unsampled evaluation (DESIGN.md section 13) on one GPU: G1 workload (46 033 articles, C = 1024, batch 256),
recent-clicks state warmed with warm_state, then 20 EVAL batches.  Each batch runs once without and once with the
unsampled ranking (NarEngine.eval_step, then unsampled_pool + rank_labels as the evaluation hook runs them), the two in
alternating order, each timed with a host clock around work that ends in a device synchronise.  The rank call alone is
also timed with CUDA events.  Prints one JSON line: ms per eval batch off / on (median), the added ms, queries Q and
mean candidates N per batch, (query, candidate) pairs/s of the rank call, and the GPU name, power limit and max SM clock
read in the same call.  Writes nothing.
Usage: python tools/unsampled_eval_bench.py [--batches 20] [--warm-batches 30]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from tools.gpu_step_check import make_engine  # noqa: E402
from tools.predict_bench import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, default=20)
    ap.add_argument('--warm-batches', type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('unsampled_eval_bench needs a CUDA device')
    name, limit = gpu_info()
    pb = make_problem('g1', profile='B')
    warm_state(pb, args.warm_batches)
    # the EVAL graph's engine: eval sampling hparams, no dropout (nar_trainer_gcom.py:237-245)
    hp = pb.hp = pb.hp.copy(train_total_negative_samples=pb.hp.eval_total_negative_samples,
                            train_negative_samples_from_buffer=pb.hp.eval_negative_samples_from_buffer, dropout_keep_prob=1.0)
    eng = make_engine(pb)
    eng.set_params(pb.layout.init_logical(hp.init_seed))
    top_n = hp.eval_metrics_top_n
    it = pb.input_fn()
    batches = [it.get_next() for _ in range(args.batches)]
    state = pb.clicked_items_state
    hist = torch.zeros(top_n + 2, dtype=torch.int64, device=eng.dev)

    def run(f, l, buf, pop, on, ev=None):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = eng.eval_step(f, l, buf, pop, top_n=top_n)
        if on:
            pool = eng.unsampled_pool(f['item_clicked'], l['label_last_item'], buf)
            ev[0].record()
            eng.rank_labels(out['stage'], pool, top_n, hist=hist)
            ev[1].record()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out['stage']['L'], (pool.size if on else 0)

    # warm-up: every shape of the timed window (workspaces, pinned slots, the rank workspace)
    f, l = batches[0]
    for on in (False, True):
        run(f, l, state.get_recent_clicks_buffer(), state.get_articles_recent_pop_norm(), on,
            (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
    ms_off, ms_on, ms_rank, Qs, Ns = [], [], [], [], []
    for i, (f, l) in enumerate(batches):
        buf, pop = state.get_recent_clicks_buffer().copy(), state.get_articles_recent_pop_norm().copy()
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        for on in ((False, True) if i % 2 == 0 else (True, False)):
            ms, Q, N = run(f, l, buf, pop, on, ev)
            (ms_on if on else ms_off).append(ms)
            if on:
                ms_rank.append(ev[0].elapsed_time(ev[1]))
                Qs.append(Q)
                Ns.append(N)
        state.update_from_batch(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
    pairs = float(np.sum(np.asarray(Qs, np.float64) * np.asarray(Ns, np.float64)))
    print(json.dumps({
        'metric': 'unsampled_eval_ms_per_batch', 'workload': 'g1', 'batches': args.batches,
        'ms_off': round(float(np.median(ms_off)), 3), 'ms_on': round(float(np.median(ms_on)), 3),
        'ms_added': round(float(np.median(np.asarray(ms_on) - np.asarray(ms_off))), 3),
        'ms_rank_call': round(float(np.median(ms_rank)), 3),
        'Q_mean': round(float(np.mean(Qs)), 1), 'N_mean': round(float(np.mean(Ns)), 1),
        'pairs_per_s': round(pairs / (float(np.sum(ms_rank)) * 1e-3), 1),
        'gpu': name, 'power_limit_and_max_sm_clock': limit}))


if __name__ == '__main__':
    main()
