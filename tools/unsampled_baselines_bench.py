"""Cost of the baselines' unsampled evaluation (DESIGN.md section 14) on one GPU at G1 (46 033 articles, batch 256, all
seven baselines with the reference parameters): two estimators from the same seeds, the recent-clicks state warmed with
warm_state and every baseline trained on --train-steps batches (a full kNN ring after 12), one with
eval_unsampled_benchmarks off and one with it on.  Estimator.evaluate over the same --eval-batches batches, the two
alternated for --rounds rounds, each call ending in a synchronise: ms per eval batch off / on (median and spread) and the
added ms.  Then one profiled evaluate (torch.profiler, CUDA activity, a run of its own) gives each unsampled kernel's
device time per eval batch: nar::bl::rank_unsampled_kernel (the five table baselines) and nar::sknn::rank_unsampled_kernel
(one launch per kNN baseline).  Also the queries per batch, the competitors per query, each baseline's unsampled hit
rate, and the GPU name, power limit and max SM clock read in the same call.  Prints one JSON line; writes nothing.
Usage: python tools/unsampled_baselines_bench.py [--rounds 3] [--eval-batches 20] [--train-steps 12]"""
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

from chameleon_recsys_b200.baselines import KNN_SUFFIXES, SUFFIXES  # noqa: E402
from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from tools.predict_bench import gpu_info  # noqa: E402

ALL7 = [{'recommender': s, 'params': {}} for s in SUFFIXES + KNN_SUFFIXES]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--eval-batches', type=int, default=20)
    ap.add_argument('--train-steps', type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('unsampled_baselines_bench needs a CUDA device')
    name, limit = gpu_info()
    res = {'metric': 'unsampled_baselines_ms_per_eval_batch', 'workload': 'g1', 'baselines': len(ALL7),
           'eval_batches': args.eval_batches, 'gpu': name, 'power_limit_and_max_sm_clock': limit}
    ests = {}
    for on in (False, True):
        pb = make_problem('g1', profile='B')
        warm_state(pb, 3)
        hp = pb.hp.copy(eval_benchmarks=tuple(ALL7), eval_unsampled_benchmarks=on)
        est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                              pb.session_features_config, hp, pb.clicked_items_state, device=0)
        it = pb.input_fn()
        est.train(lambda: iter([it.get_next() for _ in range(args.train_steps)]))
        batches = [it.get_next() for _ in range(args.eval_batches)]
        est.evaluate(lambda b=batches: iter(b))                          # builds the evaluation graph, warms up
        ests[on] = (est, pb, batches)

    def eval_ms(on):
        est, _, batches = ests[on]
        torch.cuda.synchronize()
        t = time.perf_counter()
        ev = est.evaluate(lambda: iter(batches))
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3 / len(batches), ev
    times, last = {False: [], True: []}, {}
    for r in range(args.rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            ms, last[on] = eval_ms(on)
            times[on].append(ms)
    for on, key in ((False, 'off'), (True, 'on')):
        res['ms_' + key] = round(float(np.median(times[on])), 3)
        res['ms_spread_' + key] = round(float(max(times[on]) - min(times[on])), 3)
    res['ms_added'] = round(res['ms_on'] - res['ms_off'], 3)
    res['rounds'] = {'off': [round(t, 3) for t in times[False]], 'on': [round(t, 3) for t in times[True]]}

    est, pb, batches = ests[True]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        est.evaluate(lambda: iter(batches))
        torch.cuda.synchronize()
    n = len(batches)
    for key, tag in (('bl', 'nar::bl::rank_unsampled_kernel'), ('sknn', 'nar::sknn::rank_unsampled_kernel')):
        evs = [e for e in prof.key_averages() if tag in e.key]
        res['%s_rank_unsampled_ms_per_batch' % key] = round(sum(e.device_time_total for e in evs) / n / 1e3, 4)
        res['%s_rank_unsampled_launches_per_batch' % key] = sum(e.count for e in evs) / n
    res['Q_mean'] = round(float(np.mean([np.count_nonzero(l['label_next_item']) for _, l in batches])), 1)
    res['competitors_per_query'] = round(last[True]['unsampled_candidates_per_query'], 1)
    res['unsampled_hitrate_at_n'] = {s['recommender']: round(last[True]['unsampled_hitrate_at_n_' + s['recommender']], 4)
                                     for s in ALL7}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
