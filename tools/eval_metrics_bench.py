"""Cost of the extended evaluation metrics (NDCG, coverage, ESI-R / ESI-RR, EILD-R / EILD-RR) on one GPU at G1 (batch
256, top_n 10, all seven baselines): Estimator.evaluate wall time per batch with the switch off and on (alternated in the
same process over the same batches, whole evaluate() calls ending in a synchronise, median and spread of the rounds),
the CUDA-event time of the switch's launches for one evaluation batch (the model's and the seven baselines' lists and
the batch's clicks, replayed on the lists evaluate produced), and the oracle's CPU time for the same batch.  Prints one
JSON line with the GPU name and power limit.  Writes nothing.
Usage: python tools/eval_metrics_bench.py [--rounds 3] [--eval-batches 8] [--train-steps 10]"""
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

from chameleon_recsys_b200.baselines import KNN_SUFFIXES, SUFFIXES, BaselineTables  # noqa: E402
from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.eval_metrics import EvalMetrics  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from oracle.eval_metrics_ref import EvalMetricsRef  # noqa: E402
from tools.predict_bench import gpu_info, time_ms  # noqa: E402

ALL7 = [{'recommender': s, 'params': {}} for s in SUFFIXES + KNN_SUFFIXES]
TOP_N = 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--eval-batches', type=int, default=8)
    ap.add_argument('--train-steps', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('eval_metrics_bench needs a CUDA device')
    name, limit = gpu_info()
    res = {'gpu': name, 'power_limit': limit, 'workload': 'g1', 'top_n': TOP_N, 'baselines': len(ALL7)}

    ests = {}
    for on in (False, True):
        pb = make_problem('g1', profile='B')
        warm_state(pb, 3)
        hp = pb.hp.copy(eval_benchmarks=tuple(ALL7), eval_extended_metrics=on, eval_metrics_top_n=TOP_N)
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
    times = {False: [], True: []}
    for _ in range(args.rounds):
        for on in (False, True):
            times[on].append(eval_ms(on)[0])
    for on, key in ((False, 'off'), (True, 'on')):
        res['evaluate_ms_per_batch_' + key] = round(float(np.median(times[on])), 3)
        res['evaluate_ms_spread_' + key] = round(float(max(times[on]) - min(times[on])), 3)
    res['evaluate_ms_rounds'] = {'off': [round(t, 3) for t in times[False]], 'on': [round(t, 3) for t in times[True]]}

    # ---- the switch's launches for one batch: capture the last batch's lists, then replay them
    est, pb, batches = ests[True]
    calls, clicks = [], []
    orig_add, orig_clicks = EvalMetrics.add_lists, EvalMetrics.add_clicks

    def spy_add(self, ids, labels, pop, **kw):
        calls.append((ids.clone(), labels.clone(), pop.clone(), kw))
        return orig_add(self, ids, labels, pop, **kw)

    def spy_clicks(self, ic, ln):
        clicks.append((ic.clone(), ln.clone()))
        return orig_clicks(self, ic, ln)
    EvalMetrics.add_lists, EvalMetrics.add_clicks = spy_add, spy_clicks
    ev = est.evaluate(lambda: iter(batches[-1:]))
    EvalMetrics.add_lists, EvalMetrics.add_clicks = orig_add, orig_clicks
    em = est._eval_spec.evaluation_hooks[0].extended
    em.begin(pb.clicked_items_state.get_recent_clicks_buffer())

    def launches():
        for ids, labels, pop, kw in calls:
            em.add_lists(ids, labels, pop, **kw)
        em.add_clicks(*clicks[0])
    ms, rounds = time_ms(launches, 20)
    res['metrics_launches_ms_per_batch'] = round(ms, 4)
    res['queries_per_batch'] = int(calls[0][0].shape[0])
    res['ndcg_at_n'] = ev['ndcg_at_n']

    # ---- the oracle on the same lists (CPU)
    tab = pb.clicked_items_state.baselines
    ref = EvalMetricsRef(1 + tab.n_rows, TOP_N, pb.content_article_embeddings_matrix, 0.1)
    ref.begin(pb.clicked_items_state.get_recent_clicks_buffer())
    (mids, mcand, pop, mkw), (bids, blab, _, _) = calls
    n_cand = mids.shape[1]
    host = [x.cpu().numpy() for x in (mids, mcand.view(-1, n_cand)[:, 0], pop, bids, blab)]
    pop64 = host[2].astype(np.float64)
    t = time.perf_counter()
    ref.add_lists(0, host[0], host[1], pop64)
    for s in tab.enabled:
        ref.add_lists(1 + BaselineTables.row(s), host[3][BaselineTables.row(s)], host[4], pop64)
    ref.add_clicks(*(x.cpu().numpy() for x in clicks[0]))
    res['cpu_oracle_ms_per_batch'] = round((time.perf_counter() - t) * 1e3, 1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
