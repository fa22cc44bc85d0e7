"""Cost of the baseline recommenders on one GPU at G1 (batch 256): Estimator.train step time with all five baselines
off and on (alternated in the same process, wall time per step over whole train() calls, median of the rounds), the
pair-table update kernel (CUDA events), the scoring + ranking + metrics launch of one evaluation batch (CUDA events),
the table entries after the warm-up, and the numpy oracle's time for the same evaluation batch (CPU, wall time).
Prints one JSON line with the GPU name and power limit.  Writes nothing.
Usage: python tools/baselines_bench.py [--rounds 3] [--steps 20] [--warm-batches 10]"""
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

from chameleon_recsys_b200.baselines import SUFFIXES, BaselineTables  # noqa: E402
from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from oracle.baselines_ref import BaselinesRef  # noqa: E402
from tools.predict_bench import gpu_info, time_ms  # noqa: E402

ALL = [{'recommender': s, 'params': {}} for s in SUFFIXES]


def train_ms(est, pb, steps):
    est.train(pb.input_fn, steps=steps)
    torch.cuda.synchronize()
    t = time.perf_counter()
    est.train(pb.input_fn, steps=steps)
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warm-batches', type=int, default=10)
    args = ap.parse_args()
    res = {'gpu': gpu_info()[0], 'power_limit': gpu_info()[1], 'workload': 'g1'}

    # ---- training step, baselines off / on, alternated
    ests = {}
    for on in (False, True):
        pb = make_problem('g1', profile='B')
        warm_state(pb, 3)
        hp = pb.hp.copy(eval_benchmarks=tuple(ALL) if on else ())
        ests[on] = (build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata,
                                    pb.articles_features_config, pb.session_features_config, hp, pb.clicked_items_state,
                                    device=0), pb)
    times = {False: [], True: []}
    for _ in range(args.rounds):
        for on in (False, True):
            times[on].append(train_ms(ests[on][0], ests[on][1], args.steps))
    res['train_ms_per_step_off'] = round(float(np.median(times[False])), 3)
    res['train_ms_per_step_on'] = round(float(np.median(times[True])), 3)
    res['train_ms_rounds'] = {'off': [round(t, 3) for t in times[False]], 'on': [round(t, 3) for t in times[True]]}
    del ests
    torch.cuda.empty_cache()

    # ---- kernels on G1 batches
    pb = make_problem('g1', profile='B')
    V, K, top_n = pb.wl.num_items, pb.hp.eval_total_negative_samples, pb.hp.eval_metrics_top_n
    acr = np.asarray(pb.content_article_embeddings_matrix, dtype=np.float32)
    tab = BaselineTables(ALL, V, acr=torch.from_numpy(acr).cuda(), acr_dim=acr.shape[1])
    ref = BaselinesRef(V, acr=acr)
    it = pb.input_fn()
    batches = [it.get_next() for _ in range(args.warm_batches + 1)]
    all_items = [np.concatenate([f['item_clicked'], l['label_last_item'].reshape(-1, 1)], axis=1) for f, l in batches]
    for ai in all_items[:-1]:
        tab.update(torch.from_numpy(ai).cuda())
        ref.update(ai)
    torch.cuda.synchronize()
    res['table_entries'] = int(tab.count.item())
    res['table_capacity'] = tab.cap
    last = torch.from_numpy(all_items[-1]).cuda()

    def upd():
        tab.snapshot()
        tab.update(last)
        tab.restore()
    upd_ms, _ = time_ms(upd, 5)
    snap_ms, _ = time_ms(lambda: (tab.snapshot(), tab.restore()), 5)
    res['update_ms'] = round(upd_ms - snap_ms, 4)
    f, l = batches[-1]
    rs = np.random.RandomState(0)
    neg = rs.randint(1, V, size=f['item_clicked'].shape + (K,)).astype(np.int64)
    buf = pb.clicked_items_state.get_recent_clicks_buffer()
    pop = pb.clicked_items_state.get_articles_pop()
    ic, ln, ng = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (f['item_clicked'], l['label_next_item'], neg))
    metrics = torch.zeros(5, 3, dtype=torch.float64, device='cuda')
    bufd, popd = torch.from_numpy(np.ascontiguousarray(buf)).cuda(), torch.from_numpy(np.ascontiguousarray(pop)).cuda()
    res['score_ms_per_batch'] = round(time_ms(lambda: tab.score(ic, ln, ng, bufd, popd, top_n, metrics), 10)[0], 4)
    res['queries_per_batch'] = int(np.count_nonzero(l['label_next_item']))
    t = time.perf_counter()
    ref.score(f['item_clicked'], l['label_next_item'], neg, buf, pop, top_n)
    res['cpu_oracle_ms_per_batch'] = round((time.perf_counter() - t) * 1e3, 1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
