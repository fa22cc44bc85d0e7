"""Cost of the baselines' recommendations (DESIGN.md section 16) on one GPU at G1 (46 033 articles, batch 256, all seven
baselines with the reference parameters): the recent-clicks state warmed with warm_state and every baseline trained on
--train-steps batches (a full kNN ring after 12), then per baseline and candidate set (the recent-clicks buffer's ids,
the whole catalog) Estimator.predict(recommender=...) over one batch with positions='last': ms per batch from the host
clock around calls that end in a synchronise (median of --repeats, after a warm-up call), and the device time of one
BaselineTables.recommend call on the same queries from CUDA events (median of --repeats): its inputs already on the
device, so this is the recommend kernel plus, for pop_recent, the buffer-histogram rebuild the call makes.  Also the
queries per batch, the candidates, and the GPU name, power limit and max SM clock read in the same call.  Prints one
JSON line; writes nothing.
Usage: python tools/baseline_predict_bench.py [--repeats 5] [--train-steps 12]"""
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
from chameleon_recsys_b200.dp import session_lengths  # noqa: E402
from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from tools.predict_bench import gpu_info  # noqa: E402

ALL7 = SUFFIXES + KNN_SUFFIXES


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--train-steps', type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('baseline_predict_bench needs a CUDA device')
    name, limit = gpu_info()
    pb = make_problem('g1', profile='B')
    warm_state(pb, 3)
    hp = pb.hp.copy(eval_benchmarks=tuple({'recommender': s, 'params': {}} for s in ALL7))
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, hp, pb.clicked_items_state, device=0)
    it = pb.input_fn()
    est.train(lambda: iter([it.get_next() for _ in range(args.train_steps)]))
    batch = it.get_next()
    state = pb.clicked_items_state
    tabs = state.baselines
    f = batch[0]
    ic = np.asarray(f['item_clicked'], dtype=np.int64)
    T = ic.shape[1]
    lens = session_lengths(f['session_size'], T)
    q_pos = (np.flatnonzero(lens > 0) * T + lens[lens > 0] - 1).astype(np.int32)
    buf = state.get_recent_clicks_buffer()
    cands = {'buffer': np.unique(buf[buf != 0]), 'catalog': np.arange(1, state.num_items, dtype=np.int64)}
    top_n = int(hp.eval_metrics_top_n)
    res = {'metric': 'baseline_predict_ms_per_batch', 'workload': 'g1', 'batch': int(ic.shape[0]),
           'queries': int(q_pos.size), 'top_n': top_n, 'candidates': {k: int(v.size) for k, v in cands.items()},
           'repeats': args.repeats, 'gpu': name, 'power_limit_and_max_sm_clock': limit}
    d = tabs.dev
    ic_d, q_d = torch.from_numpy(ic).to(d), torch.from_numpy(q_pos).to(d)
    buf_d = torch.from_numpy(np.asarray(buf, dtype=np.int64)).to(d)
    pop_d = torch.from_numpy(np.asarray(state.get_articles_pop(), dtype=np.int64)).to(d)
    for cname, cand in cands.items():
        cand_d = torch.from_numpy(cand).to(d)
        for sfx in ALL7:
            kw = dict(recommender=sfx, candidates=None if cname == 'buffer' else 'catalog')
            list(est.predict(lambda: iter([batch]), **kw))                           # warm-up
            host = []
            for _ in range(args.repeats):
                torch.cuda.synchronize()
                t = time.perf_counter()
                list(est.predict(lambda: iter([batch]), **kw))
                torch.cuda.synchronize()
                host.append((time.perf_counter() - t) * 1e3)
            dev = []
            for _ in range(args.repeats):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                tabs.recommend(sfx, ic_d, q_d, cand_d, buf_d, pop_d, top_n)
                e1.record()
                torch.cuda.synchronize()
                dev.append(e0.elapsed_time(e1))
            res['%s_%s_ms' % (sfx, cname)] = round(float(np.median(host)), 3)
            res['%s_%s_call_device_ms' % (sfx, cname)] = round(float(np.median(dev)), 3)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
