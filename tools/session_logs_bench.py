"""Cost of the per-session evaluation logs on one GPU at G1 (batch 256, no baselines): Estimator.evaluate wall time per
batch with the logs off, the negatives log alone and both logs (alternated in the same process over the same batches,
whole evaluate() calls ending in a synchronise, median and spread of the rounds); for one evaluation batch the pack
kernel's device time (torch.profiler over replayed launches, and CUDA events around back-to-back launches), the bytes of
its device-to-host copy, the host time to turn the pinned slot into list entries, and the oracle's CPU time for the same
batch.  Prints one JSON line with the GPU name, power limit and max SM clock.  Writes nothing.
Usage: python tools/session_logs_bench.py [--rounds 3] [--eval-batches 8] [--train-steps 10]"""
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

from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from chameleon_recsys_b200.session_logs import SessionLogs  # noqa: E402
from oracle.session_logs_ref import session_logs_ref  # noqa: E402
from tools.predict_bench import gpu_info, time_ms  # noqa: E402

MODES = {'off': {}, 'negatives': {'sessions_negative_items_log': True},
         'both': {'sessions_negative_items_log': True, 'sessions_chameleon_recommendations_log': True}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--eval-batches', type=int, default=8)
    ap.add_argument('--train-steps', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('session_logs_bench needs a CUDA device')
    name, limit = gpu_info()
    res = {'gpu': name, 'power_limit_max_sm_clock': limit, 'workload': 'g1', 'baselines': 0}

    ests = {}
    for mode, keys in MODES.items():
        pb = make_problem('g1', profile='B')
        warm_state(pb, 3)
        logs = {k: [] for k in keys}
        est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                              pb.session_features_config, pb.hp, pb.clicked_items_state, device=0, **logs)
        it = pb.input_fn()
        est.train(lambda: iter([it.get_next() for _ in range(args.train_steps)]))
        batches = [it.get_next() for _ in range(args.eval_batches)]
        est.evaluate(lambda b=batches: iter(b))                          # builds the evaluation graph, warms up
        ests[mode] = (est, pb, batches, logs)

    def eval_ms(mode):
        est, _, batches, logs = ests[mode]
        for log in logs.values():
            del log[:]
        torch.cuda.synchronize()
        t = time.perf_counter()
        est.evaluate(lambda: iter(batches))
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3 / len(batches)
    times = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for m in MODES:
            times[m].append(eval_ms(m))
    for m in MODES:
        res['evaluate_ms_per_batch_' + m] = round(float(np.median(times[m])), 3)
        res['evaluate_ms_spread_' + m] = round(float(max(times[m]) - min(times[m])), 3)
    res['evaluate_ms_rounds'] = {m: [round(t, 3) for t in times[m]] for m in MODES}

    # ---- one batch's pack: capture the last batch's arguments, then replay them
    est, pb, batches, logs = ests['both']
    calls = []
    orig_add = SessionLogs.add

    def spy_add(self, session_ids, *a, **kw):
        calls.append((np.array(session_ids), [x.clone() if torch.is_tensor(x) else x for x in a],
                      {k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()}))
        return orig_add(self, session_ids, *a, **kw)
    SessionLogs.add = spy_add
    est.evaluate(lambda: iter(batches[-1:]))
    SessionLogs.add = orig_add
    sids, a, kw = calls[0]
    sl = SessionLogs(pb.clicked_items_state.num_items, torch.device('cuda', 0), [], [])
    sl.begin()
    host_ms = []
    for _ in range(12):
        sl.add(sids, *a, **kw)
        torch.cuda.synchronize()
        t = time.perf_counter()
        sl.drain()
        host_ms.append((time.perf_counter() - t) * 1e3)
    res['queries_per_batch'] = sum(len(e['next_click_labels']) for e in sl.recommendations_log[-len(sids):])
    res['valid_positions_per_batch'] = int(a[3])
    res['d2h_bytes_per_batch'] = int(sl.d2h_bytes)
    res['host_lists_ms_per_batch'] = round(float(np.median(host_ms[2:])), 3)

    label_next, pos_idx, sess_off, L = a
    B, K = label_next.shape[0], kw['negatives'].shape[2]
    import ctypes as C
    p = (lambda t: C.c_void_p(t.data_ptr()))
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def pack():
        sl.lib.nar_eval_session_logs_pack(p(kw['pred_ids']), p(kw['pred_probs']), p(kw['cand']), int(kw['cand_stride']),
                                          p(pos_idx), p(sess_off), p(kw['pop']), p(kw['negatives']), p(label_next), B, K,
                                          int(L), sl.num_items, sl.flags, p(sl.packed), stream)

    def pack50():
        for _ in range(50):
            pack()
    ms, _ = time_ms(pack50, 10)
    res['pack_launch_to_launch_us'] = round(ms * 1e3 / 50, 2)          # events around 50 back-to-back launches
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        pack50()
        torch.cuda.synchronize()
    dev_us = sum(e.device_time_total for e in prof.key_averages() if 'session_logs_pack' in e.key)
    res['pack_kernel_us'] = round(dev_us / 50, 2)                      # device time of the kernel alone

    # ---- the oracle on the same batch (CPU)
    host = {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in kw.items()}
    ln, pi = label_next.cpu().numpy(), pos_idx.cpu().numpy()[:int(L)]
    t = time.perf_counter()
    session_logs_ref(sids, ln, host['negatives'], host['pred_ids'], host['pred_probs'], host['pop'], pos_idx=pi)
    res['cpu_oracle_ms_per_batch'] = round((time.perf_counter() - t) * 1e3, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
