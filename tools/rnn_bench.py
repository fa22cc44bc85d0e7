"""Cost of the three session cells (rnn_cell 'ugrnn', 'gru', 'lstm') on one GPU at G1 (batch 256, H 255 -> Hp 256):
training interactions/s per cell with the inputs resident in HBM (bench.py's device loop: one engine step + TF-Adam per
batch, the next batch's sampler queued on the side stream; CUDA events around whole regions, the cells alternated in one
process, median of the rounds), the recurrence kernels' device time per training step (torch.profiler, a separate run
after the timing), and the recurrent weight bytes the kernels stream per session-step (from the shapes: the recurrent
matrices are read once per CTA step and shared by the SB = 4 sessions of a CTA).  Prints one JSON line with the GPU
name, power limit and max SM clock.  Writes nothing.
--residual: per cell, the plain stack and the residual stack (rnn_residual_connections, DESIGN.md section 15) instead,
alternated in one process, one pair of engines per cell; interactions/s of each round and their medians.
Usage: python tools/rnn_bench.py [--rounds 3] [--steps 20] [--profile-steps 5] [--residual]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from bench import make_batches  # noqa: E402
from tools.predict_bench import gpu_info  # noqa: E402

CELLS = ('ugrnn', 'gru', 'lstm')
KERNELS = {'ugrnn': ('ugrnn_fwd_kernel', 'ugrnn_bwd_kernel'), 'gru': ('gru_fwd_kernel', 'gru_bwd_kernel'),
           'lstm': ('lstm_fwd_kernel', 'lstm_bwd_kernel')}
# recurrent weight columns per unit the forward / backward products read: UGRNN Wh [Hp, 2Hp]; GRU Whg [Hp, 2Hp] + Whc
# [Hp, Hp]; LSTM Wh [Hp, 4Hp] (the backward reads the same blocks transposed)
WH_COLS = {'ugrnn': 2, 'gru': 3, 'lstm': 4}
SB = 4


def make_engine(cell, n_batches, residual=False):
    pb = make_problem('g1', profile='B', rnn_cell=cell, rnn_residual_connections=residual)
    warm_state(pb, 3)
    batches = make_batches(pb, n_batches, pb.hp.batch_size)
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, pb.hp, pb.clicked_items_state, device=0)
    eng = est._ensure_spec(None, None).model.engine
    staged = [eng.stage(f, l, buf, pop, slot='%s%d' % (cell, i)) for i, (f, l, buf, pop) in enumerate(batches)]
    torch.cuda.synchronize()
    return eng, staged


def run_steps(eng, staged):
    side = eng.side_stream()
    for i, st in enumerate(staged):
        eng.step(st, train=True)
        eng.apply_gradients(st)
        if i + 1 < len(staged):
            eng.prepare(staged[i + 1], eng.global_step + 1, stream=side)


def train_rate(eng, staged, warmup):
    run_steps(eng, staged[:warmup])
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    run_steps(eng, staged[warmup:])
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b)
    n = sum(st['L_global'] for st in staged[warmup:])
    return n / (ms * 1e-3), ms / (len(staged) - warmup)


def kernel_us_per_step(eng, staged, cell):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_steps(eng, staged)
        torch.cuda.synchronize()
    out = {}
    for k in KERNELS[cell]:
        ev = [e for e in prof.key_averages() if k in e.key]
        total = sum(getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0)) for e in ev)
        out[k] = round(total / len(staged), 2)
    return out


def residual_main(args, res, warmup):
    """Plain and residual stack of each cell, alternated round by round."""
    res['train_interactions_per_s'], res['train_interactions_per_s_rounds'], res['launches_per_step'] = {}, {}, {}
    for c in CELLS:
        engs = {r: make_engine(c, warmup + args.steps, residual=r) for r in (False, True)}
        rates = {False: [], True: []}
        for _ in range(args.rounds):
            for r in (False, True):
                n0 = engs[r][0].launches
                rates[r].append(train_rate(*engs[r], warmup)[0])
                res['launches_per_step'].setdefault(c, {})[('on' if r else 'off')] = \
                    (engs[r][0].launches - n0) // (warmup + args.steps)
        for r in (False, True):
            k = '%s_%s' % (c, 'on' if r else 'off')
            res['train_interactions_per_s'][k] = round(float(np.median(rates[r])), 1)
            res['train_interactions_per_s_rounds'][k] = [round(v, 1) for v in rates[r]]
        del engs
        torch.cuda.empty_cache()
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--profile-steps', type=int, default=5)
    ap.add_argument('--residual', action='store_true', help='plain vs residual session stack per cell')
    args = ap.parse_args()
    name, limit = gpu_info()
    res = {'gpu': name, 'power_limit_and_max_sm_clock': limit, 'workload': 'g1', 'batch': 256}
    warmup = 5
    if args.residual:
        return residual_main(args, res, warmup)
    engs = {c: make_engine(c, warmup + args.steps) for c in CELLS}
    Hp = engs['lstm'][0].Hp
    res['Hp'] = Hp
    rates = {c: [] for c in CELLS}
    ms = {c: [] for c in CELLS}
    for _ in range(args.rounds):
        for c in CELLS:
            r, m = train_rate(*engs[c], warmup)
            rates[c].append(r); ms[c].append(m)
    res['train_interactions_per_s'] = {c: round(float(np.median(rates[c])), 1) for c in CELLS}
    res['train_ms_per_step'] = {c: round(float(np.median(ms[c])), 4) for c in CELLS}
    res['train_interactions_per_s_rounds'] = {c: [round(v, 1) for v in rates[c]] for c in CELLS}
    res['recurrence_kernel_us_per_step'] = {c: kernel_us_per_step(engs[c][0], engs[c][1][:args.profile_steps], c) for c in CELLS}
    res['wh_bytes_per_session_step'] = {c: {'fwd': Hp * WH_COLS[c] * Hp * 4 // SB, 'bwd': Hp * WH_COLS[c] * Hp * 4 // SB}
                                        for c in CELLS}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
