"""N-rank NCCL data-parallel run == 1-rank run of the same global batch (launched by torchrun, one rank per GPU).

Every rank runs `steps` training steps of the data-parallel engine (sessions sharded, gradients exchanged over
NCCL); rank 0 then repeats the same steps on ONE GPU with the whole global batch and compares per-step loss,
sampled negatives, the all-reduced gradient of the last step and the final weights.  Prints one JSON line
(rank 0).  Used by tests/test_gpu_parity.py::test_nccl_two_ranks_match_single.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chameleon_recsys_b200.clicked_items_state import batch_clicks_for_state_update  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from tools.gpu_step_check import make_engine  # noqa: E402


def main():
    rank = int(os.environ.get('RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    name = os.environ.get('NAR_EQUIV_WORKLOAD', 'g1')
    per_gpu = int(os.environ.get('NAR_EQUIV_BATCH', '64'))
    steps = int(os.environ.get('NAR_EQUIV_STEPS', '3'))
    pb = make_problem(name, profile='B', batch_size=per_gpu * world)
    warm_state(pb, 10)
    it = pb.input_fn()
    batches = []
    for _ in range(steps):
        f, l = it.get_next()
        batches.append((f, l, pb.clicked_items_state.get_recent_clicks_buffer().copy(),
                        pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32)))
        items, ts = batch_clicks_for_state_update(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
        pb.clicked_items_state.update_items_state(items, ts)
    logical = pb.layout.init_logical(11)

    def run(pg):
        eng = make_engine(pb, process_group=pg)
        eng.set_params(logical)
        losses, negs = [], []
        for f, l, buf, pop in batches:
            out = eng.train_step(f, l, buf, pop)
            losses.append((out['xe_loss'], out['reg_loss']))
            negs.append((out['negatives'].clone(), out['stage']['s0'], out['stage']['Bg']))
        torch.cuda.synchronize()
        return eng, losses, negs

    eng_n, loss_n, neg_n = run(dist.group.WORLD)
    # the shards are balanced by valid positions, so their session counts differ: every rank drops its negatives into
    # its rows of a zero [Bg, T, K] tensor and the sum over ranks is the global array
    neg_r, s0_r, Bg_r = neg_n[-1]
    neg_all = torch.zeros((Bg_r,) + tuple(neg_r.shape[1:]), dtype=neg_r.dtype, device=neg_r.device)
    neg_all[s0_r:s0_r + neg_r.shape[0]] = neg_r
    dist.all_reduce(neg_all)
    res = None
    if rank == 0:
        eng_1, loss_1, neg_1 = run(None)
        g_n, g_1 = eng_n.grads, eng_1.grads
        scale = float(g_1.abs().max())
        dp = (eng_n.params - eng_1.params).abs()
        res = {'world': world, 'steps': steps, 'global_batch': per_gpu * world,
               'loss_n': loss_n, 'loss_1': loss_1,
               'loss_rel_max': max(abs(a[0] - b[0]) / abs(b[0]) for a, b in zip(loss_n, loss_1)),
               'reg_rel_max': max(abs(a[1] - b[1]) / max(abs(b[1]), 1e-30) for a, b in zip(loss_n, loss_1)),
               'negatives_equal': bool(torch.equal(neg_all, neg_1[-1][0])),
               'grad_rel_max_last_step': float((g_n - g_1).abs().max()) / scale,
               'param_diff_median': float(dp.median()), 'param_diff_max': float(dp.max()),
               'param_diff_p999': float(torch.quantile(dp[::7].float(), 0.999)), 'lr': pb.hp.learning_rate}
        print('NCCL_EQUIV ' + json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
