"""BASELINE configs[4] (stress: 1M items, E 512, H 512, K 500, global batch 8192 on 8 GPUs) as ONE rank of eight sees it:
this process stages the GLOBAL batch (8192 sessions), owns 1024 of them (rank 0 of world 8, no collective issued) and runs
full training steps; prints memory, step time and the throughput the 8-GPU job would have if every rank took this long.
   python tools/stress_probe.py [steps]"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    import bench
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 4
    world = int(os.environ.get('NAR_PROBE_WORLD', '8'))
    torch.cuda.set_device(0)
    t0 = time.time()
    pb = make_problem('stress', profile='B')
    per = pb.hp.batch_size // world
    warm_state(pb, 3)
    batches = bench.make_batches(pb, steps + 2, pb.hp.batch_size)
    t_setup = time.time() - t0
    eng = make_engine(pb)
    eng.set_params(pb.layout.init_logical(1))
    eng.world, eng.rank = world, 0            # shard like rank 0 of `world`
    times, Ls = [], []
    for i, (f, l, buf, pop) in enumerate(batches):
        st = eng.stage(f, l, buf, pop, slot='p%d' % (i & 1))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.step(st, train=True)
        eng.world = 1
        eng.apply_gradients(st)               # Adam only: the gradient exchange is what this probe leaves out
        eng.world = world
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b)); Ls.append((st['L'], st['L_global']))
    ms = float(np.median(times[2:])) if len(times) > 2 else times[-1]
    out = {'workload': 'stress (configs[4]) as rank 0 of %d' % world, 'items': pb.plan.num_items, 'acr_dim': pb.plan.acr_dim,
           'rnn_units': pb.hp.rnn_units, 'K': pb.hp.train_total_negative_samples, 'global_batch': pb.hp.batch_size,
           'local_sessions': per, 'L_local_global': Ls[-1], 'Fp': pb.plan.Fp, 'params_M': pb.layout.total / 1e6,
           'step_ms_all': [round(x, 2) for x in times], 'step_ms_median': ms,
           'interactions_per_s_if_all_ranks_alike': Ls[-1][1] / (ms * 1e-3),
           'max_mem_GB': torch.cuda.max_memory_allocated() / 2 ** 30, 'setup_s': round(t_setup, 1), 'loss': None}
    eng.loss_host.copy_(eng.loss_dev); torch.cuda.synchronize()
    out['loss'] = [float(x) for x in eng.loss_host[:3]]
    print('STRESS_PROBE ' + json.dumps(out))
    json.dump(out, open('stress_probe.json', 'w'), indent=1)


if __name__ == '__main__':
    main()
