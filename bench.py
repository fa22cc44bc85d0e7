#!/usr/bin/env python
"""bench.py - NAR train interactions/s on H100 (BASELINE.json metric), one JSON line on rank 0.

  python bench.py --gpus N --steps K --warmup W            # this repo (CUDA)
  python bench.py --impl reference --gpus N --steps K --warmup W   # reference CPU path (oracle port)
  python bench.py --steps K --warmup W --dump-outputs DIR         # + what the last timed step computed, as DIR/*.npy

A "step" = one pass of the NAR training hot path over one batch of synthetic G1-shaped sessions
(sampler -> feature gather -> CAR -> UGRNN -> FC -> scorer -> softmax-CE -> backward -> TF-Adam).
  value : interactions/s with the step inputs already resident in HBM (CUDA events over K steps)
  e2e   : the same metric through the reference-facing API (Estimator.train: model_fn / input_fn /
          ItemsStateUpdaterHook) with HOST numpy batches: per step one pinned H2D copy of the inputs,
          the host ClickedItemsState update and a D2H read of the loss, all inside the timed region
  roofline        : the dominant kernel (CAR GEMM, tensor bound) timed alone, vs MEASURED_PEAKS.json if present,
                    else the H100 SXM data sheet
  roofline_gather : the embedding-gather kernel (HBM bound; the kernel north_star names)
  cpu_baseline    : the oracle (torch-CPU restatement of the TF1.12 graph) on the same workload
Data parallel (N > 1, torchrun): weak scaling, per-GPU batch fixed, global batch = N x batch;
sessions are sharded, the sampler sees the global batch, dense + embedding grads are sum-allreduced (NCCL).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
# (CUDA_MODULE_LOADING=EAGER was tried against first-launch stalls of rarely selected GEMM variants inside the timed region: it
# also loads every kernel of libtorch - minutes of start-up.  Not used.)


_REAL_STDOUT = None


def emit(line: dict):
    out = _REAL_STDOUT or sys.stdout
    out.write(json.dumps(line) + '\n')
    out.flush()


def _peaks():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return d.get('hbm_gbs', 3350.0), d.get('bf16_tflops', 989.0), d.get('bf16_tflops_sustained', 989.0), 'measured'
    # H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 TFLOP/s dense bf16
    return 3350.0, 989.0, 989.0, 'H100 SXM data sheet'


class ClockSampler:
    """SM clock / throttle reasons DURING the timed region.  Sampled in-process through NVML (the library nvidia-smi
    itself calls) from a thread, every 10 ms: spawning `nvidia-smi -lms` inside the timed region enumerates every GPU
    of the box and can stall kernel launches on an 8-GPU node for tens of ms.  Falls back to an nvidia-smi subprocess started BEFORE the
    warm-up (only its rows from the timed region are used) when pynvml is missing."""

    REASONS = [(0x8, 'hw_slowdown'), (0x40, 'hw_thermal_slowdown'), (0x20, 'sw_thermal_slowdown'), (0x4, 'sw_power_cap')]

    def __init__(self, index=0):
        self.index = self._physical_index(index)
        self.samples, self.rows = [], []
        self.nvml = self.handle = self.proc = None
        self.running = False
        self.row0 = 0
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nvml = pynvml
            self.handle = pynvml.nvmlDeviceGetHandleByIndex(self.index)
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(self.handle, pynvml.NVML_CLOCK_SM))
        except Exception:  # noqa: BLE001
            self.nvml = None
            q = ('clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,'
                 'clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap')
            try:
                self.proc = subprocess.Popen(['nvidia-smi', '-i', str(self.index), '--query-gpu=' + q,
                                              '--format=csv,noheader,nounits', '-lms', '50'],
                                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
                threading.Thread(target=self._read_smi, daemon=True).start()
            except Exception:  # noqa: BLE001
                self.proc = None

    @staticmethod
    def _physical_index(i):
        vis = os.environ.get('CUDA_VISIBLE_DEVICES')
        if vis:
            ids = [x.strip() for x in vis.split(',') if x.strip()]
            if i < len(ids) and ids[i].isdigit():
                return int(ids[i])
        return i

    def _read_smi(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def _poll(self):
        n = self.nvml
        while self.running:
            try:
                mhz = float(n.nvmlDeviceGetClockInfo(self.handle, n.NVML_CLOCK_SM))
                try:
                    bits = int(n.nvmlDeviceGetCurrentClocksEventReasons(self.handle))
                except Exception:  # noqa: BLE001
                    bits = int(n.nvmlDeviceGetCurrentClocksThrottleReasons(self.handle))
                self.samples.append((mhz, bits))
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.01)

    def start(self):
        if self.nvml is not None:
            self.running = True
            self.thread = threading.Thread(target=self._poll, daemon=True)
            self.thread.start()
        else:
            self.row0 = len(self.rows)

    def stop(self):
        if self.nvml is not None:
            self.running = False
            self.thread.join(timeout=1)
            sm = [x[0] for x in self.samples]
            bits = 0
            for _, b in self.samples:
                bits |= b
            return {'sm_mhz': float(np.median(sm)) if sm else None, 'sm_max_mhz': self.max_mhz, 'samples': len(sm),
                    'reasons': [name for mask, name in self.REASONS if bits & mask], 'source': 'nvml'}
        if self.proc is None:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['nvml and nvidia-smi unavailable']}
        time.sleep(0.06)
        rows = self.rows[self.row0:]
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for r in rows:
            f = [x.strip() for x in r.split(',')]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for (_, name), v in zip(self.REASONS, f[3:7]):
                if v.lower().startswith('active'):
                    reasons.add(name)
        return {'sm_mhz': float(np.median(sm)) if sm else None, 'sm_max_mhz': max(mx) if mx else None,
                'samples': len(sm), 'reasons': sorted(reasons), 'source': 'nvidia-smi'}


def make_batches(pb, n, global_batch, snapshot_at=None):
    """n host batches + the host state (buffer, pop_norm) each step sees; state advances like the hook does.
    With snapshot_at=i also returns a deep copy of the ClickedItemsState as it was before batch i."""
    import copy
    it = pb.input_fn(batch_size=global_batch)
    out = []
    snap = None
    for i in range(n):
        if snapshot_at is not None and i == snapshot_at:
            snap = copy.deepcopy(pb.clicked_items_state)
        f, l = it.get_next()
        buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
        pop = pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32)
        out.append((f, l, buf, pop))
        pb.clicked_items_state.update_from_batch(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
    return out if snapshot_at is None else (out, snap)


def interactions(batch):
    f = batch[0]
    T = f['item_clicked'].shape[1]
    return int(np.clip(f['session_size'] - 1, 0, T).sum())


def oracle_for(pb):
    import torch
    from oracle.nar_oracle import NarOracle
    hp = pb.hp
    o = NarOracle(pb.session_features_config, pb.articles_features_config, pb.internal_features_config,
                  pb.content_article_embeddings_matrix, pb.articles_metadata,
                  negative_samples=hp.train_total_negative_samples, softmax_temperature=hp.softmax_temperature,
                  reg_weight_decay=hp.reg_l2, recent_clicks_for_normalization=hp.recent_clicks_for_normalization,
                  elapsed_days_smooth_log_base=hp.elapsed_days_smooth_log_base,
                  popularity_smooth_log_base=hp.popularity_smooth_log_base, CAR_embedding_size=hp.CAR_embedding_size,
                  rnn_units=hp.rnn_units, rnn_num_layers=hp.rnn_num_layers, lr=hp.learning_rate, ranking=hp.ranking,
                  dtype=torch.float32)
    o.set_params(pb.layout.init_logical(hp.init_seed))
    return o


def time_oracle(pb, batches, warmup, steps, state=None):
    """Reference CPU path: one full train step per batch - hook.before_run (state arrays) -> sampler + forward +
    backward + TF-Adam -> hook.after_run (ClickedItemsState update, numpy like the reference), all timed."""
    import torch
    from oracle import sampler_ref
    # 16 threads by default (NAR_CPU_THREADS): at these GEMM sizes more threads mostly add synchronisation cost
    torch.set_num_threads(min(os.cpu_count() or 1, int(os.environ.get('NAR_CPU_THREADS', '16'))))
    hp = pb.hp
    o = oracle_for(pb)
    n_int, t_total = 0, 0.0
    for i, (f, l, buf, pop) in enumerate(batches[:warmup + steps]):
        t0 = time.perf_counter()
        if state is not None:                       # the hook's feed: state as left by the previous step
            buf = state.get_recent_clicks_buffer()
            pop = state.get_articles_recent_pop_norm().astype(np.float32)
        allc = np.concatenate([f['item_clicked'], l['label_last_item']], axis=1)
        neg = sampler_ref.sample_negatives(allc, buf, hp.train_total_negative_samples,
                                           hp.train_negative_samples_from_buffer, hp.sampler_seed, i + 1)
        o.train_step(f, l, neg, buf, pop)
        if state is not None:
            state.update_from_batch(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
        dt = time.perf_counter() - t0
        if i >= warmup:
            t_total += dt
            n_int += interactions((f, l))
    return n_int / t_total, t_total / max(1, steps), torch.get_num_threads()


REF_STEP_SESSIONS = 256       # sessions per reference-arm step (bounded sample of the global batch)


def run_reference(args):
    """Reference arm: the CPU restatement of the TF1.12 graph (oracle/) with the numpy ClickedItemsState
    (oracle/clicked_items_state_ref.py) - nothing of the product runs here: libnar_b200.so is never loaded."""
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from oracle.clicked_items_state_ref import ClickedItemsStateRef
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return 0
    hp_over = {'batch_size': args.global_batch // args.gpus} if args.global_batch else {}
    pb = make_problem(args.workload, profile=args.profile, session_len=args.session_len, state_cls=ClickedItemsStateRef, **hp_over)
    gb = pb.hp.batch_size * args.gpus
    # bounded sample: a step of this arm processes at most REF_STEP_SESSIONS sessions of the global batch (one oracle
    # step costs ~2.5 s of CPU work per 256 sessions), so that --steps K --warmup W ends within a few minutes at any N
    sb = min(gb, REF_STEP_SESSIONS)
    warm_state(pb, args.state_warmup)
    import copy
    state = copy.deepcopy(pb.clicked_items_state)
    batches = make_batches(pb, args.warmup + args.steps, sb)
    v, sec_per_step, cores = time_oracle(pb, batches, args.warmup, args.steps, state=state)
    with open('/proc/self/maps') as fh:
        product_lib_mapped = 'libnar_b200' in fh.read()
    line = {'impl': 'reference', 'metric': 'NAR train interactions/sec', 'value': v, 'unit': 'interactions/s',
            'n_gpus': args.gpus, 'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': sec_per_step * 1e3,
            'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
            'config': workload_config(pb, args, gb),
            'cpu_baseline': {'value': v, 'unit': 'interactions/s', 'cores': cores, 'kind': 'port',
                             'sample': '%d full train steps of %d sessions each (%s) on the torch-CPU oracle, numpy '
                                       'ClickedItemsState update inside the timed region; TF1.12 itself cannot be installed '
                                       '(python 3.12, no network)' % (args.steps, sb, 'the whole global batch' if sb == gb else
                                                                     'a bounded sample of the %d-session global batch' % gb)},
            'e2e': {'value': v, 'unit': 'interactions/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
            'product_lib_mapped': product_lib_mapped}
    emit(line)
    return 0


def workload_config(pb, args, gb):
    hp = pb.hp
    return {'workload': 'G1-shaped synthetic' if args.workload == 'g1' else args.workload, 'items': pb.plan.num_items,
            'acr_dim': pb.plan.acr_dim, 'rnn_units': hp.rnn_units, 'CAR_embedding_size': hp.CAR_embedding_size,
            'global_batch_sessions': gb, 'per_gpu_batch_sessions': hp.batch_size, 'truncate_session_length': hp.truncate_session_length,
            'negatives': hp.train_total_negative_samples, 'feature_profile': pb.wl.profile, 'session_len': pb.wl.session_len,
            'rnn_cell': hp.rnn_cell, 'ranking': hp.ranking, 'parallelism': 'dp%d' % args.gpus,
            'sharding': ('contiguous session shards of the global batch, boundaries balanced by valid positions (per-GPU mean '
                         '%d sessions)' % hp.batch_size) if args.gpus > 1 and os.environ.get('NAR_DP_BALANCE', '1') == '1'
                        else 'contiguous session shards, equal counts',
            'l2_policy': 'no explicit flush: the per-step working set (X,H1,E,dE,PD activations) exceeds the 50 MB L2'}


def run_ours(args):
    import torch
    import torch.distributed as dist
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local_rank)
    pg = None
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
        pg = dist.group.WORLD
    if world != args.gpus:
        if rank == 0:
            print('warning: --gpus %d but WORLD_SIZE %d' % (args.gpus, world), file=sys.stderr)
    hp_over = {}
    if args.global_batch:
        if args.global_batch % world:
            raise SystemExit('--global-batch must be a multiple of the number of ranks')
        hp_over['batch_size'] = args.global_batch // world
    pb = make_problem(args.workload, profile=args.profile, session_len=args.session_len, **hp_over)
    hp = pb.hp
    gb = hp.batch_size * world
    warm_state(pb, args.state_warmup)
    n_total = args.warmup + args.steps
    # first half: device-resident run, second half: e2e run (the hook starts from the state before batch n_total)
    E2E_REGIONS = 3
    batches, state_e2e = make_batches(pb, n_total + args.warmup + E2E_REGIONS * args.steps, gb, snapshot_at=n_total)
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, hp, state_e2e, process_group=pg, device=local_rank)
    spec = est._ensure_spec(None, None)
    eng = spec.model.engine

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ------------------------------------------------------------------ value: inputs resident in HBM
    staged = [eng.stage(f, l, buf, pop, slot='bench%d' % i) for i, (f, l, buf, pop) in enumerate(batches[:n_total])]
    torch.cuda.synchronize()

    side = eng.side_stream()

    last_out = {}

    def dev_step(i):
        """step i on the main stream; the weight-independent front of step i+1 (sampler, row lists, statistics)
        is queued on the side stream right behind it (the reference prefetches its next batch the same way)"""
        st = staged[i]
        last_out['step'] = eng.step(st, train=True)     # ONE C call: forward + backward, every launch sequenced in libnar_b200
        eng.apply_gradients(st)              # (NCCL sum of the gradients when world > 1) + TF-Adam
        if eng.use_side_stream and i + 1 < len(staged):
            eng.prepare(staged[i + 1], eng.global_step + 1, stream=side)

    # the host may run at most `depth` steps ahead of the device (a training loop that reads its loss has depth 1-2;
    # unbounded run-ahead only grows the caching allocator's cross-stream pool).  No host sync inside a step.
    depth = int(os.environ.get('NAR_BENCH_DEPTH', '2'))
    done = {}

    enq = [0.0]
    enq_each = []

    def bounded_step(i):
        if depth > 0 and (i - depth) in done:
            done.pop(i - depth).synchronize()
        t0 = time.perf_counter()
        dev_step(i)
        dt = time.perf_counter() - t0
        enq[0] += dt                              # host time spent queueing the step (the wait above is not part of it)
        enq_each.append(dt)
        if depth > 0:
            ev = torch.cuda.Event()
            ev.record()
            done[i] = ev

    sampler = ClockSampler(local_rank) if rank == 0 else None      # NVML init / process start-up outside the timed region
    for i in range(args.warmup):
        bounded_step(i)
    barrier()
    if rank == 0:
        sampler.start()
    l0 = eng.launches + ops.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t_host0 = time.perf_counter()
    enq[0] = 0.0
    del enq_each[:]
    for i in range(args.warmup, n_total):
        bounded_step(i)
    e1.record()
    host_loop_ms = (time.perf_counter() - t_host0) * 1e3 / args.steps
    host_enqueue_ms = enq[0] * 1e3 / args.steps
    barrier()
    launches = eng.launches + ops.LAUNCHES - l0
    ms = torch.tensor([e0.elapsed_time(e1)], device='cuda')
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_total = float(ms.item())
    n_int = sum(st['L_global'] for st in staged[args.warmup:])
    value = n_int / (ms_total * 1e-3)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:       # before anything below runs the engine again
        dump_outputs(args.dump_outputs, eng, last_out['step'])

    # ------------------------------------------------------------------ BASELINE configs[3]: G1-shaped, GLOBAL batch 4096 on 8 GPUs
    # (512 sessions per GPU).  The scaling series keeps the per-GPU batch of configs[1] (weak scaling, 256 per GPU);
    # this extra device-timed measurement reports the configuration BASELINE.json names, in the same line.
    cfg3 = None
    if world == 8 and args.workload == 'g1' and not args.global_batch and os.environ.get('NAR_BENCH_CFG3', '1') == '1':
        pb3 = make_problem('g1', profile=args.profile, session_len=args.session_len, batch_size=512)
        warm_state(pb3, 20)
        w3, k3 = 3, 10
        b3 = make_batches(pb3, w3 + k3, 512 * world)
        est3 = build_estimator(None, pb3.content_article_embeddings_matrix, pb3.articles_metadata, pb3.articles_features_config,
                               pb3.session_features_config, pb3.hp, pb3.clicked_items_state, process_group=pg, device=local_rank)
        eng3 = est3._ensure_spec(None, None).model.engine
        st3 = [eng3.stage(f, l, bu, po, slot='c3_%d' % i) for i, (f, l, bu, po) in enumerate(b3)]
        torch.cuda.synchronize()
        for i in range(w3):
            eng3.step(st3[i], train=True); eng3.apply_gradients(st3[i])
        barrier()
        a3, z3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a3.record()
        for i in range(w3, w3 + k3):
            eng3.step(st3[i], train=True); eng3.apply_gradients(st3[i])
            if i + 1 < len(st3):
                eng3.prepare(st3[i + 1], eng3.global_step + 1, stream=eng3.side_stream())
        z3.record()
        barrier()
        m3 = torch.tensor([a3.elapsed_time(z3)], device='cuda')
        dist.all_reduce(m3, op=dist.ReduceOp.MAX)
        n3 = sum(s['L_global'] for s in st3[w3:])
        cfg3 = {'workload': 'BASELINE configs[3]: G1-shaped, global batch 4096 = 512 sessions per GPU, 8 GPUs', 'steps': k3, 'warmup': w3,
                'value': n3 / (float(m3.item()) * 1e-3), 'unit': 'interactions/s', 'ms_per_step': float(m3.item()) / k3,
                'interactions_per_step': n3 / k3}
        del eng3, est3, st3

    # ------------------------------------------------------------------ e2e: Estimator API, host batches
    e2e_batches = batches[n_total:]
    h2d = []

    class ListInput:
        def __init__(self, items):
            self.items = list(items)

        def get_next(self):
            from chameleon_recsys_b200.datasets import OutOfRangeError
            if not self.items:
                raise OutOfRangeError()
            f, l, _, _ = self.items.pop(0)
            return f, l

    est.train(lambda: ListInput(e2e_batches[:args.warmup]))
    # Three back-to-back timed regions of exactly K steps each; ALL are listed and the MEDIAN one is reported (on a
    # fresh box the container image is paged in lazily, and one-off host stalls - allocator slow paths, a state-buffer
    # wrap-around - land in a single region; the median neither hides nor is dominated by them).
    e2e_runs = []
    for rep in range(E2E_REGIONS):
        lo = args.warmup + rep * args.steps
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t_wall0 = time.perf_counter()
        e0.record()
        before_int = est.interactions
        est.train(lambda: ListInput(e2e_batches[lo:lo + args.steps]))
        e1.record()
        barrier()
        wall = time.perf_counter() - t_wall0
        ms2 = torch.tensor([e0.elapsed_time(e1)], device='cuda')
        if world > 1:
            dist.all_reduce(ms2, op=dist.ReduceOp.MAX)
        e2e_runs.append({'ms': float(ms2.item()), 'wall': wall, 'interactions': est.interactions - before_int})
    med = sorted(e2e_runs, key=lambda r: r['ms'] / max(1, r['interactions']))[len(e2e_runs) // 2]
    wall = med['wall']
    e2e_int = med['interactions']
    e2e_ms = med['ms']
    e2e_value = e2e_int / (e2e_ms * 1e-3)
    h2d_bytes = int(est.h2d_bytes_per_step)          # the copy Estimator.train issues per step (device-resident state: no buffer / popularity upload)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return 0

    # ------------------------------------------------------------------ rooflines (rank 0, kernels timed alone)
    hbm_peak, tf_peak, tf_sust, peak_src = _peaks()
    st = staged[-1]
    roof, roof_g = kernel_rooflines(eng, st, hbm_peak, tf_peak, peak_src)

    # ------------------------------------------------------------------ cpu baseline (bounded sample)
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        nb = max(1, args.cpu_steps)
        v, sec, cores = time_oracle(pb, batches[:nb + 1], 1, nb)
        cpu = {'value': v, 'unit': 'interactions/s', 'cores': cores, 'kind': 'port',
               'sample': '%d full train steps (batch %d sessions, %.2f s/step) on the torch-CPU oracle after 1 warm-up; '
                         'the oracle computes every padded position like the TF graph does' % (nb, gb, sec)}

    line = {'metric': 'NAR train interactions/sec', 'value': value, 'unit': 'interactions/s', 'n_gpus': world,
            'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': ms_total / args.steps, 'higher_is_better': True,
            'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32 (wgmma: %s forward, %s backward; fp32 accumulate)' % ('bf16x3 (error-compensated)' if eng.fwd_prec == 4 else '3xTF32', '3xTF32' if eng.bwd_prec == 3 else 'single-pass TF32'), 'dedup_car_layer1': bool(eng.dedup),
            'data': 'synthetic', 'config': workload_config(pb, args, gb),
            'interactions_per_step': n_int / args.steps,
            'e2e': {'value': e2e_value, 'unit': 'interactions/s', 'h2d_bytes_per_step': h2d_bytes, 'd2h_bytes_per_step': 16,
                    'ms_per_step': e2e_ms / args.steps, 'wall_ms_per_step': wall * 1e3 / args.steps,
                    'runs_ms_per_step': [r['ms'] / args.steps for r in e2e_runs], 'policy': 'median of three K-step regions',
                    'api': 'Estimator.train(input_fn) -> nar_module_model_fn -> NARModuleModel.train + ItemsStateUpdaterHook'},
            'gpu_launches': launches, 'gpu_launches_per_step': launches / args.steps,
            'host_enqueue_ms_per_step': host_enqueue_ms, 'host_enqueue_ms_median_max': [float(np.median(enq_each)) * 1e3, float(np.max(enq_each)) * 1e3],
            'host_loop_ms_per_step_incl_waiting_for_the_gpu': host_loop_ms,
            'host_run_ahead_steps': depth,
            'roofline': roof, 'roofline_gather': roof_g, 'clocks': clocks}
    if cfg3:
        line['configs3_g1_batch4096_8gpu'] = cfg3
    if cpu:
        line['cpu_baseline'] = cpu
    emit(line)
    if world > 1:
        dist.destroy_process_group()
    return 0


DUMP_BUDGET_BYTES = 64 * 1024 * 1024 - 64 * 1024     # all .npy files of one dump, headers included


def dump_outputs(out_dir, eng, out):
    """What the last timed step handed its caller, as out_dir/<name>.npy: the loss accumulators, the logits, the sampled
    negatives and the parameters after the Adam update.  Every array gets an equal share of DUMP_BUDGET_BYTES; one that
    does not fit its share is replaced by its entries at a fixed seeded set of flat indices, stored next to it as
    <name>_index.npy (float64), so that the whole dump stays within the budget."""
    import torch
    torch.cuda.synchronize()
    arrays = {'loss': out['loss'].detach().float().cpu().numpy()[:3],          # xe, l2 regulariser, novelty regulariser
              'negatives': out['negatives'].detach().cpu().numpy().astype(np.float64),
              'params': eng.params.detach().cpu().numpy()}
    if out['logits'] is not None:
        arrays['logits'] = out['logits'].detach().float().cpu().numpy()
    os.makedirs(out_dir, exist_ok=True)
    share = DUMP_BUDGET_BYTES // len(arrays)
    for name, a in arrays.items():
        if a.nbytes > share:
            k = share // (a.itemsize + 8)                   # sampled values + their float64 indices
            idx = np.sort(np.random.RandomState(0).choice(a.size, k, replace=False))
            np.save(os.path.join(out_dir, name + '_index.npy'), idx.astype(np.float64))
            a = a.reshape(-1)[idx]
        np.save(os.path.join(out_dir, name + '.npy'), a)


def kernel_rooflines(eng, st, hbm_peak, tf_peak, peak_src):
    """Time the two kernels north_star names, alone, with CUDA events on the launching stream."""
    import torch
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import ACT_TANH
    eng.step(st, train=False, keep=True)
    L, K = st['L'], eng.K
    R = L + L * (K + 1)
    plan = eng.plan
    planc = eng.feature_plan_c(st)
    t = st['t']
    row_pos, row_item = eng.last['row_pos'], eng.last['row_item']
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device='cuda')

    def timeit(fn, iters=20):
        ts = []
        for _ in range(3):
            fn()
        for _ in range(iters):
            flush.zero_()                         # L2 flush between timed iterations
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.mean(ts))

    # ---- embedding gather.  (a) the bulk form SURVEY 8(d) defines the byte count on: one feature row per (position,
    # candidate) pair, R = L*(2+K) rows; (b) what the step actually launches since the per-unique-id CAR layer 1: the
    # 2L + U base rows (every distinct negative id once) - 13x fewer bytes, a launch-latency sized kernel.
    Xfull = torch.empty(R, plan.Fp, device='cuda')
    rows_full = ops.row_layout(R, L, K + 1, ctx_col0=plan.ctx_col0)
    ms_g = timeit(lambda: ops.gather_features(planc, row_pos, row_item, rows_full, t['event_ts'], t['max_ts'], Xfull))
    zed = torch.zeros(4, device='cuda')
    ms_0 = timeit(lambda: zed.zero_())            # what an (almost) empty kernel costs between the same two events
    E = plan.acr_dim if plan.use_acr else 0
    Di = plan.item_emb_dim if plan.use_item_emb else 0
    # SURVEY.md 8(d): per interaction (2+K)*(E+Di)*4 read + same written + (2+K)*8 index bytes
    gbytes = L * ((2 + K) * (E + Di) * 4 * 2 + (2 + K) * 8)
    actual = R * plan.Fp * 4 + R * (E + Di) * 4 + R * 12
    roof_g = {'kernel': 'gather_features_kernel', 'bound': 'hbm', 'achieved': gbytes / (ms_g * 1e-3) / 1e9, 'peak': hbm_peak,
              'unit': 'GB/s', 'frac': gbytes / (ms_g * 1e-3) / 1e9 / hbm_peak, 'peak_source': peak_src,
              'rows': R, 'us': ms_g * 1e3, 'algorithmic_bytes': gbytes, 'bytes_moved_incl_all_feature_columns': actual,
              'achieved_incl_all_columns': actual / (ms_g * 1e-3) / 1e9,
              'event_pair_overhead_us': ms_0 * 1e3,
              'frac_net_of_event_overhead': gbytes / (max(ms_g - ms_0, 1e-6) * 1e-3) / 1e9 / hbm_peak,
              'note': 'bulk form: one feature row per (position, candidate) pair as SURVEY 8(d) counts it; timed alone between '
                      'two CUDA events with the L2 flushed (256 MB memset) before every iteration, so `us` includes the '
                      'event-pair overhead reported next to it; algorithmic bytes count only the ACR + item-embedding rows, '
                      'the kernel also writes the %d context / metadata / recency / novelty / padding columns of every row'
                      % (plan.Fp - E - Di)}
    # (c) the embedding gather with the table in HBM: a step touches <= 1.5 K distinct rows of the G1 tables, which L2
    # largely keeps between launches.  Same row shape (250 floats, ld 252), but a table far larger than the 50 MB L2 and
    # distinct random ids: every row comes from HBM once and is written once (nar_gather_rows_f32, the kernel behind tf.nn.embedding_lookup nar_model.py:948); plus its gradient scatter-add.
    try:
        Vb, nb_rows = 1 << 20, 1 << 18
        tab = torch.randn(Vb, 252, device='cuda')
        ids = torch.randperm(Vb, device='cuda')[:nb_rows].contiguous()
        outb = torch.empty(nb_rows, 252, device='cuda')
        ms_h = timeit(lambda: ops.gather_rows(tab, ids, outb, 250), iters=10)
        hb = nb_rows * (250 * 4 * 2 + 8)
        gtab = torch.zeros(Vb, 252, device='cuda')
        ms_s = timeit(lambda: ops.scatter_add_rows(gtab, ids, outb, 250), iters=10)
        roof_g['hbm_resident_form'] = {
            'kernel': 'gather_rows_kernel', 'rows': nb_rows, 'table_rows': Vb, 'row_floats': 250, 'us': ms_h * 1e3, 'algorithmic_bytes': hb,
            'achieved': hb / (ms_h * 1e-3) / 1e9, 'frac': hb / (ms_h * 1e-3) / 1e9 / hbm_peak,
            'frac_net_of_event_overhead': hb / (max(ms_h - ms_0, 1e-6) * 1e-3) / 1e9 / hbm_peak,
            'scatter_add': {'kernel': 'scatter_add_rows_kernel', 'us': ms_s * 1e3,
                            'achieved': nb_rows * (250 * 4 * 3 + 8) / (ms_s * 1e-3) / 1e9,      # read src + read-modify-write of the row
                            'frac': nb_rows * (250 * 4 * 3 + 8) / (ms_s * 1e-3) / 1e9 / hbm_peak},
            'note': '1 Mi x 252 fp32 table (1 GB, 20x the L2), 256 Ki distinct random ids: every row comes from HBM'}
        roof_g['frac_hbm_resident_form'] = roof_g['hbm_resident_form']['frac']
        del tab, gtab, outb, ids
    except Exception as ex:  # noqa: BLE001
        roof_g['hbm_resident_form'] = {'error': str(ex)}
    if eng.dedup:
        nb = 2 * L + K * 20 + 1
        rows_b = ops.row_layout(nb, L, 0, n_positive=L, n_full=2 * L, ctx_col0=plan.ctx_col0)
        bp, bi = eng.buffer(st, 'base_pos').view(-1), eng.buffer(st, 'base_item').view(-1)
        Xb = eng.buffer(st, 'X')
        ms_b = timeit(lambda: ops.gather_features(planc, bp, bi, rows_b, t['event_ts'], t['max_ts'], Xb))
        bbytes = nb * ((E + Di) * 4 * 2 + 8)
        roof_g['in_step'] = {'rows': nb, 'us': ms_b * 1e3, 'algorithmic_bytes': bbytes,
                             'achieved': bbytes / (ms_b * 1e-3) / 1e9, 'frac': bbytes / (ms_b * 1e-3) / 1e9 / hbm_peak,
                             'bytes_vs_bulk': bbytes / gbytes,
                             'note': 'the launch the training step makes: clicked + positive rows and ONE row per distinct '
                                     'negative id (exact per-unique-id CAR layer 1); %.1fx fewer bytes than the bulk form' % (gbytes / bbytes)}
    # ---- dominant kernel: CAR layer 2 forward GEMM [R,C]x[C,C], 3xTF32
    H1, Eb = eng.buffer(st, 'H1'), eng.buffer(st, 'E')
    W2, b2, W2lo = eng.view('W2'), eng.view('b2').view(-1), eng.view('W2', eng.params_lo)

    W2plane = ops.pack_bf16x3(W2, eng.C, eng.C)

    def car2(prec):
        if prec == 4:
            ops.gemm(H1, None, Eb, R, eng.C, eng.C, a_kmajor=True, b_kmajor=True, ldb=0, bias=b2, act=ACT_TANH, precision=4,
                     b_bf16=W2plane, ld_bf16=W2plane.stride(0))
        else:
            ops.gemm(H1, W2, Eb, R, eng.C, eng.C, a_kmajor=True, b_kmajor=False, bias=b2, act=ACT_TANH, precision=prec,
                     b_lo=W2lo if prec == 3 else None)
    flops = 2.0 * R * eng.C * eng.C
    ms_3 = timeit(lambda: car2(3), iters=10)
    ms_4 = timeit(lambda: car2(4), iters=10)
    ms_1 = timeit(lambda: car2(1), iters=10)
    used = eng.fwd_prec
    ms_m = ms_4 if used == 4 else ms_3
    # operand bytes TMA brings into shared memory per 128x128 output tile and 32-k tile, times the tiles
    tiles = ((R + 127) // 128) * ((eng.C + 127) // 128) * ((eng.C + 31) // 32)
    roof = {'kernel': ('gemm_kernel<MODE 4: bf16x3, A split in registers, pre-split bf16 weight plane>'
                       if used == 4 else 'gemm_kernel<MODE 2: 3xTF32, A split in registers, B_lo plane from HBM>') +
                      ' (CAR_representation layer 2 forward)', 'bound': 'tensor',
            'achieved': flops / (ms_m * 1e-3) / 1e12, 'peak': tf_peak, 'unit': 'TFLOP/s',
            'frac': flops / (ms_m * 1e-3) / 1e12 / tf_peak,
            'peak_source': peak_src,
            'issued_mma_flops_frac_of_peak': (3.0 * flops / (ms_m * 1e-3) / 1e12) / (tf_peak if used == 4 else tf_peak / 2.0),
            'shape': [R, eng.C, eng.C], 'us': ms_m * 1e3, 'forward_precision': used,
            'smem_ingest_GBps': tiles * (32768 if used == 4 else 49152) / (ms_m * 1e-3) / 1e9,
            'note': 'achieved = algorithmic fp32 FLOPs (2MNK) per second; the kernel issues 3 MMAs per product (error-compensated: '
                    'fp32-grade logits) - tf32 ones at half the bf16 rate (precision 3) or bf16 ones at the full rate (precision 4)',
            'variants_us': {'3xTF32 (precision 3)': ms_3 * 1e3, 'bf16x3 (precision 4)': ms_4 * 1e3, 'single-pass TF32 (precision 1)': ms_1 * 1e3},
            'tf32_single_pass': {'achieved': flops / (ms_1 * 1e-3) / 1e12, 'us': ms_1 * 1e3,
                                 'frac_of_bf16_peak': flops / (ms_1 * 1e-3) / 1e12 / tf_peak}}
    return roof, roof_g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--workload', default='g1')
    ap.add_argument('--profile', default='B', choices=['A', 'B'])
    ap.add_argument('--session-len', default='g1', choices=['g1', 'dense'])
    ap.add_argument('--state-warmup', type=int, default=100)
    ap.add_argument('--cpu-steps', type=int, default=5)
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--dump-outputs', metavar='DIR', default=None,
                    help='after the timed steps, write what the last timed step computed as DIR/<name>.npy')
    ap.add_argument('--global-batch', type=int, default=0,
                    help='sessions per step over ALL ranks (per-GPU batch = this / world); 0 = the workload batch per GPU (weak scaling)')
    args = ap.parse_args()
    # the contract is ONE JSON line on stdout: libraries (NCCL prints its version banner there) get stderr instead
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.fdopen(os.dup(1), 'w')
    os.dup2(2, 1)
    if args.warmup < 3 and args.impl == 'ours':
        args.warmup = 3
    if args.impl == 'reference':
        if args.dump_outputs:
            ap.error('--dump-outputs writes what the CUDA path computed; it does not apply to --impl reference')
        args.warmup = max(1, args.warmup)
        return run_reference(args)
    return run_ours(args)


if __name__ == '__main__':
    sys.exit(main())
