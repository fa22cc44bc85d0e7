"""Data-parallel prediction on the GPU (pytest -m gpu): NarEngine.recommend and Estimator.predict over a process group
return on every rank, bit for bit, what one process returns (tools/predict_dp_check.py holds the checks).  2 and 3
processes share cuda:0 over gloo, so this runs on a one-GPU machine; the same checks over NCCL with one rank per GPU
run when there are two GPUs."""
import os
import subprocess
import sys
import traceback

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

TIMEOUT_S = 900


def _worker(rank, world, port, model_dir, queue):
    try:
        os.environ['NAR_WS_BUDGET_GB'] = '2'          # several engines per process, several processes on one device
        sys.path.insert(0, ROOT)
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(0)
        dist.init_process_group('gloo', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world)
        try:
            from tools.predict_dp_check import run_checks
            res = run_checks(dist.group.WORLD, rank, world, 0, model_dir)
        finally:
            dist.destroy_process_group()
        queue.put((rank, 'ok', res))
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test
        queue.put((rank, 'error', traceback.format_exc()))


@pytest.mark.parametrize('world', [2, 3])
def test_recommend_and_predict_match_one_process_gloo(world, tmp_path):
    import queue as _queue

    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 23000 + (os.getpid() % 3000) + 11 * world
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path), q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        while len(got) < world:
            try:
                rank, status, res = q.get(timeout=TIMEOUT_S)
            except _queue.Empty:
                pytest.fail('workers did not finish within %d s (done: %s)' % (TIMEOUT_S, sorted(got)))
            got[rank] = (status, res)
            if status != 'ok':
                pytest.fail('rank %d failed:\n%s' % (rank, res))
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:                                # no worker outlives the test
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = [got[r][1] for r in range(world)]
    assert all(r == res[0] for r in res)               # every rank saw the same query counts
    assert res[0]['one_session'][0] == 1 and res[0]['no_session'] == [0, 0]


def test_recommend_and_predict_match_one_process_nccl(tmp_path):
    """The same checks over NCCL, one rank per GPU (torchrun).  Needs 2 GPUs (skipped on a 1-GPU machine)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', '29631', os.path.join(ROOT, 'tools', 'predict_dp_check.py'), str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=TIMEOUT_S, cwd=ROOT,
                       env=dict(os.environ, NAR_WS_BUDGET_GB='2'))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert any(x.startswith('PREDICT_DP_CHECK ') for x in r.stdout.splitlines()), r.stdout[-3000:]
