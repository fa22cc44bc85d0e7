"""GPU parity tests (pytest -m gpu): the CUDA path, called through the C ABI (ops.py -> libnar_b200.so),
against the oracle / fp64 references on the same seeded inputs.

Tolerances (north_star): sampled negatives bit-exact; loss and logits within 1e-3 relative.  Gradients are compared at
IDENTICAL leaky_relu slope choices (tools/gpu_step_check.py hands the engine's activation signs to the oracle): a 1e-5
forward difference that flips one pre-activation across the kink moves the oracle's own bias gradients by up to 10 %
(DESIGN.md section 3), which says nothing about either implementation.  Additional bars we
hold ourselves to: feature rows 1e-5, 3xTF32 GEMM 2e-5, TF32 GEMM 3e-3, gradients 3e-2 of the tensor max
(backward GEMMs run single-pass TF32), Adam update within 0.2*lr where the gradient is far above eps.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


def _fails(results):
    return [r for r in results if not r.get('ok')]


@pytest.mark.parametrize('fam', ['gemm_kk', 'gemm_km', 'gemm_mk', 'gemm_mm', 'gemm_epi', 'gemm_bf16'])
def test_gemm_tcgen05(fam):
    """nar_gemm_tf32 (csrc/gemm_wgmma.cu) against fp64 for every operand major, precision and epilogue."""
    from tools import gpu_diag
    assert not _fails(gpu_diag.FAMILIES[fam]())


def test_gather_and_scatter_add_rows():
    from tools import gpu_diag
    assert not _fails(gpu_diag.fam_gather())


def test_sampler_bit_exact_vs_oracle():
    from tools import gpu_diag
    res = gpu_diag.fam_sampler()
    assert all(r['equal'] and r['equal_dp_slice'] for r in res), res


def test_ugrnn_forward_backward():
    from tools import gpu_diag
    assert not _fails(gpu_diag.fam_rnn())


def test_scorer_softmax_ce_mlp_and_cosine():
    from tools import gpu_diag
    assert not _fails(gpu_diag.fam_loss())


def test_dropout_masks_match_spec():
    """nar_dropout_rows draws exactly the bits oracle/dropout_ref.py specifies, for feature rows (tensor ids 1-3 by row
    kind, negatives keyed by position*K + k) and for a fixed tensor id."""
    import torch
    from chameleon_recsys_b200 import ops
    from oracle import dropout_ref
    L, K, F = 7, 5, 24
    n_cand = K + 1
    R = L + L * n_cand
    rs = np.random.RandomState(0)
    pos = np.sort(rs.choice(2000, L, replace=False)).astype(np.int32) + (1 << 20)
    row_pos = np.concatenate([pos, np.repeat(pos, n_cand)]).astype(np.int32)
    x = torch.ones(R, F, device='cuda')
    y = torch.empty_like(x)
    ops.dropout_rows(x, y, R, F, F, torch.from_numpy(row_pos).cuda(), L, n_cand, K, 0, 0.75, 1234567890123, 9)
    got = y.cpu().numpy()
    want = np.zeros((R, F), dtype=bool)
    want[:L] = dropout_ref.keep_mask(1234567890123, 9, 1, pos.astype(np.int64), F, 0.75)
    cand = want[L:].reshape(L, n_cand, F)
    cand[:, 0] = dropout_ref.keep_mask(1234567890123, 9, 2, pos.astype(np.int64), F, 0.75)
    cand[:, 1:] = dropout_ref.keep_mask(1234567890123, 9, 3, pos.astype(np.int64)[:, None] * K + np.arange(K), F, 0.75)
    assert np.array_equal(got != 0, want)
    assert np.allclose(got[want], 1.0 / 0.75)
    z = torch.empty(L, F, device='cuda')
    ops.dropout_rows(x[:L], z, L, F, F, torch.from_numpy(pos).cuda(), 0, 0, 0, 9, 0.5, 42, 3)
    assert np.array_equal(z.cpu().numpy() != 0, dropout_ref.keep_mask(42, 3, 9, pos.astype(np.int64), F, 0.5))


def test_adam_colsum_l2():
    from tools import gpu_diag
    assert not _fails(gpu_diag.fam_misc())


def _check_steps(res, grad_tol=3e-2, update_tol=0.2):
    for s in res['steps']:
        assert s['neg_equal'], 'negatives must be bit-exact'
        assert max(s['x_in'], s['x_pos'], s['x_neg']) < 1e-5, s
        assert max(s['e_in'], s['e_pos'], s['e_neg'], s['rnn'], s['pred']) < 2e-4, s
        assert s['logits_rel_max'] < 1e-3, s
        assert s['xe_rel'] < 1e-3 and s['total_rel'] < 1e-3, s
        assert s['grad_rel_max'] < grad_tol, sorted(s['grad_rel'].items(), key=lambda kv: -kv[1])[:6]
        if s['step'] > 1:          # at t = 1 Adam's update is lr*sign(g): a sign flip of a ~0 gradient is not an error
            assert s['update_err_over_lr'] < update_tol, s


@pytest.mark.parametrize('case', ['tinyA', 'tinyB', 'tinyB_cold', 'tinyB_cos', 'tinyB_2l', 'tinyB_nov', 'tinyB_cos_nov', 'tinyB_drop',
                                  'tinyB_2l_drop', 'tinyB_pad', 'tinyB_gru', 'tinyB_gru_2l_drop', 'tinyB_gru_cos', 'tinyB_bf16',
                                  'tinyA_bf16', 'tinyB_gru_bf16'])
def test_full_step_parity_tiny(case):
    import torch
    from tools import gpu_step_check as g
    cfg = {'tinyA': ('A', 5, 3, None), 'tinyB': ('B', 5, 3, None), 'tinyB_cold': ('B', 0, 2, None),
           'tinyB_cos': ('B', 5, 2, dict(ranking='cosine')), 'tinyB_2l': ('B', 5, 2, dict(rnn_num_layers=2)),
           # novelty regulariser (nar_model.py:673-683) and dropout (:338-340, :417-419, :1330-1333)
           'tinyB_nov': ('B', 5, 2, dict(novelty_reg_factor=0.5)),
           'tinyB_cos_nov': ('B', 5, 2, dict(ranking='cosine', novelty_reg_factor=0.5)),
           'tinyB_drop': ('B', 5, 2, dict(dropout_keep_prob=0.8)),
           'tinyB_2l_drop': ('B', 5, 2, dict(rnn_num_layers=2, dropout_keep_prob=0.7)),
           # two sessions, empty buffer: the candidate pool runs out, negatives are zero padded (the padding slot of
           # the per-unique-id layer 1 and its backward segment sum)
           'tinyB_pad': ('B', 0, 2, dict(batch_size=2)),
           # rnn_cell='gru' (north_star's "session GRU"; nar_model.py:1315)
           'tinyB_gru': ('B', 5, 3, dict(rnn_cell='gru')),
           'tinyB_gru_2l_drop': ('B', 5, 2, dict(rnn_cell='gru', rnn_num_layers=2, dropout_keep_prob=0.8)),
           'tinyB_gru_cos': ('B', 5, 2, dict(rnn_cell='gru', ranking='cosine')),
           # forward GEMMs as bf16x3 (fwd_precision 4)
           'tinyB_bf16': ('B', 5, 3, None), 'tinyA_bf16': ('A', 5, 2, None), 'tinyB_gru_bf16': ('B', 5, 2, dict(rnn_cell='gru'))}[case]
    # the two-layer dropout case checks the mask plumbing (which output is dropped where, forward and backward): it runs
    # the backward GEMMs error-compensated so that a wrong mask cannot hide in TF32 noise
    ekw = dict(bwd_precision=3) if case in ('tinyB_2l_drop', 'tinyB_gru_2l_drop') else None
    if case.endswith('_bf16'):
        ekw = dict(fwd_precision=4)
    res = g.run_case('tiny', cfg[0], cfg[1], cfg[2], hp_over=cfg[3], oracle_dtype=torch.float64, engine_kw=ekw)
    # (5 positions in the padding case: Adam turns the TF32 noise of near-zero gradients into larger relative updates)
    _check_steps(res, grad_tol=2e-3 if (ekw and 'bwd_precision' in ekw) else 3e-2, update_tol=0.5 if case == 'tinyB_pad' else 0.2)


@pytest.mark.parametrize('case', ['tinyB', 'tinyB_cold', 'g1'])
def test_full_step_parity_every_candidate_row(case):
    """dedup=False: every candidate row gathered and multiplied by W1 (the layout dropout will need) - same bars."""
    import torch
    from tools import gpu_step_check as g
    if case == 'g1':
        res = g.run_case('g1', 'B', 30, 2, hp_over=dict(batch_size=48), oracle_dtype=torch.float32, engine_kw=dict(dedup=False))
    else:
        res = g.run_case('tiny', 'B', 0 if case == 'tinyB_cold' else 5, 2, oracle_dtype=torch.float64, engine_kw=dict(dedup=False))
    _check_steps(res)


def test_dedup_matches_every_candidate_row():
    """The per-unique-id CAR layer 1 is exact: same logits / loss as the path that materialises every candidate row, to
    fp32 summation order (3xTF32 forward); gradients agree to the TF32 backward noise; run twice: bit-reproducible."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools import gpu_step_check as g
    pb = make_problem('g1', profile='B', batch_size=64)
    warm_state(pb, 10)
    f, l = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32)
    logical = pb.layout.init_logical(5)
    res = {}
    for dd in (False, True, True):
        eng = g.make_engine(pb, dedup=dd)
        eng.set_params(logical)
        st = eng.stage(f, l, buf, pop)
        eng.step(st, train=True, keep=True)
        torch.cuda.synchronize()
        res.setdefault(dd, []).append((eng.last['logits'].clone(), eng.loss_dev.clone(), eng.grads.clone(), eng.last['E'].clone()))
    (lg0, ls0, g0, e0), (lg1, ls1, g1, e1), (lg2, ls2, g2, e2) = res[False][0], res[True][0], res[True][1]
    assert float((e0 - e1).abs().max()) < 2e-5
    assert float((lg0 - lg1).abs().max()) / float(lg0.abs().max()) < 2e-5
    assert abs(float(ls0[0]) - float(ls1[0])) / float(ls0[0]) < 1e-5
    scale = float(g0.abs().max())
    assert float((g0 - g1).abs().max()) / scale < 2e-2
    assert torch.equal(lg1, lg2) and torch.equal(e1, e2)            # forward: no atomics anywhere


@pytest.mark.parametrize('fwd', [3, 4])
def test_full_step_parity_g1_shapes(fwd):
    """G1 dims (46K items, E=250, H=255, C=1024, K=50, F=477) at a batch the fp32 oracle finishes in seconds; forward GEMMs
    as 3xTF32 (fwd 3) and as bf16x3 (fwd 4)."""
    import torch
    from tools import gpu_step_check as g
    res = g.run_case('g1', 'B', 30, 2, hp_over=dict(batch_size=48), oracle_dtype=torch.float32, engine_kw=dict(fwd_precision=fwd))
    _check_steps(res, update_tol=0.3)      # 76 positions: Adam's +-lr on near-zero gradients weighs more than at full batch


def test_full_step_parity_g1_full_batch():
    """BASELINE configs[1] at its REAL size (batch 256, seq <= 20, K 50, 46K items): one full step vs the fp32 oracle
    (the oracle needs ~3 s for it)."""
    import torch
    from tools import gpu_step_check as g
    res = g.run_case('g1', 'B', 30, 1, oracle_dtype=torch.float32)
    assert res['steps'][0]['B'] == 256
    _check_steps(res)


@pytest.mark.parametrize('bwd', [1, 3])
def test_unsynced_trajectory_g1(bwd):
    """30 steps WITHOUT reloading the oracle's state into the engine: each side follows its own Adam trajectory.  The
    loss must stay within 1e-3 relative at every step - the test that says whether single-pass TF32 backward GEMMs
    (bwd=1; the reference's gradients are fp32) are acceptable; bwd=3 (3xTF32 backward) is the control."""
    import torch
    from tools import gpu_step_check as g
    res = g.run_trajectory('g1', 'B', 30, 30, hp_over=dict(batch_size=64), oracle_dtype=torch.float32,
                           engine_kw=dict(bwd_precision=bwd))
    assert all(s['neg_equal'] for s in res['steps'])
    assert res['max_rel'] < 1e-3, [(s['step'], s['rel']) for s in res['steps'] if s['rel'] >= 1e-3]


def test_nccl_two_ranks_match_single():
    """Real NCCL: a 2-rank data-parallel run (torchrun, one rank per GPU) reproduces the 1-rank run of the same global
    batch - negatives bit-exact, loss within 1e-5, all-reduced gradient within the TF32 backward noise (3e-3 of its max), weights within Adam's
    +-lr noise on near-zero gradients.  Needs 2 GPUs (skipped on a 1-GPU machine)."""
    import json
    import subprocess
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', '29617', os.path.join(ROOT, 'tools', 'nccl_equiv.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [x for x in r.stdout.splitlines() if x.startswith('NCCL_EQUIV ')][-1]
    res = json.loads(line[len('NCCL_EQUIV '):])
    assert res['negatives_equal']
    assert res['loss_rel_max'] < 1e-5 and res['reg_rel_max'] < 1e-5, res
    # the all-reduced gradient differs by the TF32 backward noise: each rank truncates ITS partial sums (per-unique-id
    # segment sums, split-K partials) to tf32 before the next GEMM, so sharding changes what gets truncated: ~2^-11
    assert res['grad_rel_max_last_step'] < 3e-3, res
    assert res['param_diff_median'] < 1e-6 and res['param_diff_max'] <= 2.5 * res['steps'] * res['lr'], res


@pytest.mark.parametrize('wl', ['adressa', 'stress'])
def test_full_step_parity_other_baseline_shapes(wl):
    """BASELINE configs[2] (Adressa-shaped: 13K items, K 100, seq <= 30, 5000 from the buffer) and configs[4] (stress: 1M
    items, E 512, H 512, K 500) at a batch the fp32 oracle finishes in seconds: one full step, same bars."""
    import torch
    from tools import gpu_step_check as g
    if wl == 'adressa':
        res = g.run_case('adressa', 'B', 20, 1, hp_over=dict(batch_size=32), oracle_dtype=torch.float32)
    else:
        res = g.run_case('stress', 'B', 4, 1, hp_over=dict(batch_size=8), oracle_dtype=torch.float32)
    _check_steps(res)


def test_full_size_properties_g1():
    """BASELINE config[1] at full size over several steps: size-independent properties of every step."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine
    pb = make_problem('g1', profile='B')
    warm_state(pb, 20)
    eng = make_engine(pb)
    eng.set_params(pb.layout.init_logical(42))
    it = pb.input_fn()
    losses = []
    for i in range(4):
        f, l = it.get_next()
        buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
        pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
        out = eng.train_step(f, l, buf, pop, keep=True)
        neg = out['negatives'].cpu().numpy()
        allc = np.concatenate([f['item_clicked'], l['label_last_item']], axis=1)
        T = f['item_clicked'].shape[1]
        mask = np.arange(T)[None, :] < (f['session_size'] - 1)[:, None]
        assert not neg[~mask].any()                                   # padded clicks -> all-zero rows
        for b in range(0, neg.shape[0], 17):
            for p in range(T):
                row = neg[b, p][neg[b, p] != 0]
                assert len(set(row)) == len(row)                      # unique per click
                assert not set(row) & set(allc[b])                     # session items excluded
        lg = eng.last['logits']
        p = torch.softmax(lg, -1)
        assert torch.allclose(p.sum(-1), torch.ones_like(p[:, 0]), atol=1e-5)
        xe = -(torch.log_softmax(lg.double(), -1)[:, 0]).mean().item()
        assert abs(xe - out['xe_loss']) / xe < 1e-5                   # fused CE == log-softmax of the stored logits
        assert np.isfinite(out['total_loss'])
        losses.append(out['total_loss'])
        # padded H columns of the RNN state stay exactly zero (H=255 -> 256)
        assert float(eng.last['HO'][-1][:, pb.hp.rnn_units:].abs().max()) == 0.0
    flat = eng.params.cpu().numpy()
    logical = pb.layout.to_logical(flat)
    assert np.count_nonzero(flat) <= sum(v.size for v in logical.values())    # layout padding still zero after Adam


def test_two_process_data_parallel_matches_single():
    """1-vs-2 rank equivalence of the data-parallel step on ONE GPU (two ranks share cuda:0, NCCL needs 2 devices,
    so the collective here is gloo on CPU tensors is not available for CUDA -> emulate: run both shards in one process
    and sum the gradients; negatives and loss must equal the single-process global batch)."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 5)
    f, l = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    logical = pb.layout.init_logical(42)
    e1 = make_engine(pb); e1.set_params(logical)
    st = e1.stage(f, l, buf, pop); e1.grads.zero_(); o1 = e1.step(st, train=True)
    g_full = e1.grads.clone(); neg_full = o1['negatives'].clone(); loss_full = e1.loss_dev.clone()
    gsum = torch.zeros_like(g_full); loss_sum = torch.zeros_like(loss_full); negs = []
    for r in range(2):
        e = make_engine(pb); e.set_params(logical)
        e.world, e.rank = 2, r                    # shard selection + loss normaliser use (world, rank) only
        st = e.stage(f, l, buf, pop); e.grads.zero_(); o = e.step(st, train=True)
        gsum += e.grads; loss_sum += e.loss_dev; negs.append(o['negatives'].clone())
    assert torch.equal(torch.cat(negs, 0), neg_full)
    assert abs(loss_sum[0].item() - loss_full[0].item()) / loss_full[0].item() < 1e-5
    assert abs(loss_sum[1].item() - loss_full[1].item()) / max(loss_full[1].item(), 1e-12) < 1e-5
    scale = g_full.abs().max().item()
    assert (gsum - g_full).abs().max().item() / scale < 2e-3


def test_eval_ranking_and_metrics_vs_oracle():
    """ModeKeys.EVAL: predicted_item_ids / probs (tf.nn.top_k order) and the HR@n / MRR@n sums against the oracle.
    Ranks are compared where the oracle's probability gaps exceed the forward tolerance (a 1e-5 logit difference may
    swap two near-tied candidates, which is not an error); the streaming sums must agree to within those swaps."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from oracle import sampler_ref
    from tools import gpu_step_check as g
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 5)
    hp = pb.hp
    eng = g.make_engine(pb)
    orc = g.make_oracle(pb, torch.float64)
    logical = pb.layout.init_logical(7)
    eng.set_params(logical); orc.set_params(logical)
    it = pb.input_fn()
    top_n = 3
    metrics = torch.zeros(3, device='cuda', dtype=torch.float64)
    tot = np.zeros(3)
    for step in range(3):
        f, l = it.get_next()
        buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
        pop = pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32)
        out = eng.eval_step(f, l, buf, pop, top_n=top_n, metrics=metrics, step_id=step + 1)
        allc = np.concatenate([f['item_clicked'], l['label_last_item']], axis=1)
        neg = sampler_ref.sample_negatives(allc, buf, hp.train_total_negative_samples, hp.train_negative_samples_from_buffer,
                                           hp.sampler_seed, step + 1)
        assert np.array_equal(out['negatives'].cpu().numpy(), neg)
        o = orc.forward(f, l, neg, buf, pop)
        ids, probs, hits, rr, cnt = orc.rank_and_metrics(o, l, neg, top_n)
        tot += [hits, rr, cnt]
        mask = o['mask'].cpu().numpy().astype(bool)
        gp = out['predicted_item_probs'].cpu().numpy(); gi = out['predicted_item_ids'].cpu().numpy()
        op, oi = probs[mask], ids[mask]                               # valid positions, session-major == engine row order
        assert gp.shape == op.shape
        assert np.abs(gp - op).max() < 1e-4
        assert (np.diff(gp, axis=1) <= 0).all()                        # sorted, descending
        gap_ok = np.ones_like(op, dtype=bool)
        gap = np.abs(np.diff(op, axis=1)) > 1e-4
        gap_ok[:, 1:] &= gap; gap_ok[:, :-1] &= gap                    # both neighbours clearly separated
        assert (gi[gap_ok] == oi[gap_ok]).all()
        assert abs(out['total_loss'] - float(o['total_loss'])) / abs(float(o['total_loss'])) < 1e-3
    m = metrics.cpu().numpy()
    assert m[2] == tot[2]
    assert abs(m[0] - tot[0]) <= 1 and abs(m[1] - tot[1]) <= 0.5        # at most one near-tie swap at the top_n boundary


def test_estimator_evaluate_roundtrip():
    """Estimator.train then Estimator.evaluate (nar_trainer_gcom.py:511-530): EVAL shares the trained weights, returns
    finite metrics in [0,1], leaves the weights untouched and restores ClickedItemsState (hook begin/end)."""
    import torch
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 5)
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, pb.hp, pb.clicked_items_state)
    est.train(lambda: pb.input_fn(), steps=4)
    w0 = est.model.engine.params.clone()
    buf0 = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    res = est.evaluate(lambda: pb.input_fn(), steps=3)
    assert set(res) >= {'loss', 'hitrate_at_n', 'mrr_at_n', 'global_step'}
    assert np.isfinite(res['loss']) and 0.0 <= res['mrr_at_n'] <= res['hitrate_at_n'] <= 1.0
    assert res['global_step'] == 4
    assert torch.equal(w0, est.model.engine.params)
    assert np.array_equal(buf0, pb.clicked_items_state.get_recent_clicks_buffer())
    k_eval = pb.hp.eval_total_negative_samples
    assert est._eval_spec.model.predicted_item_ids.shape[1] == 1 + k_eval


def test_device_resident_state_training_loop(monkeypatch):
    """Estimator.train with the recent-clicks state in HBM (default) == the loop with the hook's host update and per-step
    upload: same negatives (so same buffer at every step), same losses to float-atomics noise, identical host state
    afterwards (buffer, popularity counters, float64 pop-norm), and a smaller per-step H2D copy."""
    import copy
    import torch
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state
    runs = {}
    for mode in ('1', '0'):
        monkeypatch.setenv('NAR_DEVICE_STATE', mode)
        pb = make_problem('tiny', profile='B')
        warm_state(pb, 5)
        est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                              pb.session_features_config, pb.hp, pb.clicked_items_state)
        losses = []
        for rep in range(2):                                     # two train() calls: attach / detach twice
            it = pb.input_fn()
            est.train(lambda: it, steps=6)
            losses.append(est.last_loss)
        st = pb.clicked_items_state
        runs[mode] = (losses, est.model.engine.params.clone(), copy.deepcopy(st.pop_recent_clicks_buffer),
                      st.get_articles_recent_pop_norm().copy(), st.get_articles_pop().copy(), est.h2d_bytes_per_step)
    a, b = runs['1'], runs['0']
    for x, y in zip(a[0], b[0]):
        assert abs(x - y) / abs(y) < 1e-4
    # (two runs of the SAME loop differ by Adam's +-lr on near-zero gradients - float atomics order; 12 steps at lr 1e-4)
    assert float((a[1] - b[1]).abs().median()) < 2e-5
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]) and np.array_equal(a[4], b[4])
    assert a[5] < b[5]


def test_checkpoint_resume_matches_uninterrupted_run(tmp_path):
    """A checkpoint restores weights, TF-Adam slots, step and host state EXACTLY; training on from it tracks the run
    that was never interrupted (to float-atomics noise: Adam turns a +-1e-12 "zero" gradient into a +-lr update, so
    single entries differ by O(lr) between ANY two runs)."""
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state

    def fresh():
        pb = make_problem('tiny', profile='B')
        warm_state(pb, 5)
        it = pb.input_fn()
        return pb, [it.get_next() for _ in range(4)]

    def estimator(pb, model_dir):
        return build_estimator(model_dir, pb.content_article_embeddings_matrix, pb.articles_metadata,
                               pb.articles_features_config, pb.session_features_config, pb.hp, pb.clicked_items_state)

    d = str(tmp_path / 'model')
    pb_a, batches = fresh()
    est_a = estimator(pb_a, d)
    est_a.train(lambda: iter(batches[:2]))                              # 2 steps, checkpoint written at the end
    assert ckpt.latest_checkpoint(d).endswith('model.ckpt-2.npz')
    pb_b, batches_b = fresh()                                           # "new process": fresh weights and host state
    est_b = estimator(pb_b, d)
    est_b._ensure_spec(*batches_b[2])                                   # builds the model and restores model.ckpt-2
    ea, eb = est_a.model.engine, est_b.model.engine
    assert eb.global_step == 2
    assert torch.equal(ea.params, eb.params) and torch.equal(ea.adam_m, eb.adam_m) and torch.equal(ea.adam_v, eb.adam_v)
    assert torch.equal(ea.params_lo, eb.params_lo)
    sa, sb = pb_a.clicked_items_state, pb_b.clicked_items_state
    assert np.array_equal(sa.get_recent_clicks_buffer(), sb.get_recent_clicks_buffer())
    assert np.array_equal(sa.get_articles_recent_pop_norm(), sb.get_articles_recent_pop_norm())
    assert np.array_equal(sa.get_articles_pop(), sb.get_articles_pop())
    est_a.train(lambda: iter(batches[2:]))                              # the uninterrupted run goes on
    est_b.train(lambda: iter(batches_b[2:]))                            # the restored one too
    assert eb.global_step == 4 and ea.global_step == 4
    assert abs(est_b.last_loss - est_a.last_loss) / abs(est_a.last_loss) < 1e-3
    dp = (ea.params - eb.params).abs()
    assert float(dp.median()) < 1e-6
    assert np.array_equal(sa.get_recent_clicks_buffer(), sb.get_recent_clicks_buffer())
    assert ckpt.latest_checkpoint(d).endswith('model.ckpt-4.npz')


def test_aux_stream_gradients_match_single_stream():
    """Weight / bias gradients computed on the auxiliary stream (engine._on_aux) equal the single-stream ones: any
    missing event or reused buffer would show up as a difference far above the float-atomics noise."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools import gpu_step_check as g
    pb = make_problem('g1', profile='B', batch_size=64)
    warm_state(pb, 10)
    it = pb.input_fn()
    batches = []
    for _ in range(3):
        f, l = it.get_next()
        batches.append((f, l, pb.clicked_items_state.get_recent_clicks_buffer().copy(),
                        pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32)))
    logical = pb.layout.init_logical(3)
    grads = {}
    for aux in (False, True):
        eng = g.make_engine(pb)
        eng.use_aux_stream = aux
        eng.set_params(logical)
        outs = []
        for rep in range(2):                                            # twice: races are not deterministic
            for f, l, buf, pop in batches:
                st = eng.stage(f, l, buf, pop)
                eng.grads.zero_()
                eng.step(st, train=True)
                torch.cuda.synchronize()
                outs.append(eng.grads.clone())
        grads[aux] = outs
    for a, b in zip(grads[False], grads[True]):
        scale = float(a.abs().max())
        assert float((a - b).abs().max()) <= 2e-5 * scale, (float((a - b).abs().max()), scale)
    for i in range(3):                                                  # and run to run
        assert float((grads[True][i] - grads[True][i + 3]).abs().max()) <= 2e-5 * float(grads[True][i].abs().max())
