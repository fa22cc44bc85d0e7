"""rnn_residual_connections=True on the GPU (pytest -m gpu): the residual session stack (DESIGN.md section 15) through the
training step, EVAL, PREDICT and checkpoints, against the oracle (oracle/residual_ref.py) at the bars of
tests/test_gpu_parity.py.  rnn_units is 48 at the tiny shape (padded to 64) and 255 at G1 (padded to 256), so the padded
columns of the projection and of every layer's output are part of every case."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

CELLS = ('ugrnn', 'gru', 'lstm')
RES = dict(rnn_residual_connections=True)
TINY = dict(RES, rnn_units=48)


def _check_steps(res, grad_tol=3e-2, update_tol=0.2):
    """The bars of tests/test_gpu_parity.py::_check_steps."""
    for s in res['steps']:
        assert s['neg_equal'], 'negatives must be bit-exact'
        assert max(s['x_in'], s['x_pos'], s['x_neg']) < 1e-5, s
        assert max(s['e_in'], s['e_pos'], s['e_neg'], s['rnn'], s['pred']) < 2e-4, s
        assert s['logits_rel_max'] < 1e-3, s
        assert s['xe_rel'] < 1e-3 and s['total_rel'] < 1e-3, s
        assert s['grad_rel_max'] < grad_tol, sorted(s['grad_rel'].items(), key=lambda kv: -kv[1])[:6]
        if s['step'] > 1:
            assert s['update_err_over_lr'] < update_tol, s


@pytest.mark.parametrize('keep_prob', [1.0, 0.8])
@pytest.mark.parametrize('layers', [1, 2, 4])
@pytest.mark.parametrize('cell', CELLS)
def test_full_step_parity_tiny(cell, layers, keep_prob):
    import torch
    from tools import gpu_step_check as g
    res = g.run_case('tiny', 'B', 5, 2, hp_over=dict(TINY, rnn_cell=cell, rnn_num_layers=layers, dropout_keep_prob=keep_prob),
                     oracle_dtype=torch.float64)
    assert res['steps'][0]['L'] > 0
    assert all(k in res['steps'][0]['grad_rel'] for k in ('input_projection_wrapper/kernel', 'input_projection_wrapper/bias'))
    _check_steps(res)


@pytest.mark.parametrize('cell', CELLS)
def test_full_step_parity_g1(cell):
    """G1 at batch 48, rnn_units 255 (Hp 256), against the fp32 oracle."""
    import torch
    from tools import gpu_step_check as g
    res = g.run_case('g1', 'B', 30, 2, hp_over=dict(RES, batch_size=48, rnn_cell=cell), oracle_dtype=torch.float32)
    assert res['steps'][0]['L'] > 0
    _check_steps(res, update_tol=0.3)


def test_switch_off_issues_the_parent_launches():
    """The residual launches sit behind the switch: a plain stack issues the same number of launches per step whatever
    the other settings, and the residual stack adds a fixed number (the projection, one residual add per layer, the
    projection's dgrad and its weight and bias gradients)."""
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine
    counts = {}
    for res in (False, True):
        pb = make_problem('tiny', profile='B', rnn_num_layers=2, rnn_residual_connections=res)
        warm_state(pb, 3)
        eng = make_engine(pb)
        eng.set_params(pb.layout.init_logical(1))
        f, l = pb.input_fn().get_next()
        st = pb.clicked_items_state
        eng.train_step(f, l, st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy())
        n0 = eng.launches
        eng.train_step(f, l, st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy())
        counts[res] = eng.launches - n0
    # forward: P GEMM + 2 adds; backward: the Wp dgrad, its wgrad and bias sum (the layer dgrads are replaced, not added)
    assert counts[True] - counts[False] == 1 + 2 + 3, counts


def test_eval_ranking_and_metrics_vs_oracle():
    """ModeKeys.EVAL with two residual layers: ranked ids / probabilities and the HR@n / MRR@n sums against the oracle
    (ranks compared where the oracle's probability gaps exceed the forward tolerance)."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from oracle import sampler_ref
    from tools import gpu_step_check as g
    pb = make_problem('tiny', profile='B', rnn_num_layers=2, **TINY)
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
        op, oi = probs[mask], ids[mask]
        assert gp.shape == op.shape
        assert np.abs(gp - op).max() < 1e-4
        gap_ok = np.ones_like(op, dtype=bool)
        gap = np.abs(np.diff(op, axis=1)) > 1e-4
        gap_ok[:, 1:] &= gap; gap_ok[:, :-1] &= gap
        assert (gi[gap_ok] == oi[gap_ok]).all()
        assert abs(out['total_loss'] - float(o['total_loss'])) / abs(float(o['total_loss'])) < 1e-3
    m = metrics.cpu().numpy()
    assert m[2] == tot[2]
    assert abs(m[0] - tot[0]) <= 1 and abs(m[1] - tot[1]) <= 0.5


def _estimator(pb, model_dir):
    from chameleon_recsys_b200.estimator import build_estimator
    return build_estimator(model_dir, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                           pb.session_features_config, pb.hp, pb.clicked_items_state, device=0)


def _trained(tmp_path, cell='ugrnn', steps=3, **hp):
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B', rnn_cell=cell, batch_size=24, rnn_num_layers=2, **dict(TINY, **hp))
    warm_state(pb, 5)
    est = _estimator(pb, str(tmp_path))
    est.train(pb.input_fn, steps=steps)
    return pb, est


@pytest.mark.parametrize('cell', CELLS)
def test_predict_reproduces_eval_logits(cell, tmp_path):
    """After Estimator.train: the EVAL logits of a batch's 1+K sampled candidates per position, and recommend over their
    union (the path Estimator.predict runs) gives every one of them within 1e-4 of the largest."""
    pb, est = _trained(tmp_path, cell)
    eng = est.model.engine
    feats, labels = pb.input_fn().get_next()
    st = pb.clicked_items_state
    buf, pop = st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy()
    out = eng.eval_step(feats, labels, buf, pop, top_n=3)
    L, n_cand = out['stage']['L'], eng.K + 1
    lg = out['logits'].cpu().numpy().reshape(L, n_cand)
    ids = eng.buffer(out['stage'], 'row_item').view(-1)[L:L + L * n_cand].cpu().numpy().reshape(L, n_cand)
    cand = np.unique(ids[ids != 0])
    rec = eng.recommend(feats, buf, pop, cand.size, candidates=cand, positions='all', exclude_session_clicks=False)
    tol = 1e-4 * np.abs(lg).max()
    for q in range(L):
        score = dict(zip(rec['predicted_item_ids'][q].tolist(), rec['predicted_item_scores'][q].tolist()))
        for j in range(n_cand):
            if ids[q, j]:
                assert abs(score[int(ids[q, j])] - lg[q, j]) <= tol, (q, j)


def test_estimator_predict_vs_oracle(tmp_path):
    """Estimator.predict (top-n over the catalog after every session's last position) against the every-row oracle with
    the trained weights."""
    import torch
    from oracle.recommend_ref import recommend
    from tools.gpu_step_check import make_oracle
    pb, est = _trained(tmp_path)
    batch = pb.input_fn().get_next()
    st = pb.clicked_items_state
    buf, pop = st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy()
    preds = list(est.predict(lambda: iter([batch]), top_n=10, candidates='catalog'))
    orc = make_oracle(pb, torch.float64)
    orc.set_params(est.model.engine.get_params())
    ref = recommend(orc, batch[0], buf, pop, 'catalog', 10, positions='last', exclude_session_clicks=True)
    assert len(preds) == ref['predicted_item_ids'].shape[0]
    column = {int(c): i for i, c in enumerate(ref['candidates'])}
    tol = 1e-3 * np.abs(ref['scores']).max()
    for q, p in enumerate(preds):
        ids = p['predicted_item_ids']
        real = ids != 0
        assert np.array_equal(real, ref['predicted_item_ids'][q] != 0)
        assert np.abs(p['predicted_item_scores'][real] - ref['scores'][q, [column[int(i)] for i in ids[real]]]).max() <= tol


def test_checkpoint_round_trip_and_cross_setting_restore(tmp_path):
    """save -> a fresh Estimator -> restore gives the same predictions; the checkpoint holds the projection under its TF
    names; restoring it into a plain stack (and a plain checkpoint into a residual stack) raises, naming a missing
    variable, and leaves the engine's weights untouched."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb, est = _trained(tmp_path / 'a')
    path = est.save_checkpoint(str(tmp_path / 'res.npz'))
    names = set(np.load(path).files)
    for n in ('input_projection_wrapper/kernel', 'input_projection_wrapper/bias', 'input_projection_wrapper/ugrnn_cell/kernel',
              'cell_1/ugrnn_cell/kernel'):
        assert 'params/main/RNN/rnn/multi_rnn_cell/' + ('' if n.startswith('cell_1') else 'cell_0/') + n in names, n
    batch = pb.input_fn().get_next()
    st = pb.clicked_items_state
    buf, pop = st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy()
    want = est.model.engine.recommend(batch[0], buf, pop, 10, candidates='catalog')

    def fresh(res):
        p = make_problem('tiny', profile='B', batch_size=24, rnn_num_layers=2, **dict(TINY, rnn_residual_connections=res))
        warm_state(p, 5)
        e = _estimator(p, str(tmp_path / ('b%d' % res)))
        e._ensure_spec(*p.input_fn().get_next())
        return e

    est_b = fresh(True)
    assert est_b.restore_checkpoint(path) == est.model.engine.global_step
    got = est_b.model.engine.recommend(batch[0], buf, pop, 10, candidates='catalog')
    assert np.array_equal(got['predicted_item_ids'], want['predicted_item_ids'])
    assert np.array_equal(got['predicted_item_scores'], want['predicted_item_scores'])

    est_c = fresh(False)
    before = est_c.model.engine.params.clone()
    with pytest.raises(KeyError, match='cell_0/ugrnn_cell/kernel'):
        est_c.restore_checkpoint(path)
    assert torch.equal(est_c.model.engine.params, before)
    plain = est_c.save_checkpoint(str(tmp_path / 'plain.npz'))
    before = est_b.model.engine.params.clone()
    with pytest.raises(KeyError, match='input_projection_wrapper'):
        est_b.restore_checkpoint(plain)
    assert torch.equal(est_b.model.engine.params, before)


@pytest.mark.parametrize('cell', CELLS)
def test_padded_columns_stay_zero(cell):
    """After 3 Adam steps the padded columns H..Hp of Wp, bp, P and every layer's output HR are exactly 0, and the
    residual outputs are HO + the layer input."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine
    pb = make_problem('tiny', profile='B', rnn_cell=cell, rnn_num_layers=2, **TINY)
    warm_state(pb, 5)
    eng = make_engine(pb)
    eng.set_params(pb.layout.init_logical(3))
    H, Hp = pb.layout.H, pb.layout.Hp
    assert (H, Hp) == (48, 64)
    it = pb.input_fn()
    st = pb.clicked_items_state
    for _ in range(3):
        f, l = it.get_next()
        eng.train_step(f, l, st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy(), keep=True)
        st.update_from_batch(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
    assert eng.global_step == 3
    torch.cuda.synchronize()
    Wp, bp = eng.view('rnn0/Wp'), eng.view('rnn0/bp')
    assert Wp[:, :H].abs().max() > 0 and not Wp[:, H:].any() and not bp[:, H:].any()
    for buf in (eng.adam_m, eng.adam_v):
        assert not eng.view('rnn0/Wp', buf)[:, H:].any() and not eng.view('rnn0/bp', buf)[:, H:].any()
    f, l = it.get_next()
    out = eng.eval_step(f, l, st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy(), top_n=3)
    L = out['stage']['L']
    for n in ('P', 'HR0', 'HR1'):
        b = eng.buffer(out['stage'], n)[:L]
        assert b[:, :H].abs().max() > 0 and not b[:, H:].any(), n


def test_padded_buffers_and_residual_sum():
    """P, HR0, HR1 of an EVAL step: zero padded columns, HR0 = HO0 + P and HR1 = HO1 + HR0 exactly (fp32 adds)."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine
    pb = make_problem('tiny', profile='B', rnn_num_layers=2, **TINY)
    warm_state(pb, 5)
    eng = make_engine(pb)
    eng.set_params(pb.layout.init_logical(3))
    st = pb.clicked_items_state
    f, l = pb.input_fn().get_next()
    out = eng.eval_step(f, l, st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy(), top_n=3)
    s = out['stage']
    L, H = s['L'], pb.layout.H
    b = {n: eng.buffer(s, n)[:L].clone() for n in ('P', 'HO0', 'HO1', 'HR0', 'HR1')}
    for n in ('P', 'HO0', 'HO1', 'HR0', 'HR1'):
        assert not b[n][:, H:].any(), n
    assert b['P'][:, :H].abs().max() > 0
    assert torch.equal(b['HR0'], b['HO0'] + b['P'])
    assert torch.equal(b['HR1'], b['HO1'] + b['HR0'])
