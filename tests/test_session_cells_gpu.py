"""rnn_cell='gru' and 'lstm' on the GPU (pytest -m gpu): the whole training / EVAL / PREDICT / checkpoint path against the
oracle (oracle/nar_oracle.py, oracle/lstm_ref.py) at the bars of tests/test_gpu_parity.py, at the tiny, G1 and Adressa
shapes.  The recurrence kernels (csrc/rnn.cu) are tested against fp64 in tests/test_rnn_cells_gpu.py."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

CELLS = ('gru', 'lstm')


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


STEP_CASES = {
    'tinyB': ('tiny', 'B', 5, 3, dict(batch_size=64), None),
    'tinyB_2l_drop': ('tiny', 'B', 5, 2, dict(rnn_num_layers=2, dropout_keep_prob=0.8), dict(bwd_precision=3)),
    'tinyB_cos': ('tiny', 'B', 5, 2, dict(ranking='cosine'), None),
    'tinyB_fwd3': ('tiny', 'B', 5, 2, {}, dict(fwd_precision=3)),
    'tinyB_bf16': ('tiny', 'B', 5, 2, {}, dict(fwd_precision=4)),
    'g1_b48': ('g1', 'B', 30, 2, dict(batch_size=48), None),
    'g1_b256': ('g1', 'B', 30, 1, {}, None),
    'adressa_b32': ('adressa', 'B', 20, 1, dict(batch_size=32), None),
}


@pytest.mark.parametrize('case', sorted(STEP_CASES))
@pytest.mark.parametrize('cell', CELLS)
def test_full_step_parity(cell, case):
    import torch
    from tools import gpu_step_check as g
    name, profile, warm, steps, hp, ekw = STEP_CASES[case]
    dtype = torch.float64 if name == 'tiny' else torch.float32
    res = g.run_case(name, profile, warm, steps, hp_over=dict(rnn_cell=cell, **hp), oracle_dtype=dtype, engine_kw=ekw)
    assert res['steps'][0]['L'] > 0
    _check_steps(res, grad_tol=2e-3 if (ekw and 'bwd_precision' in ekw) else 3e-2,
                 update_tol=0.3 if case == 'g1_b48' else 0.2)


@pytest.mark.parametrize('cell', CELLS)
def test_unsynced_trajectory_g1(cell):
    """30 steps, each side on its own Adam trajectory: the loss stays within 1e-3 relative of the fp32 oracle's."""
    import torch
    from tools import gpu_step_check as g
    res = g.run_trajectory('g1', 'B', 30, 30, hp_over=dict(batch_size=64, rnn_cell=cell), oracle_dtype=torch.float32)
    assert all(s['neg_equal'] for s in res['steps'])
    assert res['max_rel'] < 1e-3, [(s['step'], s['rel']) for s in res['steps'] if s['rel'] >= 1e-3]


@pytest.mark.parametrize('cell', CELLS)
def test_eval_ranking_and_metrics_vs_oracle(cell):
    """ModeKeys.EVAL with the session cell `cell`: ranked ids / probabilities and the HR@n / MRR@n sums against the oracle (ranks
    compared where the oracle's probability gaps exceed the forward tolerance)."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from oracle import sampler_ref
    from tools import gpu_step_check as g
    pb = make_problem('tiny', profile='B', rnn_cell=cell, rnn_num_layers=2)
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


@pytest.mark.parametrize('cell', CELLS)
def test_estimator_predict_vs_oracle(cell, tmp_path):
    """Estimator.train then Estimator.predict (top-n over the catalog after every session's last position) against the
    every-row oracle (oracle/recommend_ref.py) with the trained weights."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from oracle.recommend_ref import recommend
    from tools.gpu_step_check import make_oracle
    pb = make_problem('tiny', profile='B', rnn_cell=cell, batch_size=24)
    warm_state(pb, 5)
    est = _estimator(pb, str(tmp_path))
    est.train(pb.input_fn, steps=3)
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
        nth = ref['predicted_item_scores'][q][real].min()
        for d in set(ids[real].tolist()) ^ set(ref['predicted_item_ids'][q][real].tolist()):
            assert abs(ref['scores'][q, column[d]] - nth) <= tol, (q, d)


# the TF variables of layer 0's cell a checkpoint holds
TF_NAMES = {'gru': ('gru_cell/gates/kernel', 'gru_cell/gates/bias', 'gru_cell/candidate/kernel', 'gru_cell/candidate/bias'),
            'lstm': ('lstm_cell/kernel', 'lstm_cell/bias')}


@pytest.mark.parametrize('cell', CELLS)
def test_checkpoint_resume_matches_uninterrupted_run(cell, tmp_path):
    """A checkpoint of a GRU or LSTM model holds the cell's TF variable names, restores weights, Adam slots and step
    exactly, and training on from it tracks the run that was never interrupted."""
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.harness import make_problem, warm_state

    def fresh():
        pb = make_problem('tiny', profile='B', rnn_cell=cell)
        warm_state(pb, 5)
        it = pb.input_fn()
        return pb, [it.get_next() for _ in range(4)]

    d = str(tmp_path / 'model')
    pb_a, batches = fresh()
    est_a = _estimator(pb_a, d)
    est_a.train(lambda: iter(batches[:2]))
    path = ckpt.latest_checkpoint(d)
    assert path.endswith('model.ckpt-2.npz')
    names = set(np.load(path).files)
    for tf_name in TF_NAMES[cell]:
        assert any(n.endswith('multi_rnn_cell/cell_0/' + tf_name) for n in names), tf_name
    pb_b, batches_b = fresh()
    est_b = _estimator(pb_b, d)
    est_b._ensure_spec(*batches_b[2])
    ea, eb = est_a.model.engine, est_b.model.engine
    assert eb.global_step == 2
    assert torch.equal(ea.params, eb.params) and torch.equal(ea.adam_m, eb.adam_m) and torch.equal(ea.adam_v, eb.adam_v)
    est_a.train(lambda: iter(batches[2:]))
    est_b.train(lambda: iter(batches_b[2:]))
    assert eb.global_step == 4 and ea.global_step == 4
    assert abs(est_b.last_loss - est_a.last_loss) / abs(est_a.last_loss) < 1e-3
    assert float((ea.params - eb.params).abs().median()) < 1e-6
