"""Recommendation on the GPU (pytest -m gpu): nar_topn_candidates against numpy, NarEngine.recommend against the every-row
oracle (oracle/recommend_ref.py), against the EVAL logits of the same weights, chunking invariance, the G1 full catalog and
Estimator.predict."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


def _setup(name='tiny', profile='B', warm=5, oracle_dtype=None, engine_kw=None, **hp):
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine, make_oracle
    pb = make_problem(name, profile=profile, **hp)
    if warm:
        warm_state(pb, warm)
    eng = make_engine(pb, **(engine_kw or {}))
    logical = pb.layout.init_logical(pb.hp.init_seed)
    eng.set_params(logical)
    orc = None
    if oracle_dtype is not None:
        orc = make_oracle(pb, oracle_dtype or torch.float64)
        orc.set_params(logical)
    feats, labels = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    return pb, eng, orc, feats, labels, buf, pop


def _check_vs_oracle(rec, ref, rel_tol=1e-3):
    """Scores of the returned ids match the oracle's scores of the same ids within rel_tol of the largest |score|; the
    id sets differ only where the oracle's gap at the n-th place is below that tolerance."""
    assert np.array_equal(rec['query_session'], ref['query_session'])
    assert np.array_equal(rec['query_position'], ref['query_position'])
    assert np.array_equal(rec['candidates'], ref['candidates'])
    column = {int(c): i for i, c in enumerate(ref['candidates'])}
    tol = rel_tol * np.abs(ref['scores']).max()
    for q in range(rec['predicted_item_ids'].shape[0]):
        ids = rec['predicted_item_ids'][q]
        real = ids != 0
        col = [column[int(i)] for i in ids[real]]
        assert np.abs(rec['predicted_item_scores'][q][real] - ref['scores'][q, col]).max() <= tol, q
        want = ref['predicted_item_ids'][q]
        assert np.array_equal(real, want != 0), q
        nth = ref['predicted_item_scores'][q][real].min() if real.any() else 0.0
        for d in set(ids[real].tolist()) ^ set(want[want != 0].tolist()):
            assert abs(ref['scores'][q, column[d]] - nth) <= tol, (q, d)
        assert np.all(np.diff(rec['predicted_item_scores'][q][real]) <= 0)


@pytest.mark.parametrize('N', [1, 31, 4097, 1 << 20])
def test_topn_kernel_matches_numpy(N):
    import torch
    from chameleon_recsys_b200 import ops
    from oracle.recommend_ref import topn_rule
    rs = np.random.RandomState(N % 1000)
    Q = 3 if N > 100000 else 7
    lg = rs.randn(Q, N).astype(np.float32) * 3
    lg[1] = np.round(lg[1])                                     # planted exact ties (a handful of distinct values)
    if N > 4:
        lg[2, : N // 2] = lg[2, N // 2]
    cand = (rs.permutation(2 * N)[:N] + 1).astype(np.int64)
    T = 6
    ic = rs.randint(1, 2 * N + 10, size=(Q, T)).astype(np.int64)  # ids inside and outside the candidate set
    ic[:, 1] = cand[rs.randint(0, N, Q)]
    ic[:, 2] = ic[:, 1]                                         # repeats
    q_pos = (np.arange(Q) * T + rs.randint(0, T, Q)).astype(np.int32)
    d = torch.device('cuda')
    for top_n in sorted({1, min(N, 5), min(N, 4096)}):
        for excl in (False, True):
            ids = torch.empty(Q, top_n, dtype=torch.int64, device=d)
            sc = torch.empty(Q, top_n, device=d)
            pr = torch.empty(Q, top_n, device=d)
            ops.topn_candidates(torch.from_numpy(lg).to(d), torch.from_numpy(cand).to(d), Q, N, top_n, ids, sc, pr,
                                torch.from_numpy(ic).to(d) if excl else None, torch.from_numpy(q_pos).to(d), T)
            ex = [set(ic[q, :q_pos[q] % T + 1].tolist()) for q in range(Q)] if excl else None
            wid, wsc, wpr = topn_rule(lg, cand, top_n, ex)
            assert np.array_equal(ids.cpu().numpy(), wid), (top_n, excl)
            assert np.array_equal(sc.cpu().numpy().astype(np.float64), wsc), (top_n, excl)
            got = pr.cpu().numpy().astype(np.float64)
            assert np.all(np.abs(got - wpr) <= 1e-6 * wpr + 1e-30), (top_n, excl, np.abs(got - wpr).max())


ENGINE_CASES = {
    'A_mlp_last_warm': ('A', {}, 4, 'last', True, 5, None),
    'B_mlp_all_warm_fp3': ('B', {}, 3, 'all', True, 5, None),
    'B_gru_last_noexcl': ('B', dict(rnn_cell='gru'), 4, 'last', False, 5, None),
    'B_cos_all_warm': ('B', dict(ranking='cosine'), 4, 'all', True, 5, None),
    'A_gru_cos_last_fp3': ('A', dict(rnn_cell='gru', ranking='cosine'), 3, 'last', True, 5, None),
    'B_mlp_empty_catalog': ('B', {}, 4, 'last', True, 0, 'catalog'),
    'B_cos_empty_catalog_all': ('B', dict(ranking='cosine'), 3, 'all', False, 0, 'catalog'),
    'B_2l_ids': ('B', dict(rnn_num_layers=2), 4, 'all', True, 5, 'ids'),
}


@pytest.mark.parametrize('case', sorted(ENGINE_CASES))
def test_engine_recommend_vs_oracle(case):
    import torch
    profile, hp, fp, positions, excl, warm, cands = ENGINE_CASES[case]
    pb, eng, orc, feats, labels, buf, pop = _setup(profile=profile, warm=warm, oracle_dtype=torch.float64,
                                                    engine_kw=dict(fwd_precision=fp), batch_size=24, **hp)
    if cands == 'ids':
        cands = np.random.RandomState(1).choice(np.arange(1, pb.wl.num_items), 300, replace=False)
    rec = eng.recommend(feats, buf, pop, 10, candidates=cands, positions=positions, exclude_session_clicks=excl)
    from oracle.recommend_ref import recommend
    ref = recommend(orc, feats, buf, pop, cands, 10, positions=positions, exclude_session_clicks=excl)
    _check_vs_oracle(rec, ref)
    np.testing.assert_allclose(rec['predicted_item_probs'], ref['predicted_item_probs'], rtol=2e-2, atol=1e-6)


@pytest.mark.parametrize('ranking', ['mlp', 'cosine'])
def test_recommend_reproduces_eval_logits(ranking):
    """EVAL ranks the 1+K sampled candidates of every position; recommend over their union must give every one of
    those logits (the positive row takes PP in EVAL and PC + PI here: layer 1 associates differently)."""
    pb, eng, _, feats, labels, buf, pop = _setup(warm=5, ranking=ranking)
    out = eng.eval_step(feats, labels, buf, pop, top_n=3)
    st = out['stage']
    L, n_cand = st['L'], eng.K + 1
    lg = out['logits'].cpu().numpy().reshape(L, n_cand)
    ids = eng.buffer(st, 'row_item').view(-1)[L:L + L * n_cand].cpu().numpy().reshape(L, n_cand)
    cand = np.unique(ids[ids != 0])
    rec = eng.recommend(feats, buf, pop, cand.size, candidates=cand, positions='all', exclude_session_clicks=False)
    tol = 1e-4 * np.abs(lg).max()
    for q in range(L):
        score = dict(zip(rec['predicted_item_ids'][q].tolist(), rec['predicted_item_scores'][q].tolist()))
        for j in range(n_cand):
            if ids[q, j]:
                assert abs(score[int(ids[q, j])] - lg[q, j]) <= tol, (q, j)


@pytest.mark.parametrize('ranking,positions', [('mlp', 'last'), ('mlp', 'all'), ('cosine', 'all')])
def test_recommend_chunking_is_bit_identical(ranking, positions):
    pb, eng, _, feats, labels, buf, pop = _setup(warm=5, ranking=ranking)
    full = eng.recommend(feats, buf, pop, 20, candidates='catalog', positions=positions)
    assert full['n_block'] == full['candidates'].size or ranking == 'cosine'
    for budget in (4 << 20, 2 << 20):             # (the fixed part - feature rows, session branch - is ~1.5 MB here)
        small = eng.recommend(feats, buf, pop, 20, candidates='catalog', positions=positions, ws_budget=budget)
        assert small['n_block'] < full['candidates'].size
        for k in ('predicted_item_ids', 'predicted_item_scores', 'predicted_item_probs'):
            assert np.array_equal(small[k], full[k]), (budget, k)
    if positions == 'all':
        assert small['q_block'] < full['predicted_item_ids'].shape[0]


def test_g1_full_catalog_batch():
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine, make_oracle
    pb = make_problem('g1', profile='B')
    warm_state(pb, 20)
    eng = make_engine(pb)
    logical = pb.layout.init_logical(pb.hp.init_seed)
    eng.set_params(logical)
    feats, labels = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    rec = eng.recommend(feats, buf, pop, 10, candidates='catalog')
    B = feats['item_clicked'].shape[0]
    assert B == 256 and rec['predicted_item_ids'].shape == (B, 10) and rec['candidates'].size == 46033
    # two sessions through the fp32 oracle: one of them holds the batch's latest click, so max_ts is unchanged
    s_max = int(np.argmax(np.asarray(feats['event_timestamp']).max(1)))
    pick = [3 if s_max != 3 else 4, s_max]
    sub = {k: np.asarray(v)[pick] for k, v in feats.items()}
    orc = make_oracle(pb, torch.float32)
    orc.set_params(logical)
    from oracle.recommend_ref import recommend
    ref = recommend(orc, sub, buf, pop, 'catalog', 10)
    mine = {k: rec[k][pick] for k in ('predicted_item_ids', 'predicted_item_scores', 'predicted_item_probs')}
    mine.update(query_session=np.arange(2), query_position=rec['query_position'][pick], candidates=rec['candidates'])
    _check_vs_oracle(mine, ref)


def test_estimator_predict(tmp_path):
    import copy
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 3)
    hp = pb.hp

    def est_for(d, state):
        return build_estimator(str(d), pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                               pb.session_features_config, hp, state, device=0)

    est = est_for(tmp_path, pb.clicked_items_state)
    est.train(pb.input_fn, steps=4)
    eng = est.model.engine
    p0, m0, step0 = eng.get_params(), eng.adam_m.clone(), eng.global_step
    st = pb.clicked_items_state
    buf0, pop0 = st.get_recent_clicks_buffer().copy(), st.get_articles_recent_pop_norm().copy()
    batch = pb.input_fn().get_next()          # (the session stream is stateful: every predict call gets this batch)
    feats = batch[0]

    def one_batch():
        return iter([batch])
    preds = list(est.predict(one_batch))
    assert len(preds) == feats['item_clicked'].shape[0]
    for p in preds:
        assert set(p) == {'session_id', 'predicted_item_ids', 'predicted_item_scores', 'predicted_item_probs'}
        assert p['predicted_item_ids'].shape == (hp.eval_metrics_top_n,)
    p1 = eng.get_params()
    assert all(np.array_equal(p0[k], p1[k]) for k in p0)
    assert bool((eng.adam_m == m0).all()) and eng.global_step == step0
    assert np.array_equal(st.get_recent_clicks_buffer(), buf0) and np.array_equal(st.get_articles_recent_pop_norm(), pop0)
    # a fresh Estimator on the same model_dir serves the checkpoint
    fresh = est_for(tmp_path, copy.deepcopy(st))
    again = list(fresh.predict(one_batch))
    for a, b in zip(preds, again):
        assert np.array_equal(a['predicted_item_ids'], b['predicted_item_ids'])
        np.testing.assert_allclose(a['predicted_item_scores'], b['predicted_item_scores'], rtol=1e-6)
    empty = tmp_path / 'empty'
    empty.mkdir()
    with pytest.raises(ValueError):
        list(est_for(empty, st).predict(one_batch))
    V = pb.wl.num_items
    for bad in ([0, 1], [5, 5], [V], 'everything', np.array([1.5, 2.5])):
        with pytest.raises(ValueError):
            list(est.predict(one_batch, candidates=bad))
    for bad in (0, 5000, 1.5):
        with pytest.raises(ValueError):
            list(est.predict(one_batch, top_n=bad))
    with pytest.raises(ValueError):
        list(est.predict(one_batch, positions='first'))
