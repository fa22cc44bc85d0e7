"""Recommendation semantics on the CPU oracle (no GPU): oracle/recommend_ref.recommend scores a candidate for a query
position exactly like a sampled negative of that position - checked against NarOracle.forward, which
test_oracle_reference_model.py pins to the reference graph - and its top-n rule (order, ties, exclusion, probabilities)."""
import numpy as np
import pytest
import torch

from chameleon_recsys_b200.harness import make_problem, warm_state
from oracle import sampler_ref
from oracle.recommend_ref import recommend, topn_rule
from tools.gpu_step_check import make_oracle


def _case(profile, warm, batch_size=12, **hp):
    pb = make_problem('tiny', profile=profile, batch_size=batch_size, **hp)
    if warm:
        warm_state(pb, warm)
    orc = make_oracle(pb, torch.float64)
    orc.set_params(pb.layout.init_logical(pb.hp.init_seed))
    feats, labels = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    return pb, orc, feats, labels, buf, pop


@pytest.mark.parametrize('profile,hp', [('A', {}), ('B', {}), ('B', dict(rnn_cell='gru')), ('B', dict(ranking='cosine')),
                                        ('A', dict(rnn_cell='gru', ranking='cosine'))])
def test_recommend_scores_equal_forward_logits(profile, hp):
    """Candidates = every positive and sampled negative of the batch: the score of (position, candidate) equals the
    forward logit of that candidate at that position (warm buffer: every row group uses the buffer's statistics)."""
    pb, orc, feats, labels, buf, pop = _case(profile, 5, **hp)
    K = pb.hp.train_total_negative_samples
    allc = np.concatenate([feats['item_clicked'], labels['label_last_item']], axis=1)
    neg = sampler_ref.sample_negatives(allc, buf, K, pb.hp.train_negative_samples_from_buffer, pb.hp.sampler_seed, 1)
    with torch.no_grad():
        o = orc.forward(feats, labels, neg, buf, pop)
    logits = o['logits'].numpy()
    mask = o['mask'].numpy()
    ids = np.concatenate([np.asarray(labels['label_next_item'])[..., None], neg], axis=2)      # [B, T, 1+K]
    cand = np.unique(ids[mask][ids[mask] != 0])
    rec = recommend(orc, feats, buf, pop, cand, top_n=1, positions='all', exclude_session_clicks=False)
    assert np.array_equal(np.stack([rec['query_session'], rec['query_position']], 1), np.argwhere(mask))
    checked = 0
    for q, (b, t) in enumerate(zip(rec['query_session'], rec['query_position'])):
        for j in range(K + 1):
            if ids[b, t, j] == 0:
                continue
            col = np.searchsorted(cand, ids[b, t, j])
            assert abs(rec['scores'][q, col] - logits[b, t, j]) <= 1e-12 * max(1.0, abs(logits[b, t, j])), (b, t, j)
            checked += 1
    assert checked > 100


def test_recommend_empty_buffer_uses_candidate_statistics():
    """First batch (empty buffer): the candidate rows normalise recency / novelty with their own statistics, as the
    negatives do (the tf.cond at nar_model.py:1082 / :1179)."""
    pb, orc, feats, labels, buf, pop = _case('B', 0)
    assert not buf.any()
    cand = np.arange(1, 200, 3, dtype=np.int64)
    rec = recommend(orc, feats, buf, pop, cand, top_n=5, positions='last')
    x = rec['x']
    gamma = orc._p('main/user_items_contextual_features/input_features_center_scale/gamma_scale').detach()
    beta = orc._p('main/user_items_contextual_features/input_features_center_scale/beta_center').detach()
    ids = torch.as_tensor(cand)
    max_ts = torch.as_tensor(feats['event_timestamp']).long().max()
    days = orc._elapsed_days(orc.meta['created_at_ts'][ids], max_ts)
    raw = {'recency': orc._log_base(days + 1.0, orc.rec_base),
           'novelty': -orc._log_base(torch.as_tensor(pop, dtype=torch.float64)[ids], orc.pop_base)}
    seen = 0
    for sg in pb.plan.segments:
        if sg.name in raw:
            want = orc._normalize_values(raw[sg.name], raw[sg.name]) * gamma[sg.log_col] + beta[sg.log_col]
            np.testing.assert_allclose(x[:, :, sg.log_col], np.broadcast_to(want.numpy(), x.shape[:2]), rtol=0, atol=1e-12)
            seen += 1
    assert seen == 2


def test_topn_rule_order_ties_exclusion_padding():
    cand = np.array([10, 11, 12, 13], dtype=np.int64)
    s = np.array([[1.0, 3.0, 3.0, 2.0]])
    ids, sc, pr = topn_rule(s, cand, 3)
    assert ids.tolist() == [[11, 12, 13]] and sc.tolist() == [[3.0, 3.0, 2.0]]           # ties: lower index first
    e = np.exp(s[0] - 3.0)
    np.testing.assert_allclose(pr[0], e[[1, 2, 3]] / e.sum(), rtol=1e-15)
    ids, sc, pr = topn_rule(s, cand, 3, [{11, 99, 11}])
    assert ids.tolist() == [[12, 13, 10]]
    e = np.exp(s[0, [0, 2, 3]] - 3.0)                                                      # softmax without the excluded id
    np.testing.assert_allclose(pr[0], e[[1, 2, 0]] / e.sum(), rtol=1e-15)
    ids, sc, pr = topn_rule(s, cand, 4, [{10, 11, 12}])
    assert ids.tolist() == [[13, 0, 0, 0]] and pr[0, 0] == 1.0 and np.isinf(sc[0, 1:]).all() and not pr[0, 1:].any()
    _, _, pr = topn_rule(np.random.RandomState(0).randn(3, 4), cand, 4)
    np.testing.assert_allclose(pr.sum(1), 1.0, rtol=1e-14)


def test_recommend_default_candidates_and_exclusion():
    pb, orc, feats, labels, buf, pop = _case('B', 5)
    rec = recommend(orc, feats, buf, pop, None, top_n=8, positions='all')
    assert np.array_equal(rec['candidates'], np.unique(buf[buf != 0]))
    ic = np.asarray(feats['item_clicked'])
    for q, (b, t) in enumerate(zip(rec['query_session'], rec['query_position'])):
        assert not np.isin(rec['predicted_item_ids'][q], ic[b, :t + 1]).any()
        assert np.all(np.diff(rec['predicted_item_scores'][q]) <= 0)
    full = recommend(orc, feats, buf, pop, None, top_n=rec['candidates'].size, positions='last', exclude_session_clicks=False)
    np.testing.assert_allclose(full['predicted_item_probs'].sum(1), 1.0, rtol=1e-12)
    lens = np.clip(np.asarray(feats['session_size']) - 1, 0, ic.shape[1])
    assert np.array_equal(full['query_position'], (lens - 1)[lens > 0])
    cat = recommend(orc, feats, buf, pop, 'catalog', top_n=3, positions='last')
    assert np.array_equal(cat['candidates'], np.arange(1, pb.wl.num_items))
