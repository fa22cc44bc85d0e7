"""The unsampled evaluation's definitions on the CPU (DESIGN.md section 13): the oracle's competitor sets against the
reference sampler's own support, its rank formulas against the reference's HitRate, MRR and NDCG, the histogram
conversion the product uses, and the switch's defaults."""
import os
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = np.load(os.path.join(ROOT, 'tests', 'golden', 'unsampled_golden.npz'))


@pytest.mark.parametrize('scenario', ['covering', 'empty_buffer', 'repeats'])
def test_competitor_sets_are_the_reference_samplers_support(scenario):
    from oracle.unsampled_ref import competitor_sets
    ac = GOLDEN['support/%s/all_clicked' % scenario]
    buf = GOLDEN['support/%s/buffer' % scenario]
    neg = GOLDEN['support/%s/negatives' % scenario]
    sets = competitor_sets(ac[:, :-1], ac[:, -1], buf)
    checked = 0
    for b in range(ac.shape[0]):
        for t in range(ac.shape[1] - 1):
            if ac[b, t] == 0:
                assert not neg[b, t].any()
                continue
            row = neg[b, t]
            assert np.array_equal(np.sort(row[row != 0]), sets[b]), (b, t)      # a permutation: no repeats
            checked += 1
    assert checked > 0
    if scenario == 'covering':
        assert sets[0].size == 0
    if scenario == 'empty_buffer':
        assert not buf.any()


def test_labels_are_in_the_pool_and_not_their_own_competitors():
    from oracle.unsampled_ref import competitor_sets, pool
    ac = GOLDEN['support/repeats/all_clicked']
    buf = GOLDEN['support/repeats/buffer']
    ic, ll = ac[:, :-1], ac[:, -1]
    p, sets = pool(ic, ll, buf), competitor_sets(ic, ll, buf)
    label_next = np.concatenate([ic[:, 1:], np.zeros((ic.shape[0], 1), np.int64)], axis=1)
    for b in range(ic.shape[0]):
        for lab in list(label_next[b][label_next[b] != 0]) + ([ll[b]] if ll[b] else []):
            assert lab in p and lab not in sets[b]


@pytest.mark.parametrize('batch', [0, 1, 2])
@pytest.mark.parametrize('top_n', [1, 3, 5, 10])
def test_rank_formulas_reproduce_the_reference_metrics(batch, top_n):
    from chameleon_recsys_b200.eval_metrics import unsampled_results
    from oracle.unsampled_ref import metric_values, rank_rule
    labels = GOLDEN['metrics/b%d/labels' % batch]
    scores = GOLDEN['metrics/b%d/scores' % batch]
    per = GOLDEN['metrics/b%d/top%d/per_query' % (batch, top_n)]
    streamed = GOLDEN['metrics/b%d/top%d/streamed' % (batch, top_n)]
    qb, qt = np.nonzero(labels)
    ranks = np.array([rank_rule(scores[b, t, 0], scores[b, t, 1:]) for b, t in zip(qb, qt)])
    v = metric_values(ranks, top_n)
    for k, name in enumerate(('hitrate', 'mrr', 'ndcg')):
        assert np.array_equal(v[name], per[k][qb, qt]), name                 # every query, bit for bit
    assert v['hitrate'].sum() / ranks.size == streamed[0]
    assert np.mean(v['mrr']) == streamed[1] and np.mean(v['ndcg']) == streamed[2]
    # the product's integer histogram, converted in rank order, within the rounding of a different summation order
    hist = np.zeros(top_n + 2, np.int64)
    np.add.at(hist, ranks[ranks < top_n], 1)
    hist[top_n] = ranks.size
    res = unsampled_results(hist, top_n)
    assert res['unsampled_hitrate_at_n'] == streamed[0]
    assert abs(res['unsampled_mrr_at_n'] - streamed[1]) <= 1e-15
    assert abs(res['unsampled_ndcg_at_n'] - streamed[2]) <= 1e-15


def test_histogram_without_queries_is_nan():
    from chameleon_recsys_b200.eval_metrics import UNSAMPLED_KEYS, unsampled_results
    res = unsampled_results(np.zeros(7, np.int64), 5)
    assert list(res) == list(UNSAMPLED_KEYS) and all(np.isnan(v) for v in res.values())


def test_defaults_leave_the_params_unchanged():
    from chameleon_recsys_b200.hparams import NARHParams
    hp = NARHParams()
    assert hp.eval_unsampled_metrics is False
    base = hp.to_params({}, {}, {}, None)
    assert 'eval_unsampled_metrics' not in base
    on = hp.copy(eval_unsampled_metrics=True).to_params({}, {}, {}, None)
    assert on.pop('eval_unsampled_metrics') is True
    assert list(on) == list(base)


def test_data_parallel_evaluation_raises():
    from chameleon_recsys_b200.hparams import ModeKeys
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    model = types.SimpleNamespace(engine=types.SimpleNamespace(world=2))
    with pytest.raises(NotImplementedError):
        ItemsStateUpdaterHook(ModeKeys.EVAL, model, 5, clicked_items_state=None, eval_unsampled_metrics=True)
    hook = ItemsStateUpdaterHook(ModeKeys.EVAL, model, 5, clicked_items_state=None)
    assert not hook.unsampled_on and hook.unsampled_results() == {}
    train = ItemsStateUpdaterHook(ModeKeys.TRAIN, model, 5, clicked_items_state=None, eval_unsampled_metrics=True)
    assert not train.unsampled_on
