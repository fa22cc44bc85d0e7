"""oracle/baselines_ref.py against the reference's own baseline recommenders (tests/golden/make_baselines_golden.py ran
recently_popular / item_cooccurrences / item_knn / content_based / sequential_rules and ClickedItemsState in the hook's
order).  No GPU."""
import os

import numpy as np
import pytest

from oracle.baselines_ref import SUFFIXES, BaselinesRef

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'baselines_golden.npz')


@pytest.fixture(scope='module')
def g():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _all_items(g, name):
    return np.concatenate([g[name + '_ic'], g[name + '_last']], axis=1)


def _replay(g):
    """The oracle through the fixture's batches -> (oracle at the end, export after training, per-eval-batch results)."""
    V, B, T, K, top_n, n_train, n_eval = g['cfg'].tolist()
    ref = BaselinesRef(V, acr=g['acr'])
    for s in range(n_train):
        ref.update(_all_items(g, 'train%d' % s))
    trained = ref.export()
    ref.snapshot()
    res = []
    for s in range(n_eval):
        e = 'eval%d' % s
        res.append(ref.score(g[e + '_ic'], g[e + '_ln'], g[e + '_neg'], g[e + '_buffer'], g[e + '_pop'], top_n))
        ref.update(_all_items(g, e))
    return ref, trained, res


def _sr_dict(g, prefix):
    return {(int(a), int(c)): float(w) for a, c, w in zip(g[prefix + '_sr_past'], g[prefix + '_sr_active'], g[prefix + '_sr_w'])}


def test_tables_match_reference(g):
    ref, trained, _ = _replay(g)
    V = int(g['cfg'][0])
    # the state after training and after the eval batches (before the restore): co-occurrence CSR exact, SR to 1e-12
    after_train = BaselinesRef(V)
    for s in range(int(g['cfg'][5])):
        after_train.update(_all_items(g, 'train%d' % s))
    for o, prefix in ((after_train, 'train'), (ref, 'eval')):
        np.testing.assert_array_equal(o.cooc_dense(), g[prefix + '_cooc_dense'])
        want, got = _sr_dict(g, prefix), o.sr_rules()
        assert set(want) == set(got)
        for k, w in want.items():
            assert abs(got[k] - w) <= 1e-12 * abs(w), k


def test_cooccurrence_counts_each_distinct_pair_once_per_session():
    ref = BaselinesRef(10)
    ref.update(np.array([[3, 4, 3, 4, 3, 0]]))
    m = ref.cooc_dense()
    assert m[3, 4] == 1 and m[4, 3] == 1 and m[3, 3] == 1 and m[4, 4] == 1
    assert ref.sr_w[(3, 4)] == 2520 + 840 + 2520          # (j, i) = (0, 1), (0, 3), (2, 3)
    assert ref.sr_w[(3, 3)] == 1260 + 630 + 1260           # (0, 2), (0, 4), (2, 4)


def _check_groups(sfx, want, got, scores, tol):
    """want / got: top-n id lists; scores: {id: score} of every admissible candidate.  The lists agree as sequences of
    equal-score groups: the same scores rank by rank, the same ids above the cut, and both take the ids at the cut from
    the candidates with the cut's score."""
    n = min(len(want), len(scores))
    if n == 0:
        return
    want, got = [int(c) for c in want[:n]], [int(c) for c in got[:n]]
    sw, sg = [scores[c] for c in want], [scores[c] for c in got]
    np.testing.assert_allclose(sg, sw, rtol=0, atol=tol, err_msg=sfx)
    cut = sw[-1]
    above_w = {c for c, v in zip(want, sw) if v - cut > tol}
    above_g = {c for c, v in zip(got, sg) if v - cut > tol}
    assert above_w == above_g, sfx
    at_cut = {c for c, v in scores.items() if abs(v - cut) <= tol}
    assert set(want) - above_w <= at_cut and set(got) - above_g <= at_cut, sfx


def test_predictions_and_metrics_match_reference(g):
    """pop_recent / sr: id for id and the same HR / MRR; coocurrent / item_knn / cb: equal-score groups, and the
    reference's HR / MRR lie inside the oracle's [pessimistic, optimistic] bounds over all orders of ties."""
    V, B, T, K, top_n, n_train, n_eval = g['cfg'].tolist()
    for sfx in SUFFIXES:
        ref = BaselinesRef(V, acr=g['acr'])
        for s in range(n_train):
            ref.update(_all_items(g, 'train%d' % s))
        hits = rr = cnt = lo_h = hi_h = lo_r = hi_r = 0.0
        for s in range(n_eval):
            e = 'eval%d' % s
            r = ref.score(g[e + '_ic'], g[e + '_ln'], g[e + '_neg'], g[e + '_buffer'], g[e + '_pop'], top_n, suffixes=(sfx,))[sfx]
            want = g['%s_pred_%s' % (e, sfx)].reshape(B * T, top_n)
            ln, ic, neg = g[e + '_ln'].reshape(-1), g[e + '_ic'].reshape(-1), g[e + '_neg'].reshape(B * T, K)
            for q in np.flatnonzero(ln):
                if sfx in ('pop_recent', 'sr'):
                    np.testing.assert_array_equal(r['ids'][q], want[q], err_msg='%s %s q%d' % (sfx, e, q))
                else:
                    scores = ref.candidate_scores(sfx, ic[q], [ln[q]] + neg[q].tolist(), g[e + '_buffer'], g[e + '_pop'])
                    _check_groups(sfx, want[q], r['ids'][q], scores, 1e-12 if sfx == 'cb' else 0.0)
            hits += r['hits']; rr += r['rr']; cnt += r['count']
            lo_h += r['bounds'][0]; hi_h += r['bounds'][1]; lo_r += r['bounds'][2]; hi_r += r['bounds'][3]
            ref.update(_all_items(g, e))
        ref_hr, ref_mrr = float(g['hr_' + sfx]), float(g['mrr_' + sfx])
        assert lo_h / cnt - 1e-12 <= ref_hr <= hi_h / cnt + 1e-12, sfx
        assert lo_r / cnt - 1e-12 <= ref_mrr <= hi_r / cnt + 1e-12, sfx
        if sfx in ('pop_recent', 'sr'):
            assert abs(hits / cnt - ref_hr) < 1e-12 and abs(rr / cnt - ref_mrr) < 1e-12, sfx


def test_snapshot_restore_leaves_tables_unchanged(g):
    ref, trained, _ = _replay(g)
    ref.restore()
    after = ref.export()
    for k in trained:
        np.testing.assert_array_equal(after[k], trained[k])
    np.testing.assert_array_equal(ref.cooc_dense(), g['restored_cooc_dense'])
    assert set(ref.sr_rules()) == set(_sr_dict(g, 'restored'))
