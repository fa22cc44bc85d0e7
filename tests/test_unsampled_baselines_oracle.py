"""The baselines' unsampled evaluation on the CPU (DESIGN.md section 14): oracle/unsampled_baselines_ref.py against the
reference's own recommenders ranking the whole competitor set (tests/golden/make_unsampled_baselines_golden.py), its ranks
against the sampled oracles' when the pool is the label and its logged negatives, and the switch's plumbing.  No GPU."""
import os
import sys
import types
from collections import Counter

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.baselines_ref import SUFFIXES, BaselinesRef  # noqa: E402
from oracle.sknn_ref import SknnRef  # noqa: E402
from oracle.unsampled_baselines_ref import MISS, histogram, metrics, ranks  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')


def _load(name):
    with np.load(os.path.join(GOLDEN_DIR, name)) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope='module')
def g():
    return _load('unsampled_baselines_golden.npz')


def _all_items(g, name):
    return np.concatenate([g[name + '_ic'], g[name + '_last']], axis=1)


def _make_ref(g, sfx):
    if sfx in SUFFIXES:
        return BaselinesRef(int(g['cfg'][0]), acr=g['acr'])
    k = ('v-sknn', 'sknn').index(sfx)
    S, C, NN = g['knn_params'][k].tolist()
    return SknnRef(S, C, NN, str(g['knn_similarity'][k]), str(g['knn_decay'][k]))


def _fold(ref, g, name):
    if isinstance(ref, BaselinesRef):
        ref.update(_all_items(g, name))
    else:
        ref.update(g[name + '_sid'], _all_items(g, name))


def _same_neighbours(g, e, sfx, q, ref, P):
    """The reference's neighbour list of flat query q as a multiset of (id, sim) equals the oracle's (not so where the
    neighbour cut falls inside a group of equal similarities, which the reference orders by set iteration)."""
    p = '%s_%s_' % (e, sfx)
    off = g[p + 'nb_off']
    want = zip(g[p + 'nb_sid'][off[q]:off[q + 1]].tolist(), g[p + 'nb_sim'][off[q]:off[q + 1]].tolist())
    return Counter(want) == Counter(ref.neighbors(P))


def _reference_rank(pred, label):
    hit = np.flatnonzero(pred == label)
    return int(hit[0]) if hit.size else MISS


@pytest.mark.parametrize('sfx', SUFFIXES + ('v-sknn', 'sknn'))
def test_oracle_reproduces_the_reference_recommenders(g, sfx):
    """pop_recent and sr rank for rank; coocurrent, item_knn, cb and the session kNN baselines within the equal-score
    group of the label; the same labels missed; the reference's HR / MRR / NDCG inside the oracle's tie bounds (equal to
    them for pop_recent and sr).  A kNN query whose neighbour cut splits a group of equal similarities (the reference
    then keeps other neighbours) is counted, not compared, and widens the metric bounds by one query each."""
    V, B, T, top_n, n_train, n_eval = g['cfg'].tolist()
    ref = _make_ref(g, sfx)
    for s in range(n_train):
        _fold(ref, g, 'train%d' % s)
    allr = {'rank': [], 'rank_lo': [], 'rank_hi': [], 'n_comp': []}
    ties = split = 0
    for s in range(n_eval):
        e = 'eval%d' % s
        r = ranks(ref, sfx, g[e + '_ic'], g[e + '_ln'], g[e + '_last'], g[e + '_buffer'], g[e + '_pop'])
        pred = g['%s_pred_%s' % (e, sfx)].reshape(B * T, -1)
        ln = g[e + '_ln'].reshape(-1)
        valid = g[e + '_valid'].reshape(B * T, -1)
        assert np.array_equal(r['q'], np.flatnonzero(ln))
        for i, q in enumerate(r['q']):
            assert r['n_comp'][i] == np.unique(valid[q]).size - 1
            want = _reference_rank(pred[q], ln[q])
            got = int(r['rank'][i])
            b, t = divmod(int(q), T)
            if sfx not in SUFFIXES and not _same_neighbours(g, e, sfx, q, ref, g[e + '_ic'][b, :t + 1].tolist()):
                split += 1
                continue
            assert (want == MISS) == (got == MISS), (sfx, e, q, want, got)
            if sfx in ('pop_recent', 'sr'):
                assert got == want, (sfx, e, q)
            elif sfx in SUFFIXES:
                assert r['rank_hi'][i] <= want <= r['rank_lo'][i], (sfx, e, q, want, r['rank_hi'][i], r['rank_lo'][i])
            elif got != MISS:
                # the reference orders neighbours of equal similarity by set iteration, so its item sums may differ
                # in the last bits: its rank lies in the label's equal-score group up to that rounding
                scores, _ = ref.item_scores(g[e + '_ic'][b, :t + 1].tolist())
                comp = [x for x in np.unique(valid[q]) if x != ln[q] and x in scores]
                sl, tol = scores[ln[q]], 1e-12 * max(scores.values())
                assert sum(scores[x] > sl + tol for x in comp) <= want <= sum(scores[x] >= sl - tol for x in comp), \
                    (sfx, e, q)
            ties += r['rank_lo'][i] > r['rank_hi'][i]
        for k in allr:
            allr[k].append(r[k])
        _fold(ref, g, e)
    allr = {k: np.concatenate(v) for k, v in allr.items()}
    m = metrics(allr, top_n)
    Q = allr['rank'].size
    assert Q > 5 * split, (Q, split)
    for name in ('hr', 'mrr', 'ndcg'):
        k = {'hr': 'hitrate'}.get(name, name)
        want = float(g['%s_%s' % (name, sfx)])
        slack = split / Q + 1e-12
        assert m[k + '_lo'] - slack <= want <= m[k + '_hi'] + slack, (sfx, name, want, m[k + '_lo'], m[k + '_hi'])
        if sfx in ('pop_recent', 'sr'):
            assert abs(m[k] - want) <= 1e-12, (sfx, name)
    h = histogram(allr, top_n)
    assert h[top_n] == allr['rank'].size and h[:top_n].sum() == np.count_nonzero(allr['rank'] < top_n)
    print('%s: %d queries, %d with equal-score competitors, %d with a split neighbour cut' % (sfx, Q, ties, split))


def _sampled_rank(ids, label, top_n):
    hit = np.flatnonzero(ids == label)
    return int(hit[0]) if hit.size else top_n


def _consistent(ref, sfx, e, g, top_n, sampled):
    B, T = g[e + '_ic'].shape
    ln, ic, last = g[e + '_ln'], g[e + '_ic'], g[e + '_last']
    neg = g[e + '_neg'].reshape(B * T, -1)
    checked = 0
    for q in np.flatnonzero(ln.reshape(-1)):
        b = q // T
        row = np.append(ic[b], last[b])
        if not neg[q].all() or np.isin(neg[q], row).any():
            continue                                # a zero-padded negative, or one the pool's exclusion would drop
        kw = dict(articles_pop=g.get(e + '_pop'), candidates=np.append(neg[q], ln.reshape(-1)[q]))
        r = ranks(ref, sfx, ic, ln, last, g.get(e + '_buffer', np.zeros(1, np.int64)), **kw)
        got = int(r['rank'][np.flatnonzero(r['q'] == q)[0]])
        assert min(got, top_n) == _sampled_rank(sampled[q], ln.reshape(-1)[q], top_n), (sfx, e, q)
        checked += 1
    return checked


@pytest.mark.parametrize('sfx', SUFFIXES)
def test_rank_against_the_logged_negatives_is_the_sampled_rank(sfx):
    """Pool = {label} | its negatives: the oracle's unsampled rank is BaselinesRef.score's sampled rank (or a miss)."""
    g = _load('baselines_golden.npz')
    V, B, T, K, top_n, n_train, n_eval = g['cfg'].tolist()
    ref = BaselinesRef(V, acr=g['acr'])
    for s in range(n_train):
        ref.update(_all_items(g, 'train%d' % s))
    checked = 0
    for s in range(n_eval):
        e = 'eval%d' % s
        sampled = ref.score(g[e + '_ic'], g[e + '_ln'], g[e + '_neg'], g[e + '_buffer'], g[e + '_pop'], top_n,
                            suffixes=(sfx,))[sfx]['ids']
        checked += _consistent(ref, sfx, e, g, top_n, sampled)
        ref.update(_all_items(g, e))
    assert checked > 0


@pytest.mark.parametrize('config', [0, 1])
def test_knn_rank_against_the_logged_negatives_is_the_sampled_rank(config):
    """The same for SknnRef.score (sknn_golden.npz's 'div' + cosine and 'same' + jaccard configurations)."""
    g = _load('sknn_golden.npz')
    V, B, T, K, top_n, n_train, n_eval = g['cfg'].tolist()
    S, C, NN = g['params'][config].tolist()
    ref = SknnRef(S, C, NN, str(g['similarity'][config]), str(g['decay'][config]))
    for s in range(n_train):
        ref.update(g['train%d_sid' % s], _all_items(g, 'train%d' % s))
    checked = 0
    for s in range(n_eval):
        e = 'eval%d' % s
        sampled = ref.score(g[e + '_ic'], g[e + '_ln'], g[e + '_neg'], top_n)['ids']
        checked += _consistent(ref, ref.suffix, e, g, top_n, sampled)
        ref.update(g[e + '_sid'], _all_items(g, e))
    assert checked > 0


def test_switch_goes_into_params_only_when_on():
    from chameleon_recsys_b200.hparams import NARHParams
    hp = NARHParams()
    assert hp.eval_unsampled_benchmarks is False
    base = hp.to_params({}, {}, {}, None)
    assert 'eval_unsampled_benchmarks' not in base
    on = hp.copy(eval_unsampled_benchmarks=True).to_params({}, {}, {}, None)
    assert on.pop('eval_unsampled_benchmarks') is True
    assert list(on) == list(base)


def _estimator(**params):
    from chameleon_recsys_b200.estimator import Estimator, nar_module_model_fn
    return Estimator(nar_module_model_fn, params)


def test_empty_evaluate_returns_the_keys_as_nan():
    from chameleon_recsys_b200.eval_metrics import UNSAMPLED_KEYS
    bench = ['pop_recent', 'sr', 'v-sknn']
    out = _estimator(eval_benchmarks=bench, eval_unsampled_benchmarks=True).evaluate(lambda: iter([]))
    want = {'unsampled_%s_at_n_%s' % (m, s) for m in ('hitrate', 'mrr', 'ndcg') for s in bench}
    want.add('unsampled_candidates_per_query')
    assert want <= set(out) and all(np.isnan(out[k]) for k in want)
    assert not set(UNSAMPLED_KEYS[:3]) & set(out)                # the model's own keys only come with their switch
    both = _estimator(eval_benchmarks=bench, eval_unsampled_benchmarks=True,
                      eval_unsampled_metrics=True).evaluate(lambda: iter([]))
    assert set(both) == set(out) | set(UNSAMPLED_KEYS)


def test_switch_without_baselines_raises():
    from chameleon_recsys_b200.hparams import ModeKeys
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    with pytest.raises(ValueError):
        _estimator(eval_unsampled_benchmarks=True).evaluate(lambda: iter([]))
    model = types.SimpleNamespace(engine=types.SimpleNamespace(world=1))
    with pytest.raises(ValueError):
        ItemsStateUpdaterHook(ModeKeys.EVAL, model, 5, clicked_items_state=None, eval_unsampled_benchmarks=True)
    train = ItemsStateUpdaterHook(ModeKeys.TRAIN, model, 5, clicked_items_state=None, eval_unsampled_benchmarks=True)
    assert not train.unsampled_bench_on and train.unsampled_benchmark_results() == {}


def test_data_parallel_evaluation_raises():
    from chameleon_recsys_b200.hparams import ModeKeys
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    model = types.SimpleNamespace(engine=types.SimpleNamespace(world=2))
    with pytest.raises(NotImplementedError):
        ItemsStateUpdaterHook(ModeKeys.EVAL, model, 5, clicked_items_state=None, eval_unsampled_benchmarks=True,
                              eval_benchmark_classifiers=['pop_recent'])
