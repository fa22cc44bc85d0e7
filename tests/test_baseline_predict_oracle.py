"""The baselines' recommendations on the CPU (DESIGN.md section 16): oracle/baseline_predict_ref.py against the reference's
own seven ``predict`` methods with each query's valid set (tests/golden/make_baseline_predict_golden.py), and the
argument checks of Estimator.predict(recommender=...) that run before anything reaches a GPU.  No GPU."""
import os
import sys
import types
from collections import Counter

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.baseline_predict_ref import ranked, recommend, valid_set  # noqa: E402
from oracle.baselines_ref import SUFFIXES, BaselinesRef  # noqa: E402
from oracle.sknn_ref import SknnRef  # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'baseline_predict_golden.npz')
ALL7 = SUFFIXES + ('v-sknn', 'sknn')


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


def _check_split(g, e, sfx, q, ref, P, valid, want, got, got_scores):
    """A query whose neighbour cut falls inside a group of equal similarities s_b: the reference keeps its own subset of
    that group (set-iteration order), the oracle keeps the higher session ids.  The neighbours above s_b are the same
    in both (as multisets of (id, sim)).  The reference's list is its valid ids ranked by the item scores of its own
    recorded neighbours, within equal-score groups; and every id's score in either list lies in the tie bounds: at least
    the sum over the neighbours above s_b, at most that plus every candidate neighbour at s_b holding it."""
    p = '%s_%s_' % (e, sfx)
    off = g[p + 'nb_off']
    nb_ref = list(zip(g[p + 'nb_sid'][off[q]:off[q + 1]].tolist(), g[p + 'nb_sim'][off[q]:off[q + 1]].tolist()))
    uncut = ref.neighbors(P, cut=False)
    s_b = min(sim for _, sim in nb_ref)
    assert Counter(x for x in nb_ref if x[1] > s_b) == Counter(x for x in uncut if x[1] > s_b), (sfx, e, q)

    def sums(nbs):
        out = {}
        for s, sim in nbs:
            for x in ref.buffer[ref.find(s)][1]:
                out[x] = out.get(x, 0) + sim
        return out
    ref_sc = sums(nb_ref)
    lo = sums([x for x in uncut if x[1] > s_b])
    hi = sums([x for x in uncut if x[1] >= s_b])
    tol = 1e-12 * max(hi.values())
    adm = sorted((ref_sc[c] for c in dict.fromkeys(valid) if c in ref_sc), reverse=True)
    n = min(len(want), len(adm))
    assert (want[n:] == 0).all() and len(set(want[:n].tolist())) == n, (sfx, e, q)
    for r in range(n):
        c = int(want[r])
        assert abs(ref_sc[c] - adm[r]) <= tol, (sfx, e, q, r)
        assert lo.get(c, 0.0) - tol <= ref_sc[c] <= hi[c] + tol, (sfx, e, q, r)
    for c, sc in zip(got.tolist(), got_scores.tolist()):
        if c:
            assert lo.get(c, 0.0) - tol <= sc <= hi[c] + tol, (sfx, e, q)


@pytest.mark.parametrize('sfx', ALL7)
def test_oracle_reproduces_the_reference_predict(sfx):
    """Every query (a nonzero click) of every eval batch, for the buffer's and the catalog's ids, exclusion on and off, at
    top n and at a width past every valid set: the reference pads with 0 exactly where the oracle does; pop_recent and
    sr give the same ids in the same order; coocurrent, item_knn and cb put at every rank an id of the oracle's score at
    that rank (they differ only inside groups of equal scores); the kNN baselines the same up to the last bits of the item
    sums, whose neighbours the reference adds in set-iteration order.  A kNN query whose neighbour cut splits a group of
    equal similarities (the reference then keeps other neighbours) is held to the tie bounds instead (_check_split)."""
    with np.load(GOLDEN) as z:
        g = {k: z[k] for k in z.files}
    V, B, T, top_n, n_train, n_eval, big = g['cfg'].tolist()
    ref = _make_ref(g, sfx)
    for s in range(n_train):
        _fold(ref, g, 'train%d' % s)
    checked = split = tied = padded = 0
    for s in range(n_eval):
        e = 'eval%d' % s
        ic, buf, pop = g[e + '_ic'], g[e + '_buffer'], g[e + '_pop']
        q_pos = np.flatnonzero(ic.reshape(-1))
        for cname in ('buf', 'cat'):
            cand = g['%s_cand_%s' % (e, cname)]
            for ex in (1, 0):
                for k in (top_n, big):
                    pred = g['%s_pred_%s_%s_%d_%d' % (e, sfx, cname, ex, k)].reshape(B * T, k)
                    ids, scores = recommend(ref, sfx, ic, q_pos, cand, k, buffer=buf, articles_pop=pop, exclude=bool(ex))
                    for i, q in enumerate(q_pos.tolist()):
                        b, t = divmod(q, T)
                        if sfx not in SUFFIXES and not _same_neighbours(g, e, sfx, q, ref, ic[b, :t + 1].tolist()):
                            _check_split(g, e, sfx, q, ref, ic[b, :t + 1].tolist(),
                                         valid_set(cand, ic, b, t, bool(ex)), pred[q], ids[i], scores[i])
                            split += 1
                            continue
                        full = ranked(ref, sfx, ic, b, t, valid_set(cand, ic, b, t, bool(ex)), buf, pop)
                        n = min(k, len(full))
                        want, got = pred[q], ids[i]
                        assert (want[n:] == 0).all() and (got[n:] == 0).all() and np.isnan(scores[i, n:]).all()
                        assert (want[:n] != 0).all() and len(set(want[:n].tolist())) == n, (sfx, e, q)
                        padded += n < k
                        key = {c: sc for sc, _, c in full}
                        checked += 1
                        if sfx in ('pop_recent', 'sr'):
                            assert np.array_equal(want, got), (sfx, e, cname, ex, k, q)
                            continue
                        tol = 0.0 if sfx in SUFFIXES else 1e-12 * max((abs(v) for v in key.values()), default=0.0)
                        for r in range(n):
                            assert int(want[r]) in key, (sfx, e, q, r)
                            assert abs(key[int(want[r])] - scores[i, r]) <= tol, (sfx, e, cname, ex, k, q, r)
                        tied += not np.array_equal(want, got)
        _fold(ref, g, e)
    assert padded > 0 and split * 5 < checked + split + 1
    print('%s: %d rows compared, %d differing only inside equal-score groups, %d padded, %d held to the tie bounds'
          % (sfx, checked, tied, padded, split))


def _estimator(**params):
    from chameleon_recsys_b200.estimator import Estimator, nar_module_model_fn
    return Estimator(nar_module_model_fn, params)


def test_predict_argument_errors_raise_before_any_batch():
    """An unknown suffix, a suffix outside eval_benchmarks (or without any) raise ValueError when the generator starts,
    before the first batch is read or anything is built."""
    read = []

    def input_fn():
        read.append(1)
        return iter([])
    for params, rec in (({'eval_benchmarks': ['pop_recent']}, 'vsknn'), ({'eval_benchmarks': ['pop_recent']}, 'sr'),
                        ({}, 'pop_recent'), ({'eval_benchmarks': [{'recommender': 'cb', 'params': {}}]}, 'item_knn')):
        with pytest.raises(ValueError):
            next(_estimator(**params).predict(input_fn, recommender=rec))
    assert not read


def test_model_level_checks():
    """NARModuleModel.recommend_baseline: data parallel raises NotImplementedError; an unknown or disabled suffix, bad
    positions, a top_n out of range and bad candidates raise ValueError - all before any device work."""
    from chameleon_recsys_b200.nar_model import NARModuleModel

    class Eng:
        V, world = 50, 1

        def resolve_candidates(self, candidates, buffer):
            from chameleon_recsys_b200.engine import NarEngine
            return NarEngine.resolve_candidates(self, candidates, buffer)
    model = types.SimpleNamespace(engine=Eng(), metrics_top_n=5)
    tabs = types.SimpleNamespace(enabled=['pop_recent', 'sknn'])
    feats = {'item_clicked': np.ones((2, 3), np.int64), 'session_size': np.array([4, 2])}
    buf = np.arange(1, 9)

    def call(rec='pop_recent', **kw):
        return NARModuleModel.recommend_baseline(model, rec, tabs, feats, buf, None, **kw)
    for rec in ('bogus', 'sr', 'item_knn'):
        with pytest.raises(ValueError):
            call(rec)
    for kw in ({'positions': 'first'}, {'top_n': 0}, {'top_n': 9}, {'top_n': 2.0}, {'candidates': [3, 3]},
               {'candidates': [0, 4]}, {'candidates': 'all'}, {'candidates': np.zeros(0, np.int64)}):
        with pytest.raises(ValueError):
            call(**kw)
    with pytest.raises(ValueError):                          # the kNN baselines keep a 64-bit position mask per session
        NARModuleModel.recommend_baseline(model, 'sknn', tabs, {'item_clicked': np.ones((1, 65), np.int64),
                                                                'session_size': np.array([3])}, buf, None)
    model.engine.world = 2
    with pytest.raises(NotImplementedError):
        call()
