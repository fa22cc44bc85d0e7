"""oracle/sknn_ref.py against the reference's own session-based kNN recommender (tests/golden/make_sknn_golden.py ran
session_knn.py and ClickedItemsState in the hook's order, for 'div' + cosine, 'same' + jaccard and both decays without
the 'recent' cut).  No GPU."""
import os
from collections import Counter

import numpy as np
import pytest

from oracle.sknn_ref import SknnRef

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'sknn_golden.npz')


@pytest.fixture(scope='module')
def g():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _all_items(g, name):
    return np.concatenate([g[name + '_ic'], g[name + '_last']], axis=1)


def _ref(g, c):
    S, C, NN = g['params'][c].tolist()
    return SknnRef(S, C, NN, str(g['similarity'][c]), str(g['decay'][c]))


def _configs(g):
    return range(len(g['params']))


def _check_export(got, g, prefix):
    n = got['ids'].size
    np.testing.assert_array_equal(got['ids'], g[prefix + '_ids'], err_msg=prefix)
    W = g[prefix + '_items'].shape[1]
    items = np.zeros((n, W), dtype=np.int64)
    live = np.zeros((n, W), dtype=bool)
    items[:, :got['items'].shape[1]] = got['items']
    live[:, :got['live'].shape[1]] = got['live']
    np.testing.assert_array_equal(items, g[prefix + '_items'], err_msg=prefix)
    np.testing.assert_array_equal(live, g[prefix + '_live'], err_msg=prefix)


def test_fixture_exercises_every_branch(g):
    V, B, T, K, top_n, n_train, n_eval = g['cfg'].tolist()
    assert np.array_equal(g['train1_sid'], g['train2_sid'])                      # a batch trained twice
    assert np.all(np.diff(g['train3_sid']) < 0)                                   # ids going backwards
    ge1 = 0                                          # similarities >= 1.0 dropped (any parameter set)
    for c in _configs(g):
        ref = _ref(g, c)
        evicted = cut = nn_cut = misses = 0
        for s in range(n_train):
            before = len(ref.buffer)
            ref.update(g['train%d_sid' % s], _all_items(g, 'train%d' % s))
            evicted += before + B - len(ref.buffer)
        assert evicted > 0
        assert not g['c%d_train_live' % c][g['c%d_train_items' % c] > 0].all()   # the discard quirk left dead items
        misses += sum(ref.find(int(s)) == -1 for s, _ in ref.buffer)
        for s in range(n_eval):
            e = 'eval%d' % s
            ic, ln = g[e + '_ic'], g[e + '_ln']
            for b, t in zip(*np.nonzero(ln)):
                P = ic[b, :t + 1].tolist()
                m = Counter()
                for x in P:
                    for sid in ref.map.get(int(x), ()):
                        if ref.find(sid) != -1:
                            m[sid] += 1
                cut += ref.C > 0 and sum(m.values()) > ref.C
                full = ref.neighbors(P, cut=False)
                nn_cut += len(full) > ref.NN
                for sid, k in ref.candidates(P).items():
                    ge1 += ref._sim(P, ref.buffer[ref.find(sid)][1]) >= 1.0
            ref.update(g[e + '_sid'], _all_items(g, e))
        assert misses > 0, c
        assert nn_cut > 0, c
        if ref.C > 0:
            assert cut > 0, c
    assert ge1 > 0


@pytest.mark.parametrize('c', range(4))
def test_buffer_matches_reference(g, c):
    V, B, T, K, top_n, n_train, n_eval = g['cfg'].tolist()
    ref = _ref(g, c)
    for s in range(n_train):
        ref.update(g['train%d_sid' % s], _all_items(g, 'train%d' % s))
    _check_export(ref.export(), g, 'c%d_train' % c)
    ref.snapshot()
    for s in range(n_eval):
        ref.update(g['eval%d_sid' % s], _all_items(g, 'eval%d' % s))
    _check_export(ref.export(), g, 'c%d_eval' % c)
    ref.restore()
    _check_export(ref.export(), g, 'c%d_restored' % c)


def _groups(lst):
    """[(sim, Counter of ids)] of consecutive equal-similarity runs."""
    out = []
    for sid, sim in lst:
        if out and out[-1][0] == sim:
            out[-1][1][sid] += 1
        else:
            out.append((sim, Counter({sid: 1})))
    return out


def _neighbors_agree(want, got, full):
    """The reference's list and the oracle's hold the same copies, in order except within equal-similarity groups; the
    group at the nearest-neighbour cut may take different copies of that group (the reference's order there is set
    iteration order), but as many, all from the group."""
    if len(want) != len(got):
        return False
    gw, gg = _groups(want), _groups(got)
    if [s for s, _ in gw] != [s for s, _ in gg]:
        return False
    for i, ((s, cw), (_, cg)) in enumerate(zip(gw, gg)):
        if cw == cg:
            continue
        if i != len(gw) - 1 or len(full) == len(want):
            return False
        pool = Counter(sid for sid, v in full if v == s)
        if sum(cw.values()) != sum(cg.values()) or cw - pool or cg - pool:
            return False
    return True


@pytest.mark.parametrize('c', range(4))
def test_neighbors_predictions_and_metrics_match_reference(g, c):
    """Neighbour lists as multisets of (id, sim) with == on the similarities; predictions id for id except within
    equal-score groups; HR / MRR exact where no order of ties matters, else inside the oracle's bounds."""
    V, B, T, K, top_n, n_train, n_eval = g['cfg'].tolist()
    ref = _ref(g, c)
    for s in range(n_train):
        ref.update(g['train%d_sid' % s], _all_items(g, 'train%d' % s))
    hits = rr = cnt = lo_h = hi_h = lo_r = hi_r = 0.0
    split = compared = 0
    for s in range(n_eval):
        e = 'eval%d' % s
        p = 'c%d_%s' % (c, e)
        ic, ln, neg = g[e + '_ic'], g[e + '_ln'], g[e + '_neg']
        want_pred = g[p + '_pred']
        off, nb_sid, nb_sim = g[p + '_nb_off'], g[p + '_nb_sid'], g[p + '_nb_sim']
        r = ref.score(ic, ln, neg, top_n)
        q = 0
        for b in range(B):
            for t in range(T):
                if ln[b, t] == 0:
                    assert off[q + 1] == off[q]
                    q += 1
                    continue
                P = ic[b, :t + 1].tolist()
                want = list(zip(nb_sid[off[q]:off[q + 1]].tolist(), nb_sim[off[q]:off[q + 1]].tolist()))
                got = ref.neighbors(P)
                q += 1
                assert _neighbors_agree(want, got, ref.neighbors(P, cut=False)), (c, e, b, t)
                if Counter(want) != Counter(got):
                    split += 1                   # a cut inside an equal-similarity group: item scores may differ
                    continue
                compared += 1
                scores, _ = ref.item_scores(P)
                wp, gp = want_pred[b, t].tolist(), r['ids'][b * T + t].tolist()
                assert [scores.get(x, 0) for x in wp] == [scores.get(x, 0) for x in gp], (c, e, b, t)
                for i in range(top_n):
                    # equal-score groups: the same score rank by rank; ids may differ only where the score ties another
                    if wp[i] != gp[i]:
                        tied = [x for x in scores if scores[x] == scores[gp[i]]]
                        assert len(tied) > 1 and wp[i] in tied, (c, e, b, t)
        hits += r['hits']; rr += r['rr']; cnt += r['count']
        lo_h += r['bounds'][0]; hi_h += r['bounds'][1]; lo_r += r['bounds'][2]; hi_r += r['bounds'][3]
        ref.update(g[e + '_sid'], _all_items(g, e))
    assert compared > 5 * split, (compared, split)
    ref_hr, ref_mrr = float(g['c%d_hr' % c]), float(g['c%d_mrr' % c])
    if split == 0:
        assert lo_h / cnt - 1e-12 <= ref_hr <= hi_h / cnt + 1e-12
        assert lo_r / cnt - 1e-12 <= ref_mrr <= hi_r / cnt + 1e-12
        if lo_h == hi_h and lo_r == hi_r:
            assert abs(hits / cnt - ref_hr) < 1e-12 and abs(rr / cnt - ref_mrr) < 1e-12
    else:
        assert abs(hits / cnt - ref_hr) <= split / cnt + (hi_h - lo_h) / cnt + 1e-12
