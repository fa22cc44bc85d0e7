"""The baselines' recommendations on the H100 (DESIGN.md section 16): BaselineTables.recommend (nar_baselines_recommend,
nar_sknn_recommend) against oracle/baseline_predict_ref.py bit for bit, ids and float64 scores; run-to-run and grid
invariance; agreement with the sampled scoring's top-n lists; nothing written; Estimator.predict(recommender=...) after
train() and from a checkpoint; the argument errors."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.baseline_predict_ref import recommend as ref_recommend  # noqa: E402
from oracle.baselines_ref import SUFFIXES, BaselinesRef  # noqa: E402
from oracle.sknn_ref import SknnRef  # noqa: E402

pytestmark = pytest.mark.gpu

ALL7 = SUFFIXES + ('v-sknn', 'sknn')
KNN_PARAMS = {'v-sknn': dict(sessions_buffer_size=24, candidate_sessions_sample_size=14,
                             nearest_neighbor_session_for_scoring=7, similarity='cosine'),
              'sknn': dict(sessions_buffer_size=24, candidate_sessions_sample_size=0,
                           nearest_neighbor_session_for_scoring=7, similarity='jaccard')}
ACR_DIM, ACR_LD = 24, 32


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class World:
    """BaselineTables (all seven baselines, item_knn with alpha 1: exact scores) and the oracles, trained on the same
    batches; integer ACR rows, so cosines are exact too.  Ids >= V - absent are never clicked: no baseline but cb admits
    them."""

    def __init__(self, seed, V=60, absent=6, n_train=5, B=8, T1=7, ties=False, suffixes=ALL7):
        import torch
        from chameleon_recsys_b200.baselines import BaselineTables
        rs = np.random.RandomState(seed)
        self.V, self.rs, self.absent = V, rs, absent
        acr = np.zeros((V, ACR_LD), dtype=np.float32)
        acr[:, :ACR_DIM] = rs.randint(-3, 4, size=(V, ACR_DIM))
        acr[0] = 0.0
        acr[3] = 0.0                                              # a zero row: its cosines are 0
        clfs = [{'recommender': s, 'params': ({'reg_lambda': 20, 'alpha': 1.0} if s == 'item_knn' else
                                              KNN_PARAMS.get(s, {}))} for s in suffixes]
        self.tab = BaselineTables(clfs, V, acr=_dev(acr), acr_dim=ACR_DIM)
        self.ref = BaselinesRef(V, acr=acr[:, :ACR_DIM].astype(np.float64), reg_lambda=20, alpha=1.0)
        self.knn = {s: SknnRef(first_session_clicks_decay='div' if s == 'v-sknn' else 'same', **KNN_PARAMS[s])
                    for s in suffixes if s in KNN_PARAMS}
        self.suffixes = suffixes
        batches, sid0 = [], 100
        for i in range(n_train):
            if i == 2 and batches:
                batches.append(batches[-1])                       # the same session ids again: repeated in the ring
                continue
            L = 3 if ties else T1
            ai = np.zeros((B, L), dtype=np.int64)
            for b in range(B):
                n = rs.randint(2, L + 1)
                ai[b, :n] = rs.randint(1, V - absent, size=n)
            sid = sid0 + 10 * np.arange(B, dtype=np.int64) + rs.randint(0, 5, size=B)
            sid0 += 10 * B
            batches.append((sid, ai))
        for sid, ai in batches:
            self.tab.update(_dev(ai), session_ids=sid)
            self.ref.update(ai)
            for r in self.knn.values():
                r.update(sid, ai)
        if ties:
            self.buf = rs.permutation(np.arange(1, V - absent)).astype(np.int64)   # every count 1: first index decides
        else:
            self.buf = np.where(rs.rand(4 * B) < 0.8, rs.randint(1, V - absent, size=4 * B), 0).astype(np.int64)
        # pop + reg_lambda a power of two: CUDA's pow (within 2 ulp) and numpy's are both exact there, so the item_knn
        # scores can be compared bit for bit
        self.pop = rs.choice([12, 44, 108, 236], size=V).astype(np.int64)
        torch.cuda.synchronize()

    def clicks(self, B, T, zeros=0.2):
        """item_clicked [B, T] with trailing zero padding, and the flat positions of its nonzero clicks."""
        ic = self.rs.randint(1, self.V - self.absent, size=(B, T)).astype(np.int64)
        ic[0, 0] = 3                                              # the zero ACR row as a current click
        for b in range(1, B):
            ic[b, max(1, int(T * (1 - zeros * self.rs.rand()))):] = 0
        return ic, np.flatnonzero(ic.reshape(-1)).astype(np.int32)

    def run(self, sfx, ic, q_pos, cand, top_n, exclude=True, max_blocks=0):
        import torch
        ids, sc = self.tab.recommend(sfx, _dev(ic), _dev(q_pos), _dev(np.sort(cand)), self.buf, self.pop, top_n,
                                     exclude_session_clicks=exclude, max_blocks=max_blocks)
        self.tab.check_errors()
        torch.cuda.synchronize()
        return ids.cpu().numpy(), sc.cpu().numpy()

    def oracle(self, sfx, ic, q_pos, cand, top_n, exclude=True):
        r = self.knn[sfx] if sfx in self.knn else self.ref
        return ref_recommend(r, sfx, ic, q_pos, cand, top_n, buffer=self.buf, articles_pop=self.pop, exclude=exclude)


def _same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def _check(w, ic, q_pos, cand, top_n, exclude=True):
    """Every baseline of ``w`` against the oracle: ids and the bits of the scores.  -> {sfx: admissible per query}."""
    adm = {}
    for sfx in w.suffixes:
        ids, sc = w.run(sfx, ic, q_pos, cand, top_n, exclude)
        want_ids, want_sc = w.oracle(sfx, ic, q_pos, cand, top_n, exclude)
        np.testing.assert_array_equal(ids, want_ids, err_msg=sfx)
        assert _same_bits(np.where(ids == 0, np.nan, sc), want_sc), sfx
        assert np.isnan(sc[ids == 0]).all(), sfx
        adm[sfx] = (ids != 0).sum(axis=1)
    return adm


CASES = ['buffer', 'ties', 'absent', 'n1', 'odd', 'catalog', 'no_exclusion', 'top1', 'wide', 'row_covers']


@pytest.mark.parametrize('case', CASES)
def test_every_baseline_matches_the_oracle(case):
    """All seven baselines bit for bit, ids and scores, at every nonzero click: the buffer's ids, planted ties (equal
    buffer counts, equal co-occurrence counts, a zero ACR row), candidates no baseline but cb admits, N = 1, N = 613 (not a
    multiple of either CTA's tile), the 46 033-id catalog, exclusion off, top_n = 1, top_n past the admissible ids, and
    session rows that exclude every candidate (1 024 positions for the table baselines, 64 for the kNN ones)."""
    top_n = {'top1': 1, 'wide': 40}.get(case, 5)
    if case == 'catalog':
        w = World(7, V=46034, absent=10, n_train=8, B=20, T1=12)
        ic, q_pos = w.clicks(6, 5)
        _check(w, ic, q_pos, np.arange(1, 46034), top_n)
        return
    if case == 'row_covers':
        w = World(8, suffixes=SUFFIXES)
        rs = np.random.RandomState(3)
        T = 1024
        cand = np.arange(1, 41)
        ic = np.repeat(cand, 26)[:T][None, :].repeat(2, axis=0)
        ic[0] = ic[0][rs.permutation(T)]
        q_pos = np.array([T - 1, 2 * T - 1], np.int32)          # the last position: every candidate is a click before it
        adm = _check(w, ic, q_pos, cand, top_n)
        assert all((a == 0).all() for a in adm.values())
        w = World(9, suffixes=('v-sknn', 'sknn'))
        T = 64
        ic = np.tile(np.arange(1, 41), 2)[:T][None, :].repeat(2, axis=0)
        adm = _check(w, ic, np.array([T - 1, 2 * T - 1], np.int32), cand, top_n)
        assert all((a == 0).all() for a in adm.values())
        return
    w = World({'buffer': 1, 'ties': 2, 'absent': 3, 'n1': 4, 'odd': 5, 'no_exclusion': 6, 'top1': 10,
               'wide': 11}[case], V=700 if case == 'odd' else 60, ties=case == 'ties')
    ic, q_pos = w.clicks(9, 6)
    buf_ids = np.unique(w.buf[w.buf != 0])
    cand = {'absent': np.arange(w.V - w.absent, w.V), 'n1': np.array([int(ic[0, 1])]), 'odd': np.arange(1, 614),
            'wide': np.arange(1, w.V)}.get(case, buf_ids)
    adm = _check(w, ic, q_pos, cand, top_n, exclude=case != 'no_exclusion')
    if case == 'absent':
        assert all((adm[s] == 0).all() for s in ALL7 if s != 'cb') and (adm['cb'] == top_n).all()
    if case == 'wide':
        assert all((adm[s] < top_n).any() for s in ALL7 if s != 'cb') and (adm['cb'] == top_n).all(), adm
    if case == 'ties':
        ids, sc = w.run('pop_recent', ic, q_pos, cand, top_n)
        assert (sc[:, 0] == sc[:, 1]).all()                      # every count is 1: the buffer order decides


def test_same_bits_every_run_and_for_one_cta():
    w = World(13, V=300, B=20)
    ic, q_pos = w.clicks(30, 6)
    cand = np.arange(1, 300)
    for sfx in ALL7:
        a = w.run(sfx, ic, q_pos, cand, 7)
        b = w.run(sfx, ic, q_pos, cand, 7)
        c = w.run(sfx, ic, q_pos, cand, 7, max_blocks=1)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[0], c[0]), sfx
        assert _same_bits(a[1], b[1]) and _same_bits(a[1], c[1]), sfx


@pytest.mark.parametrize('top_n', [2, 3, 255, 256, 257, 1024])
def test_top_n_around_the_tile_and_the_list_bound(top_n):
    """top_n just below, at and above one tile (256 candidates), small values where the list first fills within a tile,
    and the largest list: every baseline bit for bit against the oracle over 1 299 candidates, and the same bits with one
    CTA (one CTA walks every query after another through the same shared state)."""
    w = World(21, V=1400, absent=40)
    ic, q_pos = w.clicks(6, 6)
    cand = np.arange(1, 1300)
    _check(w, ic, q_pos, cand, top_n)
    for sfx in ALL7:
        a = w.run(sfx, ic, q_pos, cand, top_n)
        c = w.run(sfx, ic, q_pos, cand, top_n, max_blocks=1)
        assert np.array_equal(a[0], c[0]) and _same_bits(a[1], c[1]), sfx


def test_unsorted_or_repeated_candidates_raise():
    """Candidates that are not strictly ascending set the error flag on the device; check_errors raises ValueError and
    clears it, so the tables serve the next call."""
    w = World(22)
    ic, q_pos = w.clicks(4, 5)
    for sfx in ('pop_recent', 'cb', 'v-sknn'):
        for cand in (np.array([5, 4, 9]), np.array([4, 4, 9])):
            w.tab.recommend(sfx, _dev(ic), _dev(q_pos), _dev(cand), w.buf, w.pop, 2)
            with pytest.raises(ValueError):
                w.tab.check_errors()
        ids, _ = w.run(sfx, ic, q_pos, np.arange(1, w.V), 3)
        np.testing.assert_array_equal(ids, w.oracle(sfx, ic, q_pos, np.arange(1, w.V), 3)[0], err_msg=sfx)


def test_label_and_negatives_give_the_sampled_top_n():
    """A query whose candidates are its label and its logged negatives, with exclusion off, gets the ids the sampled
    scoring wrote to out_ids for that query."""
    import torch
    from chameleon_recsys_b200.baselines import BaselineTables
    top_n = 4
    w = World(12)
    B, T, K = 6, 6, 9
    ic, _ = w.clicks(B, T, zeros=0.0)
    ln = w.rs.randint(1, w.V, size=(B, T)).astype(np.int64)
    neg = w.rs.randint(1, w.V, size=(B, T, K)).astype(np.int64)
    met = torch.zeros(w.tab.n_rows, 3, dtype=torch.float64, device='cuda')
    out = torch.zeros(w.tab.n_rows, B * T, top_n, dtype=torch.int64, device='cuda')
    w.tab.score(_dev(ic), _dev(ln), _dev(neg), w.buf, w.pop, top_n, met, out_ids=out)
    out = out.cpu().numpy()
    for q in range(B * T):
        cand = np.unique(np.append(neg.reshape(B * T, K)[q], ln.reshape(-1)[q]))
        for sfx in ALL7:
            ids, _ = w.run(sfx, ic, np.array([q], np.int32), cand, top_n, exclude=False)
            assert np.array_equal(ids[0], out[BaselineTables.row(sfx), q]), (sfx, q)


def test_predict_writes_nothing():
    """The pair table, its entry count, the kNN rings and the error flag are byte-identical after recommend calls of
    every baseline."""
    import torch
    w = World(14)
    ic, q_pos = w.clicks(8, 6)
    t = w.tab

    def snap():
        torch.cuda.synchronize()
        out = [x.clone() for x in t._tables()] + [t.count.clone(), t.err.clone()]
        for ring in t.knn.values():
            out += [ring.ids.clone(), ring.lens.clone(), ring.items.clone()]
        return out, (t.cap, t.batch_seq, [(r.head, r.count) for r in t.knn.values()])
    before, meta = snap()
    for sfx in ALL7:
        w.run(sfx, ic, q_pos, np.arange(1, w.V), 5)
    after, meta2 = snap()
    assert meta == meta2 and all(torch.equal(a, b) for a, b in zip(before, after))


def _problem():
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 2)
    return pb


def test_estimator_predict_after_train_and_from_a_checkpoint(tmp_path):
    """Estimator.predict(recommender=s) for every baseline and both position modes: the same dicts right after train()
    and from the checkpoint in a fresh Estimator and state; ClickedItemsState and the weights unchanged; the model's own
    predict still yields its probabilities.  Then the argument errors."""
    import copy
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.estimator import build_estimator
    pb = _problem()
    it = pb.input_fn()
    train = [it.get_next() for _ in range(6)]
    batches = [it.get_next() for _ in range(2)]
    d = str(tmp_path)
    all7 = tuple({'recommender': s, 'params': {}} for s in ALL7)

    def est(state):
        return build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                               pb.session_features_config, pb.hp.copy(eval_benchmarks=all7), state, device=0)
    e1 = est(pb.clicked_items_state)
    e1.train(lambda: iter(train))
    saved = ckpt.load(ckpt.latest_checkpoint(d))
    st = pb.clicked_items_state
    fresh = ClickedItemsState(st.recent_clicks_buffer_hours, st.recent_clicks_buffer_max_size,
                              st.recent_clicks_for_normalization, st.num_items)
    for f in ckpt.STATE_FIELDS:
        setattr(fresh, f, np.array(saved['state'][f]))
    e2 = est(fresh)
    before = {f: copy.deepcopy(getattr(st, f)) for f in ckpt.STATE_FIELDS}
    w0 = e1.model.engine.get_params()
    for sfx in ALL7:
        for positions in ('last', 'all'):
            kw = dict(recommender=sfx, positions=positions, candidates='catalog' if sfx == 'cb' else None)
            a = list(e1.predict(lambda: iter(batches), **kw))
            b = list(e2.predict(lambda: iter(batches), **kw))
            assert len(a) == len(b) == sum(np.asarray(f['item_clicked']).shape[0] for f, _ in batches)
            for x, y in zip(a, b):
                assert set(x) == {'session_id', 'predicted_item_ids', 'predicted_item_scores'}
                assert np.array_equal(x['predicted_item_ids'], y['predicted_item_ids']), (sfx, positions)
                assert _same_bits(x['predicted_item_scores'], y['predicted_item_scores']), (sfx, positions)
                assert x['predicted_item_scores'].dtype == np.float64
            if positions == 'last':
                assert any(r['predicted_item_ids'].size and r['predicted_item_ids'][0] != 0 for r in a), sfx
    for f in ckpt.STATE_FIELDS:
        assert np.array_equal(np.asarray(getattr(st, f)), np.asarray(before[f])), f
    w1 = e1.model.engine.get_params()
    assert all(np.array_equal(w0[k], w1[k]) for k in w0)
    assert 'predicted_item_probs' in next(iter(e1.predict(lambda: iter(batches))))
    for kw in ({'recommender': 'vsknn'}, {'recommender': 'pop_recent', 'top_n': 0},
               {'recommender': 'pop_recent', 'top_n': 5000}, {'recommender': 'sr', 'candidates': [0, 1]},
               {'recommender': 'cb', 'candidates': [2, 2]}):
        with pytest.raises(ValueError):
            next(e1.predict(lambda: iter(batches), **kw))
    other = build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                            pb.session_features_config, pb.hp.copy(eval_benchmarks=('pop_recent',)), fresh, device=0)
    with pytest.raises(ValueError):
        next(other.predict(lambda: iter(batches), recommender='sr'))
    torch.cuda.synchronize()


def test_g1_catalog_predict():
    """G1 (46 033 articles, batch 256): every baseline recommends from the whole catalog; the lists hold distinct
    admissible ids in descending score order, and a session's own clicks never appear."""
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('g1', profile='B')
    warm_state(pb, 10)
    it = pb.input_fn()
    train = [it.get_next() for _ in range(3)]
    batch = it.get_next()
    all7 = tuple({'recommender': s, 'params': {}} for s in ALL7)
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, pb.hp.copy(eval_benchmarks=all7), pb.clicked_items_state, device=0)
    est.train(lambda: iter(train))
    f = batch[0]
    for sfx in ALL7:
        rows = list(est.predict(lambda: iter([batch]), recommender=sfx, candidates='catalog', top_n=10))
        for b, r in enumerate(rows):
            ids, sc = r['predicted_item_ids'], r['predicted_item_scores']
            if ids.size == 0:
                continue
            live = ids[ids != 0]
            assert len(set(live.tolist())) == live.size and (np.diff(sc[ids != 0]) <= 0).all(), sfx
            assert not np.isin(live, np.asarray(f['item_clicked'])[b]).any(), sfx
