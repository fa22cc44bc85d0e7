"""The baselines' unsampled evaluation on the H100 (DESIGN.md section 14): BaselineTables.rank_unsampled
(nar_baselines_rank_unsampled, nar_sknn_rank_unsampled) against oracle/unsampled_baselines_ref.py bit for bit, its ranks
against the sampled kernels' when the pool is one query's label and negatives, run-to-run and grid invariance, the switch
changing nothing else in Estimator.evaluate, and a G1-shaped evaluate."""
import copy
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.baselines_ref import SUFFIXES, BaselinesRef  # noqa: E402
from oracle.sknn_ref import SknnRef  # noqa: E402
from oracle.unsampled_baselines_ref import MISS, histogram, ranks  # noqa: E402

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
    batches; integer ACR rows, so cosines are exact too (test_baselines_kernels_gpu.py)."""

    def __init__(self, seed, V=60, absent=6, n_train=5, B=8, T1=7, ties=False, suffixes=ALL7):
        import torch
        from chameleon_recsys_b200.baselines import BaselineTables
        rs = np.random.RandomState(seed)
        self.V, self.rs = V, rs
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
        self.pop = rs.randint(0, 40, size=V).astype(np.int64)
        torch.cuda.synchronize()

    def queries(self, B, T, K=0, label_p=0.9):
        """item_clicked / label_next [B, T] (labels partly partners of the item in the pair table, partly never-clicked
        ids: not admissible), label_last_item [B], negatives [B, T, K]."""
        rs = self.rs
        ic = rs.randint(1, self.V, size=(B, T)).astype(np.int64)
        ln = rs.randint(1, self.V, size=(B, T)).astype(np.int64)
        partners = {}
        for (a, c) in self.ref.cooc:
            partners.setdefault(a, []).append(c)
        for b in range(B):
            for t in range(T):
                p = partners.get(int(ic[b, t]))
                if p and rs.rand() < 0.5:
                    ln[b, t] = p[rs.randint(len(p))]
        ic[0, 0] = 3                                              # the zero ACR row as a current click
        ln[rs.rand(B, T) > label_p] = 0
        last = rs.randint(1, self.V, size=B).astype(np.int64)
        neg = rs.randint(1, self.V, size=(B, T, K)).astype(np.int64)
        return ic, ln, last, neg

    def run(self, ic, ln, last, pool, top_n, neg=None, max_blocks=0, times=1):
        """score (builds the buffer histogram), then rank_unsampled ``times`` times -> (rank [7, B*T], hist [7, top_n+2],
        sampled out_ids [7, B*T, top_n])."""
        import torch
        B, T = ic.shape
        neg = np.zeros((B, T, 0), np.int64) if neg is None else neg
        n_rows = self.tab.n_rows
        met = torch.zeros(n_rows, 3, dtype=torch.float64, device='cuda')
        out_ids = torch.zeros(n_rows, B * T, top_n, dtype=torch.int64, device='cuda')
        self.tab.score(_dev(ic), _dev(ln), _dev(neg), self.buf, self.pop, top_n, met, out_ids=out_ids)
        hist = torch.zeros(n_rows, top_n + 2, dtype=torch.int64, device='cuda')
        rank = torch.full((n_rows, B * T), -7, dtype=torch.int32, device='cuda')
        ai = np.concatenate([ic, last.reshape(-1, 1)], axis=1)
        for _ in range(times):
            self.tab.rank_unsampled(_dev(ic), _dev(ln), _dev(ai), np.asarray(pool, dtype=np.int64), self.pop, top_n, hist,
                                    rank=rank, max_blocks=max_blocks)
        self.tab.check_errors()
        return rank.cpu().numpy(), hist.cpu().numpy(), out_ids.cpu().numpy()

    def oracle(self, sfx, ic, ln, last, pool):
        r = self.knn[sfx] if sfx in self.knn else self.ref
        return ranks(r, sfx, ic, ln, last, self.buf, self.pop, candidates=pool)


def _check(w, ic, ln, last, pool, top_n, **kw):
    from chameleon_recsys_b200.baselines import BaselineTables
    rank, hist, _ = w.run(ic, ln, last, pool, top_n, **kw)
    res = {}
    for sfx in w.suffixes:
        row = BaselineTables.row(sfx)
        want = w.oracle(sfx, ic, ln, last, pool)
        got = rank[row]
        np.testing.assert_array_equal(got[want['q']], want['rank'], err_msg=sfx)
        others = np.setdiff1d(np.arange(got.size), want['q'])
        assert (got[others] == -1).all(), sfx
        np.testing.assert_array_equal(hist[row], histogram(want, top_n), err_msg=sfx)
        res[sfx] = want
    for sfx in ALL7:
        if sfx not in w.suffixes and BaselineTables.row(sfx) < hist.shape[0]:
            assert not hist[BaselineTables.row(sfx)].any(), sfx
    return res


CASES = ['random', 'ties', 'n1', 'odd', 'stress', 'row_covers_pool']


@pytest.mark.parametrize('case', CASES)
def test_every_baseline_matches_the_oracle(case):
    """Per-query ranks and the histogram of all seven baselines bit for bit: planted ties (equal buffer counts, equal
    co-occurrence counts and sr weights with different first keys, a zero ACR row), labels a baseline does not admit,
    N = 1, N not a multiple of either CTA's stride, a pool of more than 10 000 ids, session rows (of 1 024 ids for the
    table baselines, with duplicates and zeros; 65 for the kNN ones) that exclude every competitor, and a session id
    repeated in the kNN rings."""
    top_n = 5
    if case == 'stress':
        w = World(7, V=12000, absent=10, n_train=8, B=20, T1=12)
        ic, ln, last, _ = w.queries(6, 5)
        pool = np.arange(1, 11500)
    elif case == 'row_covers_pool':
        w = World(8, suffixes=SUFFIXES)
        rs = np.random.RandomState(3)
        T = 1023
        ic = np.zeros((3, T), np.int64)
        pool = np.arange(1, 41)
        for b in range(3):
            row = np.concatenate([np.repeat(pool, 20), np.zeros(T - 800, np.int64)])
            ic[b] = row[rs.permutation(T)]
        ln = np.zeros((3, T), np.int64)
        ln[:, [0, 5, 900]] = rs.randint(1, 41, size=(3, 3))
        ic[:, [0, 5, 900]] = rs.randint(1, 41, size=(3, 3))
        last = np.zeros(3, np.int64)
        res = _check(w, ic, ln, last, pool, top_n)
        assert all((r['n_comp'] == 0).all() for r in res.values())
        w = World(9)                                               # and the kNN baselines' longest row: T = 64
        T = 64
        ic = np.zeros((2, T), np.int64)
        ic[:, :40] = np.arange(1, 41)
        ic[:, 40:] = rs.randint(0, 41, size=(2, T - 40))
        ic[:, 63] = 7                                              # a query's current click is nonzero
        ln = np.zeros((2, T), np.int64)
        ln[:, [3, 39, 63]] = rs.randint(1, 41, size=(2, 3))
        last = np.array([40, 0], np.int64)
        res = _check(w, ic, ln, last, pool, top_n)
        assert all((r['n_comp'] == 0).all() for r in res.values())
        return
    else:
        w = World({'random': 1, 'ties': 2, 'n1': 3, 'odd': 4}[case], ties=case == 'ties')
        ic, ln, last, _ = w.queries(9, 6)
        pool = {'random': None, 'ties': None, 'n1': np.array([int(ln[ln != 0][0])]),
                'odd': np.arange(1, 60)}[case]
        if pool is None:
            from oracle.unsampled_ref import pool as make_pool
            pool = make_pool(ic, last, w.buf)
        if case == 'odd':
            w2 = World(5, V=700)                                   # 613 pool ids: not a multiple of 256 nor of 64
            ic2, ln2, last2, _ = w2.queries(7, 5)
            _check(w2, ic2, ln2, last2, np.arange(1, 614), top_n)
    res = _check(w, ic, ln, last, pool, top_n)
    miss = {s: int((r['rank'] == MISS).sum()) for s, r in res.items()}
    if case == 'random':
        assert all(miss[s] > 0 for s in ALL7 if s != 'cb'), miss       # labels some baseline does not admit
    if case == 'ties':
        for sfx in ('pop_recent', 'coocurrent', 'sr'):
            assert (res[sfx]['rank_lo'] > res[sfx]['rank_hi']).any(), sfx     # the label ties a competitor


def test_rank_against_the_negatives_is_the_sampled_rank():
    """For every query without a zero-padded negative (and none in its session row), ranking against {label} | its
    negatives gives each baseline's sampled rank as the sampled kernels wrote it to out_ids, or a miss: exactly."""
    from chameleon_recsys_b200.baselines import BaselineTables
    top_n = 4
    w = World(12)
    ic, ln, last, neg = w.queries(6, 6, K=9)
    neg[0, 0, 0] = 0                                              # a zero-padded negative: not compared
    _, _, out = w.run(ic, ln, last, np.arange(1, w.V), top_n, neg=neg)
    B, T = ic.shape
    checked = 0
    for q in np.flatnonzero(ln.reshape(-1)):
        b = q // T
        negs = neg.reshape(B * T, -1)[q]
        if not negs.all() or np.isin(negs, np.append(ic[b], last[b])).any():
            continue
        lab = ln.reshape(-1)[q]
        rank, _, _ = w.run(ic, ln, last, np.unique(np.append(negs, lab)), top_n, neg=neg)
        for sfx in ALL7:
            row = BaselineTables.row(sfx)
            hit = np.flatnonzero(out[row, q] == lab)
            assert min(int(rank[row, q]), top_n) == (int(hit[0]) if hit.size else top_n), (sfx, q)
        checked += 1
    assert checked >= 5, checked


def test_histograms_are_the_same_every_run_and_for_one_cta():
    w = World(13, V=300, B=20)
    ic, ln, last, _ = w.queries(30, 6)
    from oracle.unsampled_ref import pool as make_pool
    pool = make_pool(ic, last, w.buf)
    r0, h0, _ = w.run(ic, ln, last, pool, 5)
    r1, h1, _ = w.run(ic, ln, last, pool, 5, times=3)
    r2, h2, _ = w.run(ic, ln, last, pool, 5, max_blocks=1)
    assert np.array_equal(r0, r1) and np.array_equal(r0, r2)
    assert np.array_equal(3 * h0, h1) and np.array_equal(h0, h2)


def _problem():
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 2)
    return pb


def test_the_switch_changes_nothing_else(tmp_path):
    """From one checkpoint, evaluate with the switch off and on, with every other evaluation extension on (the model's
    unsampled metrics included): the only new keys are the baselines' unsampled ones; every other key has the same value
    - bit for bit, except the loss and the model's MRR, held to the bounds of the existing switch test -, the
    candidates per query included; the negatives log and the ClickedItemsState afterwards are the same."""
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.eval_metrics import UNSAMPLED_KEYS, unsampled_bench_keys
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    d = str(tmp_path)
    all7 = tuple({'recommender': s, 'params': {}} for s in ALL7)

    def est(state, on, **extra):
        hp = pb.hp.copy(eval_benchmarks=all7, eval_extended_metrics=True, eval_metrics_by_session_position=True,
                        eval_unsampled_metrics=True, eval_unsampled_benchmarks=on)
        return build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                               pb.session_features_config, hp, state, device=0, **extra)
    est(pb.clicked_items_state, False).train(lambda: iter(train_batches))
    saved = ckpt.load(ckpt.latest_checkpoint(d))
    st = pb.clicked_items_state
    runs, logs, states = {}, {}, {}
    for name, on in (('off', False), ('on', True)):
        fresh = ClickedItemsState(st.recent_clicks_buffer_hours, st.recent_clicks_buffer_max_size,
                                  st.recent_clicks_for_normalization, st.num_items)
        for f in ckpt.STATE_FIELDS:
            setattr(fresh, f, np.array(saved['state'][f]))
        logs[name] = []
        runs[name] = est(fresh, on, sessions_negative_items_log=logs[name]).evaluate(lambda: iter(eval_batches))
        states[name] = {f: copy.deepcopy(getattr(fresh, f)) for f in ckpt.STATE_FIELDS}
    off, on = runs['off'], runs['on']
    new = {k for s in ALL7 for k in unsampled_bench_keys(s)}
    assert set(on) - set(off) == new
    assert all(np.isfinite(on[k]) for k in new)
    assert 'unsampled_candidates_per_query' in off and set(UNSAMPLED_KEYS) <= set(off)
    positions = max(np.asarray(f['item_clicked']).size for f, _ in eval_batches)
    queries = sum(int(np.count_nonzero(l['label_next_item'])) for _, l in eval_batches)
    tol = {'loss': 2 * (positions - 1) * 2.0 ** -24, 'mrr_at_n': 2 * queries * 2.0 ** -53}
    for k, v in off.items():
        if k in tol:
            assert abs(on[k] - v) <= tol[k] * abs(v), (k, on[k], v)
        else:
            assert on[k] == v or (np.isnan(v) and np.isnan(on[k])), (k, on[k], v)
    assert logs['on'] == logs['off'] and len(logs['on']) > 0
    for f in ckpt.STATE_FIELDS:
        assert np.array_equal(np.asarray(states['on'][f]), np.asarray(states['off'][f])), f
    torch.cuda.synchronize()


def test_g1_estimator_evaluate():
    """A G1-shaped batch through Estimator.evaluate with all seven baselines: finite keys, and the mean competitor count
    is the oracle's for the same batch and state."""
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.eval_metrics import unsampled_bench_keys
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from oracle.unsampled_ref import competitor_sets
    pb = make_problem('g1', profile='B')
    warm_state(pb, 20)
    it = pb.input_fn()
    train = [it.get_next() for _ in range(3)]
    batch = it.get_next()
    all7 = tuple({'recommender': s, 'params': {}} for s in ALL7)
    hp = pb.hp.copy(eval_benchmarks=all7, eval_unsampled_benchmarks=True)
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, hp, pb.clicked_items_state, device=0)
    est.train(lambda: iter(train))
    f, l = batch
    sets = competitor_sets(f['item_clicked'], l['label_last_item'], pb.clicked_items_state.get_recent_clicks_buffer())
    qs, _ = np.nonzero(np.asarray(l['label_next_item']))
    want = float(sum(sets[b].size for b in qs)) / qs.size
    ev = est.evaluate(lambda: iter([batch]))
    for s in ALL7:
        for k in unsampled_bench_keys(s):
            assert np.isfinite(ev[k]), k
    assert ev['unsampled_candidates_per_query'] == want
    print('G1 batch: %d queries, %.1f competitors per query; unsampled / sampled HR@n: %s'
          % (qs.size, want, ', '.join('%s %.4f / %.4f' % (s, ev['unsampled_hitrate_at_n_' + s], ev['hitrate_at_n_' + s])
                                       for s in ALL7)))
