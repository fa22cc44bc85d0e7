"""Generate tests/golden/baseline_predict_golden.npz by running the REFERENCE baseline recommenders
(benchmarks/{recently_popular,item_cooccurrences,item_knn,content_based,sequential_rules,session_knn}.py) and
ClickedItemsState, unmodified, in the order of the evaluation hook (nar_model.py:1609-1650), and asking each for its
recommendations with its own ``predict(users_ids, sessions_items, topk, valid_items)`` (benchmarks.py:32): every query
(b, t) with a nonzero click gets as valid items the candidate set (the distinct ids of the recent-clicks buffer, or the
whole catalog) minus the session's clicks item_clicked[b, 0..t] (or not, exclusion off), padded with its first valid id
(DESIGN.md section 16).  topk is the metric's n and a width larger than any valid set, so the padding with 0 shows.
Seeded synthetic train batches first (every recommender learns, the state absorbs the batch), then eval batches
(predict, then learn and absorb).  The reference package is loaded through the shim of make_baselines_golden.py; for the
session kNN baselines the fixture also holds each query's ``find_neighbors`` list.  Run once in the build container; the
.npz is committed."""
import importlib
import os
import sys
import types

import numpy as np
import pandas  # noqa: F401  (imported before the pytz stub: pandas probes pytz's version)

for name in ('tensorflow', 'pytz', 'ua_parser', 'ua_parser.user_agent_parser'):
    sys.modules[name] = types.ModuleType(name)
sys.modules['ua_parser'].user_agent_parser = sys.modules['ua_parser.user_agent_parser']
if not hasattr(np, 'asfarray'):
    # NDCG calls np.asfarray, which NumPy 2.0 removed; this is its NumPy 1.x definition
    np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)

REF_DIR = '/root/reference/nar_module/nar'
pkg = types.ModuleType('refnar')
pkg.__path__ = [REF_DIR]
sys.modules['refnar'] = pkg
cis = importlib.import_module('refnar.clicked_items_state')
bm = importlib.import_module('refnar.benchmarks')
metrics = importlib.import_module('refnar.metrics')

V, B, T, TOP_N = 40, 6, 8, 5
N_TRAIN, N_EVAL = 5, 3
KNN = {'v-sknn': (20, 12, 6, 'cosine', 'div'), 'sknn': (20, 12, 6, 'jaccard', 'same')}
rs = np.random.RandomState(31)
acr = rs.randn(V, 8)
acr[0] = 0.0
acr[7] = 0.0                                                # a zero row among the articles: cosine 0 against everything


class Scipy2018CSR(cis.csr_matrix):
    """The co-occurrence matrix as the reference's SciPy had it (see make_baselines_golden.py)."""

    def __truediv__(self, other):
        if isinstance(other, np.ndarray):
            return np.asmatrix(self.toarray() / other)
        return super().__truediv__(other)


state = cis.ClickedItemsState(1.0, 30, 20, V)
state.items_coocurrences = Scipy2018CSR(state.items_coocurrences)
clfs = [bm.RecentlyPopularRecommender(state, {}, []),
        bm.ItemCooccurrenceRecommender(state, {}, []),
        bm.ItemKNNRecommender(state, {'reg_lambda': 20, 'alpha': 0.75}, []),
        bm.ContentBasedRecommender(state, {'content_article_embeddings_matrix': acr}, []),
        bm.SequentialRulesRecommender(state, {'max_clicks_dist': 10, 'dist_between_clicks_decay': 'div'}, [])]
for S, C, NN, sim, decay in KNN.values():
    clfs.append(bm.SessionBasedKNNRecommender(state, {
        'sessions_buffer_size': S, 'candidate_sessions_sample_size': C, 'sampling_strategy': 'recent',
        'nearest_neighbor_session_for_scoring': NN, 'similarity': sim, 'first_session_clicks_decay': decay}, []))
suffixes = [c.get_clf_suffix() for c in clfs]
assert suffixes[5:] == list(KNN)
out = {'cfg': np.array([V, B, T, TOP_N, N_TRAIN, N_EVAL], dtype=np.int64), 'acr': acr,
       'knn_params': np.array([v[:3] for v in KNN.values()], dtype=np.int64),
       'knn_similarity': np.array([v[3] for v in KNN.values()]), 'knn_decay': np.array([v[4] for v in KNN.values()])}
t0 = 1506826800000


def make_batch(step):
    ic = np.zeros((B, T), dtype=np.int64)
    ts = np.zeros((B, T), dtype=np.int64)
    ln = np.zeros((B, T), dtype=np.int64)
    last = np.zeros((B, 1), dtype=np.int64)
    for b in range(B):
        n = int(rs.randint(2, T + 2))                       # clicks of the session, >= 2
        clicks = (rs.zipf(1.3, n) % (V - 1) + 1).astype(np.int64)
        ic[b, :n - 1] = clicks[:-1]
        ln[b, :n - 1] = clicks[1:]
        last[b, 0] = clicks[-1]
        ts[b, :n - 1] = t0 + step * 60000 + np.arange(n - 1) * 1000
    sid = 1000 * (step * B + np.arange(B, dtype=np.int64)) + rs.randint(0, 2500, size=B)
    return sid, ic, ts, ln, last


def fold(sid, ic, ts, ln, last):
    for c in clfs:
        c.train(None, sid, ic, ln)
    allc = np.concatenate([ic, last], axis=1)
    allts = np.concatenate([ts, np.max(ts, axis=1).reshape(-1, 1)], axis=1)
    keep = np.nonzero(allc.reshape(-1))
    state.update_items_state(allc.reshape(-1)[keep], allts.reshape(-1)[keep])
    state.update_items_coocurrences(allc)


for step in range(N_TRAIN):
    batch = make_batch(step)
    for k, v in zip(('sid', 'ic', 'ts', 'ln', 'last'), batch):
        out['train%d_%s' % (step, k)] = v
    fold(*batch)

BIG = V + 3                                                 # wider than any valid set: the tail is 0-padded
state.save_state_checkpoint()
for step in range(N_EVAL):
    sid, ic, ts, ln, last = make_batch(N_TRAIN + step)
    for k, v in (('sid', sid), ('ic', ic), ('ts', ts), ('ln', ln), ('last', last)):
        out['eval%d_%s' % (step, k)] = v
    buf = state.get_recent_clicks_buffer().copy()
    out['eval%d_buffer' % step] = buf
    out['eval%d_pop' % step] = state.get_articles_pop().copy()
    cands = {'buf': np.unique(buf[buf != 0]), 'cat': np.arange(1, V, dtype=np.int64)}
    for c, s in zip(clfs, suffixes):
        if s in KNN:                                        # the reference's own neighbour list of every query
            nb_sid, nb_sim, nb_off = [], [], [0]
            for b in range(B):
                for t in range(T):
                    if ic[b, t] != 0:
                        for sess, v in c.find_neighbors(ic[b, :t + 1]):
                            nb_sid.append(sess)
                            nb_sim.append(v)
                    nb_off.append(len(nb_sid))
            p = 'eval%d_%s_' % (step, s)
            out[p + 'nb_sid'] = np.array(nb_sid, dtype=np.int64)
            out[p + 'nb_sim'] = np.array(nb_sim, dtype=np.float64)
            out[p + 'nb_off'] = np.array(nb_off, dtype=np.int64)
    for cname, cand in cands.items():
        out['eval%d_cand_%s' % (step, cname)] = cand
        for ex in (1, 0):
            sets = {}
            for b in range(B):
                for t in range(T):
                    if ic[b, t] != 0:
                        v = [x for x in cand if not ex or x not in ic[b, :t + 1]]
                        assert v, (step, cname, b, t)
                        sets[b, t] = v
            M = max(len(v) for v in sets.values())
            valid = np.zeros((B, T, M), dtype=np.int64)
            for (b, t), v in sets.items():
                valid[b, t] = v + [v[0]] * (M - len(v))
            for c, s in zip(clfs, suffixes):
                for k in (TOP_N, BIG):
                    out['eval%d_pred_%s_%s_%d_%d' % (step, s, cname, ex, k)] = c.predict(None, ic, topk=k, valid_items=valid)
    fold(sid, ic, ts, ln, last)
out['cfg'] = np.array([V, B, T, TOP_N, N_TRAIN, N_EVAL, BIG], dtype=np.int64)
state.restore_state_checkpoint()
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'baseline_predict_golden.npz'), **out)
print('wrote', len(out), 'arrays')
