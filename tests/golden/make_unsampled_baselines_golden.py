"""Generate tests/golden/unsampled_baselines_golden.npz by running the REFERENCE baseline recommenders
(benchmarks/{recently_popular,item_cooccurrences,item_knn,content_based,sequential_rules,session_knn}.py) and
ClickedItemsState, unmodified, in the order of the evaluation hook (nar_model.py:1609-1650), with each eval query's valid
items = its label and its whole unsampled competitor set (DESIGN.md section 14: the pool of the batch - its clicks, its
last labels and the recent-clicks buffer - minus the session's row), padded with the label.  Each recommender predicts
with topk = the width of that list, so its prediction is its full ranking of the admissible valid items; HitRate, MRR
and NDCG accumulate on it.  Seeded synthetic train batches first (every recommender learns, the state absorbs the
batch), then eval batches (predict, then learn and absorb).  The reference package is loaded through the shim of
make_baselines_golden.py; for the session kNN baselines the fixture also holds each query's ``find_neighbors`` list.
Run once in the build container; the .npz is committed."""
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
rs = np.random.RandomState(23)
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

state.save_state_checkpoint()
ms = {s: (metrics.HitRate(TOP_N), metrics.MRR(TOP_N), metrics.NDCG(TOP_N)) for s in suffixes}
for trio in ms.values():
    for m in trio:
        m.reset()
for step in range(N_EVAL):
    sid, ic, ts, ln, last = make_batch(N_TRAIN + step)
    for k, v in (('sid', sid), ('ic', ic), ('ts', ts), ('ln', ln), ('last', last)):
        out['eval%d_%s' % (step, k)] = v
    buf = state.get_recent_clicks_buffer().copy()
    out['eval%d_buffer' % step] = buf
    out['eval%d_pop' % step] = state.get_articles_pop().copy()
    ids = np.concatenate([ic.reshape(-1), last.reshape(-1), buf.reshape(-1)])
    pool = np.unique(ids[ids != 0])
    comp = {}
    for b in range(B):
        row = np.append(ic[b], last[b])
        for t in range(T):
            if ln[b, t] != 0:
                comp[b, t] = [ln[b, t]] + [c for c in np.setdiff1d(pool, row) if c != ln[b, t]]
    M = max(len(v) for v in comp.values())
    valid = np.zeros((B, T, M), dtype=np.int64)
    for (b, t), v in comp.items():
        valid[b, t] = v + [v[0]] * (M - len(v))             # padded with the label
    out['eval%d_valid' % step] = valid
    for c, s in zip(clfs, suffixes):
        if s in KNN:                                        # the reference's own neighbour list of every query
            nb_sid, nb_sim, nb_off = [], [], [0]
            for b in range(B):
                for t in range(T):
                    if ln[b, t] != 0:
                        for sess, v in c.find_neighbors(ic[b, :t + 1]):
                            nb_sid.append(sess)
                            nb_sim.append(v)
                    nb_off.append(len(nb_sid))
            p = 'eval%d_%s_' % (step, s)
            out[p + 'nb_sid'] = np.array(nb_sid, dtype=np.int64)
            out[p + 'nb_sim'] = np.array(nb_sim, dtype=np.float64)
            out[p + 'nb_off'] = np.array(nb_off, dtype=np.int64)
        preds = c.predict(None, ic, topk=M, valid_items=valid)
        out['eval%d_pred_%s' % (step, s)] = preds
        for m in ms[s]:
            m.add(preds, ln)
    fold(sid, ic, ts, ln, last)
for s in suffixes:
    for name, m in zip(('hr', 'mrr', 'ndcg'), ms[s]):
        out['%s_%s' % (name, s)] = np.float64(m.result())
state.restore_state_checkpoint()
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'unsampled_baselines_golden.npz'), **out)
print('wrote', len(out), 'arrays')
