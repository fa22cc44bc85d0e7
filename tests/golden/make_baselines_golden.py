"""Generate tests/golden/baselines_golden.npz by running the REFERENCE baseline recommenders
(benchmarks/{recently_popular,item_cooccurrences,item_knn,content_based,sequential_rules}.py) and ClickedItemsState,
unmodified, in the order of the evaluation hook (nar_model.py:1609-1650): over seeded synthetic train batches (the
baselines learn, the state absorbs the batch), then eval batches with recorded negatives (every baseline predicts over
label + negatives, HitRate / MRR accumulate, then the baselines learn and the state absorbs the batch), then the state
checkpoint is restored.  The reference package is loaded through a shim package so that its relative imports resolve;
tensorflow / ua_parser / pytz are stub modules (only imported, never called).  Run once in the build container; the
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

REF_DIR = '/root/reference/nar_module/nar'
pkg = types.ModuleType('refnar')
pkg.__path__ = [REF_DIR]
sys.modules['refnar'] = pkg
cis = importlib.import_module('refnar.clicked_items_state')
bm = importlib.import_module('refnar.benchmarks')
metrics = importlib.import_module('refnar.metrics')

V, B, T, K, TOP_N = 60, 6, 8, 6, 5
N_TRAIN, N_EVAL = 5, 3
rs = np.random.RandomState(11)
acr = rs.randn(V, 8)
acr[0] = 0.0


class Scipy2018CSR(cis.csr_matrix):
    """The co-occurrence matrix as the reference's SciPy had it: ``row / dense`` was ``np.matrix(row.todense() / dense)``
    (item_knn.py:52 indexes that matrix); current SciPy returns a sparse matrix there."""

    def __truediv__(self, other):
        if isinstance(other, np.ndarray):
            return np.asmatrix(self.toarray() / other)
        return super().__truediv__(other)


state = cis.ClickedItemsState(1.0, 40, 20, V)
state.items_coocurrences = Scipy2018CSR(state.items_coocurrences)
clfs = [bm.RecentlyPopularRecommender(state, {}, []),
        bm.ItemCooccurrenceRecommender(state, {}, []),
        bm.ItemKNNRecommender(state, {'reg_lambda': 20, 'alpha': 0.75}, []),
        bm.ContentBasedRecommender(state, {'content_article_embeddings_matrix': acr}, []),
        bm.SequentialRulesRecommender(state, {'max_clicks_dist': 10, 'dist_between_clicks_decay': 'div'}, [])]
suffixes = [c.get_clf_suffix() for c in clfs]
out = {'cfg': np.array([V, B, T, K, TOP_N, N_TRAIN, N_EVAL], dtype=np.int64), 'acr': acr}
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
    return ic, ts, ln, last


def fold(ic, ts, ln, last):
    for c in clfs:
        c.train(None, None, ic, ln)
    allc = np.concatenate([ic, last], axis=1)
    allts = np.concatenate([ts, np.max(ts, axis=1).reshape(-1, 1)], axis=1)
    keep = np.nonzero(allc.reshape(-1))
    state.update_items_state(allc.reshape(-1)[keep], allts.reshape(-1)[keep])
    state.update_items_coocurrences(allc)
    assert isinstance(state.items_coocurrences, Scipy2018CSR)


def sr_rules(rules):
    past, act, w = [], [], []
    for a, d in rules.items():
        for c, v in d.items():
            past.append(a); act.append(c); w.append(v)
    return np.array(past, dtype=np.int64), np.array(act, dtype=np.int64), np.array(w, dtype=np.float64)


for step in range(N_TRAIN):
    ic, ts, ln, last = make_batch(step)
    for k, v in (('ic', ic), ('ts', ts), ('ln', ln), ('last', last)):
        out['train%d_%s' % (step, k)] = v
    fold(ic, ts, ln, last)
out['train_cooc_dense'] = state.items_coocurrences.toarray()
out['train_sr_past'], out['train_sr_active'], out['train_sr_w'] = sr_rules(state.benchmarks_states['sr']['rules'])

state.save_state_checkpoint()
hr = {s: metrics.HitRate(TOP_N) for s in suffixes}
mrr = {s: metrics.MRR(TOP_N) for s in suffixes}
for m in list(hr.values()) + list(mrr.values()):
    m.reset()
for step in range(N_EVAL):
    ic, ts, ln, last = make_batch(N_TRAIN + step)
    neg = rs.randint(1, V, size=(B, T, K)).astype(np.int64)
    neg[rs.rand(B, T, K) < 0.15] = 0                       # padding negatives
    neg[ln == 0] = 0
    for k, v in (('ic', ic), ('ts', ts), ('ln', ln), ('last', last), ('neg', neg)):
        out['eval%d_%s' % (step, k)] = v
    out['eval%d_buffer' % step] = state.get_recent_clicks_buffer().copy()
    out['eval%d_pop' % step] = state.get_articles_pop().copy()
    valid = np.concatenate([np.expand_dims(ln, axis=2), neg], axis=2)
    for c, s in zip(clfs, suffixes):
        preds = c.predict(None, ic, topk=TOP_N, valid_items=valid)
        out['eval%d_pred_%s' % (step, s)] = preds
        hr[s].add(preds, ln)
        mrr[s].add(preds, ln)
    fold(ic, ts, ln, last)
for s in suffixes:
    out['hr_' + s] = np.float64(hr[s].result())
    out['mrr_' + s] = np.float64(mrr[s].result())
out['eval_cooc_dense'] = state.items_coocurrences.toarray()
out['eval_sr_past'], out['eval_sr_active'], out['eval_sr_w'] = sr_rules(state.benchmarks_states['sr']['rules'])
state.restore_state_checkpoint()
out['restored_cooc_dense'] = state.items_coocurrences.toarray()
out['restored_sr_past'], out['restored_sr_active'], out['restored_sr_w'] = sr_rules(state.benchmarks_states['sr']['rules'])
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'baselines_golden.npz'), **out)
print('wrote', len(out), 'arrays')
