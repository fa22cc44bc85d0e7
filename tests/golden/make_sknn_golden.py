"""Generate tests/golden/sknn_golden.npz by running the REFERENCE session-based kNN recommender
(benchmarks/session_knn.py) and ClickedItemsState, unmodified, in the order of the evaluation hook
(nar_model.py:1609-1632): seeded synthetic train batches (the recommender learns), then eval batches with recorded
negatives (it predicts over label + negatives, HitRate / MRR accumulate, then it learns), then the state checkpoint is
restored.  Four parameter sets ('div' + cosine, 'same' + jaccard, and both decays without the 'recent' cut) see the
same batches.  The buffer is small, so entries are evicted, and the cuts and the ``< 1.0`` filter all fire.  Train batch
2 repeats batch 1 (the same session ids twice: an eviction discards the map entries of a newer twin), and batch 3 has
descending ids below the earlier ones (the buffer's binary search misses them).  Per query the fixture holds the
predictions and the reference's own ``find_neighbors`` list.  The reference package is loaded through the shim of
make_baselines_golden.py.  Run once in the build container; the .npz is committed."""
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

V, B, T, K, TOP_N = 30, 6, 8, 6, 5
N_TRAIN, N_EVAL = 6, 3
CONFIGS = [  # (sessions_buffer_size, candidate_sessions_sample_size, nearest_neighbor_session_for_scoring, similarity, decay)
    (20, 12, 6, 'cosine', 'div'),
    (20, 12, 6, 'jaccard', 'same'),
    (20, 0, 6, 'cosine', 'div'),
    (20, 0, 6, 'cosine', 'same'),
]
rs = np.random.RandomState(5)


def make_batch(step, backwards=False):
    ic = np.zeros((B, T), dtype=np.int64)
    ln = np.zeros((B, T), dtype=np.int64)
    last = np.zeros((B, 1), dtype=np.int64)
    for b in range(B):
        n = int(rs.randint(2, T + 2))                       # clicks of the session, >= 2
        clicks = (rs.zipf(1.3, n) % (V - 1) + 1).astype(np.int64)
        ic[b, :n - 1] = clicks[:-1]
        ln[b, :n - 1] = clicks[1:]
        last[b, 0] = clicks[-1]
    if backwards:
        sid = 500 - 10 * np.arange(B, dtype=np.int64)
    else:                                                   # ascending by batch, jittered within it
        sid = 1000 * (step * B + np.arange(B, dtype=np.int64)) + rs.randint(0, 2500, size=B)
    return sid, ic, ln, last


batches = []
for step in range(N_TRAIN):
    if step == 2:
        batches.append(batches[1])
    else:
        batches.append(make_batch(step, backwards=(step == 3)))
evals = []
for step in range(N_EVAL):
    sid, ic, ln, last = make_batch(N_TRAIN + step)
    neg = rs.randint(1, V, size=(B, T, K)).astype(np.int64)
    neg[rs.rand(B, T, K) < 0.15] = 0                       # padding negatives
    neg[ln == 0] = 0
    evals.append((sid, ic, ln, last, neg))

out = {'cfg': np.array([V, B, T, K, TOP_N, N_TRAIN, N_EVAL], dtype=np.int64),
       'params': np.array([c[:3] for c in CONFIGS], dtype=np.int64),
       'similarity': np.array([c[3] for c in CONFIGS]), 'decay': np.array([c[4] for c in CONFIGS])}
for i, (sid, ic, ln, last) in enumerate(batches):
    for k, v in (('sid', sid), ('ic', ic), ('ln', ln), ('last', last)):
        out['train%d_%s' % (i, k)] = v
for i, (sid, ic, ln, last, neg) in enumerate(evals):
    for k, v in (('sid', sid), ('ic', ic), ('ln', ln), ('last', last), ('neg', neg)):
        out['eval%d_%s' % (i, k)] = v


def export(st, prefix):
    buf, mp = st['last_sessions_buffer'], st['item_session_map']
    W = T + 1
    ids = np.array([e.session_id for e in buf], dtype=np.int64)
    items = np.zeros((len(buf), W), dtype=np.int64)
    live = np.zeros((len(buf), W), dtype=bool)
    for r, e in enumerate(buf):
        xs = sorted(int(x) for x in e.item_ids)
        items[r, :len(xs)] = xs
        live[r, :len(xs)] = [e.session_id in mp.get(x, ()) for x in xs]
    out[prefix + '_ids'], out[prefix + '_items'], out[prefix + '_live'] = ids, items, live


for c, (S, C, NN, sim, decay) in enumerate(CONFIGS):
    state = cis.ClickedItemsState(1.0, 40, 20, V)
    params = {'sessions_buffer_size': S, 'candidate_sessions_sample_size': C, 'sampling_strategy': 'recent',
              'nearest_neighbor_session_for_scoring': NN, 'similarity': sim, 'first_session_clicks_decay': decay}
    clf = bm.SessionBasedKNNRecommender(state, params, [])
    sfx = clf.get_clf_suffix()
    for sid, ic, ln, last in batches:
        clf.train(None, sid, ic, ln)
    export(state.benchmarks_states[sfx], 'c%d_train' % c)
    state.save_state_checkpoint()
    hr, mrr = metrics.HitRate(TOP_N), metrics.MRR(TOP_N)
    hr.reset()
    mrr.reset()
    for e, (sid, ic, ln, last, neg) in enumerate(evals):
        valid = np.concatenate([np.expand_dims(ln, axis=2), neg], axis=2)
        nb_sid, nb_sim, nb_off = [], [], [0]
        for b in range(B):
            for t in range(T):
                if ln[b, t] != 0:
                    for s, v in clf.find_neighbors(ic[b, :t + 1]):
                        nb_sid.append(s)
                        nb_sim.append(v)
                nb_off.append(len(nb_sid))
        preds = clf.predict(None, ic, topk=TOP_N, valid_items=valid)
        p = 'c%d_eval%d' % (c, e)
        out[p + '_pred'] = preds
        out[p + '_nb_sid'] = np.array(nb_sid, dtype=np.int64)
        out[p + '_nb_sim'] = np.array(nb_sim, dtype=np.float64)
        out[p + '_nb_off'] = np.array(nb_off, dtype=np.int64)
        hr.add(preds, ln)
        mrr.add(preds, ln)
        clf.train(None, sid, ic, ln)
    out['c%d_hr' % c] = np.float64(hr.result())
    out['c%d_mrr' % c] = np.float64(mrr.result())
    export(state.benchmarks_states[sfx], 'c%d_eval' % c)
    state.restore_state_checkpoint()
    export(state.benchmarks_states[sfx], 'c%d_restored' % c)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'sknn_golden.npz'), **out)
print('wrote', len(out), 'arrays')
