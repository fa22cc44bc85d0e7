"""Generate tests/golden/session_logs_golden.npz with the REFERENCE's own code: ``ItemsStateUpdaterHook`` in EVAL mode
(nar_model.py, imported unmodified on the TF-API stand-in tests/golden/tf1_shim.py) is given the two log lists and run
through begin / after_run over 3 batches, so its logging block (nar_model.py:1529-1581) fills them; then the trainer's
writers ``save_sessions_negative_items`` / ``save_sessions_chameleon_recommendations_log`` (nar_trainer_gcom.py:390-407,
also unmodified) write the lists to files, whose text is recorded.

The batches: sessions of lengths 0 .. T with one label-0 hole inside a session; ranked candidates = a permutation of
label + negatives (negatives zero-padded in places); float32 probabilities that sit exactly on round-half ties at the 7th
decimal (x * 1e7 = n + 0.5 in float32), below 5e-8, denormal, exactly 0 and exactly 1; the popularity is the reference
ClickedItemsState's own float64 ``get_articles_recent_pop_norm()`` (most articles at its floor), which moves between
batches as the hook folds each batch in; one session id has 17 digits.  Run once in the build container; the .npz is
committed."""
import importlib
import json
import os
import sys
import tempfile
import types

import numpy as np

if not hasattr(np, 'asfarray'):
    # the hook's NDCG metric calls np.asfarray, which NumPy 2.0 removed; this is its NumPy 1.x definition
    np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import tf1_shim as shim  # noqa: E402,F401
import pandas  # noqa: E402,F401
import google  # noqa: E402

sys.modules.setdefault('pytz', types.ModuleType('pytz'))
_ua = types.ModuleType('ua_parser')
_ua.user_agent_parser = types.ModuleType('ua_parser.user_agent_parser')
sys.modules.setdefault('ua_parser', _ua)
sys.modules.setdefault('ua_parser.user_agent_parser', _ua.user_agent_parser)
_gc = types.ModuleType('google.cloud')
_gc.storage = types.ModuleType('google.cloud.storage')
sys.modules['google.cloud'] = _gc
sys.modules['google.cloud.storage'] = _gc.storage
google.cloud = _gc
pkg = types.ModuleType('refnar')
pkg.__path__ = ['/root/reference/nar_module/nar']
sys.modules['refnar'] = pkg
ref_model = importlib.import_module('refnar.nar_model')
ref_state = importlib.import_module('refnar.clicked_items_state')
trainer = importlib.import_module('refnar.nar_trainer_gcom')

V, B, T, K, E, TOP_N = 40, 7, 5, 6, 8, 3
rs = np.random.RandomState(20240607)

# float32 values whose product with 1e7 is exactly n + 0.5 in float32: ties of the rounding
ties = []
for n in list(range(0, 40)) + [12345, 99999, 250000, 1048574]:
    x = np.float32((n + 0.5) / 1e7)
    if np.float32(x * np.float32(1e7)) == np.float32(n + 0.5):
        ties.append(x)
assert len(ties) >= 8, len(ties)
special = np.array(ties + [0.0, 1.0, 3e-8, 4.9999999e-8, 5.0000001e-8, 1e-30, 1e-40, 0.99999994, 0.33333334], dtype=np.float32)

state = ref_state.ClickedItemsState(1.0, 60, 25, V)
state.update_items_state(rs.randint(1, 12, size=30).astype(np.int64), (1500000000000 + np.arange(30) * 1000).astype(np.int64))
acr = rs.randn(V, E).astype(np.float32)
model = types.SimpleNamespace()
neg_log, rec_log = [], []
hook = ref_model.ItemsStateUpdaterHook('eval', model, TOP_N, state, [], neg_log, rec_log, acr, {}, 0.02)
hook.begin()

out = {'cfg': np.array([V, B, T, K], dtype=np.int64)}
n_neg, n_rec = [], []
for batch in range(3):
    lens = np.arange(B) % (T + 1)                                    # 0 .. T
    lens = lens[rs.permutation(B)]
    labels = rs.randint(1, V, size=(B, T)).astype(np.int64)
    labels[np.arange(T)[None, :] >= lens[:, None]] = 0
    if batch == 1:
        b = int(np.flatnonzero(lens == T)[0])
        labels[b, 2] = 0                                             # a hole inside a session
    neg = np.zeros((B, T, K), dtype=np.int64)
    ids = np.zeros((B, T, 1 + K), dtype=np.int64)
    probs = np.zeros((B, T, 1 + K), dtype=np.float32)
    for b in range(B):
        for t in range(lens[b]):
            row = rs.choice(np.arange(1, V), size=K, replace=False)
            if rs.rand() < 0.3:
                row[rs.randint(1, K):] = 0                           # a short pool: zero-padded negatives
            neg[b, t] = row
            ids[b, t] = rs.permutation(np.concatenate([[labels[b, t]], row]))
            p = np.sort(rs.dirichlet(np.ones(1 + K)).astype(np.float32))[::-1]
            m = rs.rand(1 + K) < 0.45
            p[m] = rs.choice(special, size=int(m.sum()))
            probs[b, t] = p
    sids = (1500000000 + 100 * batch + np.arange(B)).astype(np.int64)
    sids[1] = 15436781234567890 + batch                              # 17 digits
    # (the logs read the labels only; every session keeps two clicks, which the hook's state update needs)
    clicked = np.where(np.arange(T)[None, :] < np.maximum(lens, 2)[:, None], rs.randint(1, V, size=(B, T)), 0).astype(np.int64)
    ts = np.where(clicked != 0, 1500000100000 + 60000 * batch + rs.randint(0, 50000, size=(B, T)), 0).astype(np.int64)
    last = np.array([[labels[b, lens[b] - 1] if lens[b] else 0] for b in range(B)], dtype=np.int64)
    pop = state.get_articles_recent_pop_norm().copy()
    assert pop.dtype == np.float64
    results = {'clicked_items': clicked, 'clicked_timestamps': ts[..., None], 'next_item_labels': labels,
               'last_item_label': last, 'user_id': np.arange(B, dtype=np.int64), 'session_id': sids,
               'predicted_item_ids': ids, 'eval_batch_negative_items': neg, 'predicted_item_probs': probs,
               'hitrate_at_n': 0.0, 'mrr_at_n': 0.0, 'batch_items_count': int((clicked != 0).sum()),
               'batch_unique_items_count': int(np.unique(clicked[clicked != 0]).size)}
    hook.after_run(None, types.SimpleNamespace(results=results))
    for k, v in (('labels', labels), ('neg', neg), ('ids', ids), ('probs', probs), ('pop', pop), ('sids', sids), ('lens', lens)):
        out['b%d/%s' % (batch, k)] = v
    n_neg.append(len(neg_log))
    n_rec.append(len(rec_log))
hook.end()
assert n_neg == [B, 2 * B, 3 * B] and n_rec == n_neg
out['entries_after_batch'] = np.array(n_neg, dtype=np.int64)
out['neg_log_json'] = np.array(json.dumps(neg_log))
out['rec_log_json'] = np.array(json.dumps(rec_log))
with tempfile.TemporaryDirectory() as d:
    trainer.save_sessions_negative_items(d, neg_log)
    trainer.save_sessions_chameleon_recommendations_log(d, rec_log, 3)
    out['neg_file_text'] = np.array(open(os.path.join(d, 'eval_sessions_negative_samples.json')).read())
    out['rec_file_text'] = np.array(open(os.path.join(d, 'eval_chameleon_recommendations_log.json')).read())
np.savez_compressed(os.path.join(HERE, 'session_logs_golden.npz'), **out)
print('wrote', len(out), 'arrays;', sum(len(e['negative_items']) for e in neg_log), 'queries;', len(ties), 'tie values;',
      os.path.getsize(os.path.join(HERE, 'session_logs_golden.npz')) // 1024, 'KB')
