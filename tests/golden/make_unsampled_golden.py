"""Generate tests/golden/unsampled_golden.npz for the unsampled evaluation (DESIGN.md section 13) from the REFERENCE's
own code, imported unmodified:

* support: get_sample_from_recently_clicked_items_buffer -> get_batch_negative_samples -> get_negative_samples ->
  get_neg_items_session -> get_neg_items_click (/root/reference/nar_module/nar/nar_model.py:1220-1304) on the TF-API
  stand-in tests/golden/tf1_shim.py.  The buffer sample takes the whole buffer and num_neg_samples is at least the
  pool's size, so the K*20 truncation keeps every entry and each click's negatives are a permutation of everything the
  sampler could have drawn for it, zero padded: their set is deterministic.  Scenarios: repeated clicks, re-clicked
  labels, a session whose ids cover the whole pool, an empty buffer.
* metrics: HitRate, MRR and NDCG (/root/reference/nar_module/nar/metrics.py:40-134, loaded by file path) on full ranked
  lists [label | competitors] with planted ties, ordered by descending score with the label first among equal scores
  (tf.nn.top_k over [positive | negatives]).  Per-query values (one query per add) and the streamed results.
Run once in the build container; the .npz is committed."""
import importlib
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tf1_shim as shim  # noqa: E402
import pandas  # noqa: E402,F401

sys.modules.setdefault('pytz', types.ModuleType('pytz'))
_ua = types.ModuleType('ua_parser')
_ua.user_agent_parser = types.ModuleType('ua_parser.user_agent_parser')
sys.modules.setdefault('ua_parser', _ua)
sys.modules.setdefault('ua_parser.user_agent_parser', _ua.user_agent_parser)
pkg = types.ModuleType('refnar')
pkg.__path__ = ['/root/reference/nar_module/nar']
sys.modules['refnar'] = pkg
ref = importlib.import_module('refnar.nar_model')

if not hasattr(np, 'asfarray'):
    # NDCG calls np.asfarray, which NumPy 2.0 removed; this is its NumPy 1.x definition
    np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)
spec = importlib.util.spec_from_file_location('ref_metrics', '/root/reference/nar_module/nar/metrics.py')
metrics = importlib.util.module_from_spec(spec)
spec.loader.exec_module(metrics)

out = {}
# ---- support: rows are [item_clicked ... | label_last_item], zero padded inside item_clicked
SCENARIOS = {
    'repeats': (np.array([[3, 7, 3, 9, 0, 11], [5, 3, 0, 0, 0, 7], [4, 8, 4, 0, 0, 8], [12, 12, 12, 0, 0, 2],
                          [0, 0, 0, 0, 0, 0]], dtype=np.int64),
                np.array([3, 20, 0, 21, 7, 7, 0, 22, 5, 0, 23], dtype=np.int64)),
    'covering': (np.array([[1, 2, 3, 4, 5, 6], [2, 3, 0, 0, 0, 1], [4, 6, 0, 0, 0, 5]], dtype=np.int64),
                 np.array([1, 2, 0, 3, 6, 6, 0], dtype=np.int64)),
    'empty_buffer': (np.array([[9, 4, 9, 0, 2], [4, 5, 0, 0, 9], [7, 0, 0, 0, 1]], dtype=np.int64),
                     np.zeros(8, dtype=np.int64)),
}
for ci, (name, (all_clicked, buffer)) in enumerate(sorted(SCENARIOS.items())):
    shim.configure(float64=False, seed=300 + ci)
    m = object.__new__(ref.NARModuleModel)
    m.pop_recent_items_buffer = shim._t(buffer)
    K = int(np.count_nonzero(all_clicked) + np.count_nonzero(buffer))
    extra = m.get_sample_from_recently_clicked_items_buffer(buffer.size)
    neg = m.get_batch_negative_samples(shim._t(all_clicked), additional_samples=extra, num_negative_samples=K)
    out['support/%s/all_clicked' % name] = all_clicked
    out['support/%s/buffer' % name] = buffer
    out['support/%s/negatives' % name] = neg[:, :-1, :].numpy()

# ---- metrics on full ranked lists
rs = np.random.RandomState(13)
for bi, (B, T, M) in enumerate([(4, 5, 12), (3, 4, 1), (5, 6, 30)]):
    labels = np.zeros((B, T), dtype=np.int64)
    scores = np.zeros((B, T, 1 + M))
    preds = np.zeros((B, T, 1 + M), dtype=np.int64)
    for b in range(B):
        for t in range(T):
            ids = rs.permutation(np.arange(1, 1000))[:1 + M]
            s = rs.randint(0, 6, 1 + M).astype(np.float64)     # a handful of values: ties with the label everywhere
            if rs.rand() < 0.3:
                s[0] = s.max()                                   # the label tied with the best competitors
            scores[b, t] = s
            preds[b, t] = ids[np.argsort(-s, kind='stable')]    # stable: the label (index 0) first among equals
            if rs.rand() < 0.85:
                labels[b, t] = ids[0]
    out['metrics/b%d/labels' % bi] = labels
    out['metrics/b%d/scores' % bi] = scores
    for topn in (1, 3, 5, 10):
        classes = (metrics.HitRate(topn), metrics.MRR(topn), metrics.NDCG(topn))
        per = np.zeros((3, B, T))
        for b in range(B):
            for t in range(T):
                if labels[b, t]:
                    for k, cls in enumerate((metrics.HitRate, metrics.MRR, metrics.NDCG)):
                        one = cls(topn)
                        one.add(preds[b:b + 1, t:t + 1], labels[b:b + 1, t:t + 1])
                        per[k, b, t] = one.result()
        for c in classes:
            c.add(preds, labels)
        out['metrics/b%d/top%d/per_query' % (bi, topn)] = per
        out['metrics/b%d/top%d/streamed' % (bi, topn)] = np.array([c.result() for c in classes])
np.savez_compressed(os.path.join(HERE, 'unsampled_golden.npz'), **out)
print({k: v.shape for k, v in out.items()})
