"""Generate tests/golden/by_position_golden.npz with the REFERENCE's own code: ``HitRateBySessionPosition``
(/root/reference/nar_module/nar/metrics.py) driven by ``update_metrics`` / ``compute_metrics_results``
(evaluation.py), both loaded unmodified as the submodules of a package made from the reference's directory (its
``__init__.py`` is empty; numpy + sklearn only).  They are fed the way the hook and the baselines feed them
(nar_model.py:1593-1603, benchmarks.py:35-55): predictions [B, T, len], labels [B, T], labels_norm_pop = pop[labels],
preds_norm_pop = pop[predictions], clicked_items [B, T].

Cases, for top_n in {1, 3, 10}:
* 'model', recommender 'chameleon' (so the clicks and mean-popularity keys are reported too): full ranked candidate
  lists [B, T, 1 + K] (1 + K = 8, so top_n 10 reads all 8), the label at every rank, zero-padded negatives and the
  label repeated;
* 'baseline', recommender 'v-sknn': 0-padded top-n lists [B, T, top_n] (half of them full), the label at every rank
  or absent.
Sessions have lengths 0 .. T, so late positions have few queries; labels past a session's length are 0 and a few inside
are 0 too (holes).  pop is float32 over four decades, so the float32 sums depend on their order.  The result dict after
each of 4 batches is recorded as keys and float64 values (the float32 means widen exactly).  Run once in the build
container; the .npz is committed."""
import importlib
import importlib.util
import os
import sys

import numpy as np

PKG = '/root/reference/nar_module/nar'
spec = importlib.util.spec_from_file_location('ref_nar', os.path.join(PKG, '__init__.py'), submodule_search_locations=[PKG])
pkg = importlib.util.module_from_spec(spec)
sys.modules['ref_nar'] = pkg
spec.loader.exec_module(pkg)
evaluation = importlib.import_module('ref_nar.evaluation')
metrics = importlib.import_module('ref_nar.metrics')

V, B, T, K, NORM = 60, 8, 6, 7, 500
out = {}
for top_n in (1, 3, 10):
    for shape, rec in (('model', 'chameleon'), ('baseline', 'v-sknn')):
        rs = np.random.RandomState(1000 + 10 * top_n + len(shape))
        pop = (rs.rand(V) * 10.0 ** rs.uniform(-4, 0, size=V)).astype(np.float32)
        pop[rs.rand(V) < 0.2] = np.float32(1.0 / NORM)
        metric = metrics.HitRateBySessionPosition(top_n)
        metric.reset()
        pre = 'n%d_%s/' % (top_n, shape)
        for batch in range(4):
            lens = rs.randint(0, T + 1, size=B)
            lens[rs.randint(0, B)] = T
            labels = rs.randint(1, V, size=(B, T)).astype(np.int64)
            labels[np.arange(T)[None, :] >= lens[:, None]] = 0
            labels[rs.rand(B, T) < 0.1] = 0                                   # holes inside sessions
            clicked = rs.randint(0, V, size=(B, T)).astype(np.int64)
            width = 1 + K if shape == 'model' else top_n
            preds = np.zeros((B, T, width), dtype=np.int64)
            for b in range(B):
                for t in range(T):
                    lab = labels[b, t] if labels[b, t] else rs.randint(1, V)
                    others = [x for x in rs.permutation(np.arange(1, V)) if x != lab][:width]
                    if shape == 'model':
                        row = others[:K]
                        if rs.rand() < 0.3:                                 # a short pool: zero-padded negatives
                            s = rs.randint(K // 2, K)
                            row[s:] = [0] * (K - s)
                        if rs.rand() < 0.15:
                            row[rs.randint(0, K)] = lab                     # the label twice among the candidates
                        row.insert(rs.randint(0, K + 1), lab)                # the label at any rank
                    else:
                        n_valid = top_n if rs.rand() < 0.5 else rs.randint(0, top_n + 1)
                        row = others[:n_valid] + [0] * (top_n - n_valid)
                        if n_valid and rs.rand() < 0.7:
                            row[rs.randint(0, n_valid)] = lab               # present, else absent
                    preds[b, t] = row[:width]
            evaluation.update_metrics(preds, labels, pop[labels], pop[preds], clicked, [metric], recommender=rec)
            res = evaluation.compute_metrics_results([metric], recommender=rec)
            for k, v in res.items():
                if k.startswith('avg_norm_pop_by_pos'):
                    assert isinstance(v, np.float32), (k, type(v))          # the reference sums and divides in float32
            keys = sorted(res)
            out[pre + 'b%d/preds' % batch] = preds
            out[pre + 'b%d/labels' % batch] = labels
            out[pre + 'b%d/keys' % batch] = np.array(keys)
            out[pre + 'b%d/values' % batch] = np.array([float(res[k]) for k in keys], dtype=np.float64)
        out[pre + 'pop'] = pop
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'by_position_golden.npz'), **out)
print({k: v for k, v in out.items() if k.endswith('b3/keys')})
