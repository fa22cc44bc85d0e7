"""Generate tests/golden/eval_metrics_golden.npz with the REFERENCE's own streaming metric classes
(/root/reference/nar_module/nar/metrics.py, loaded by file path, unmodified; numpy + sklearn only): NDCG, ItemCoverage,
ExpectedRankSensitiveNovelty, ExpectedRankRelevanceSensitiveNovelty, ContentExpectedRankRelativeSensitiveIntraListDiversity
and ContentExpectedRankRelativeRelevanceSensitiveIntraListDiversity - the six that
ItemsStateUpdaterHook.create_eval_metrics (nar_model.py:1696-1721) adds to HR / MRR.  They are fed the way the hook
feeds them (evaluation.py update_metrics): predictions [B, T, len], labels [B, T], predictions_norm_pop = pop[predictions],
clicked_items [B, T].

Cases, for top_n in {2, 3, 10}:
* 'model': full ranked candidate lists [B, T, 1 + K] (1 + K = 8, so top_n 10 scores all 8), the label at every rank,
  zero-padded negatives and repeated ids (the label more than once included);
* 'baseline': 0-padded top-n lists [B, T, top_n], the label at every rank or absent.
The ACR matrix is float32 with a zero row 0 and two identical rows (5 and 6); pop is float32-representable with many
values at the 1 / recent_clicks_for_normalization floor; the recent-clicks buffer holds zero padding.  The streaming
result after each of 4 batches is recorded, with the two coverage set sizes.  Run once in the build container; the
.npz is committed."""
import importlib.util
import os

import numpy as np

if not hasattr(np, 'asfarray'):
    # NDCG calls np.asfarray, which NumPy 2.0 removed; this is its NumPy 1.x definition
    np.asfarray = lambda a, dtype=np.float64: np.asarray(a, dtype=dtype)

REF = '/root/reference/nar_module/nar/metrics.py'
spec = importlib.util.spec_from_file_location('ref_metrics', REF)
mod = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mod)

V, DIM, B, T, K, NEG_REL, NORM = 60, 12, 8, 6, 7, 0.1, 500
out = {}
for top_n in (2, 3, 10):
    for shape in ('model', 'baseline'):
        rs = np.random.RandomState(100 * top_n + len(shape))
        acr = rs.randn(V, DIM).astype(np.float32)
        acr[0] = 0.0
        acr[6] = acr[5]
        pop = rs.randint(1, 40, size=V).astype(np.float32) / np.float32(NORM)
        pop[rs.rand(V) < 0.4] = np.float32(1.0 / NORM)
        pop = pop.astype(np.float64)
        buffer = np.zeros(30, dtype=np.int64)
        buffer[:18] = rs.randint(1, V, size=18)
        metrics = [mod.NDCG(top_n), mod.ItemCoverage(top_n, buffer),
                   mod.ExpectedRankSensitiveNovelty(top_n),
                   mod.ExpectedRankRelevanceSensitiveNovelty(top_n, 1.0, NEG_REL),
                   mod.ContentExpectedRankRelativeSensitiveIntraListDiversity(top_n, acr),
                   mod.ContentExpectedRankRelativeRelevanceSensitiveIntraListDiversity(top_n, acr, 1.0, NEG_REL)]
        res = {k: [] for k in ('ndcg', 'esi-r', 'esi-rr', 'eild-r', 'eild-rr', 'coverage', 'recommended', 'clicked')}
        pre = 'n%d_%s/' % (top_n, shape)
        for batch in range(4):
            labels = rs.randint(1, V, size=(B, T)).astype(np.int64)
            labels[rs.rand(B, T) < 0.25] = 0
            clicked = rs.randint(0, V, size=(B, T)).astype(np.int64)
            width = 1 + K if shape == 'model' else top_n
            preds = np.zeros((B, T, width), dtype=np.int64)
            for b in range(B):
                for t in range(T):
                    lab = labels[b, t] if labels[b, t] else rs.randint(1, V)
                    others = [x for x in rs.permutation(np.arange(1, V)) if x != lab][:width]
                    if shape == 'model':
                        row = others[:K]
                        if rs.rand() < 0.3:                             # a short pool: zero-padded negatives
                            s = rs.randint(K // 2, K)
                            row[s:] = [0] * (K - s)
                        if rs.rand() < 0.15:
                            row[rs.randint(0, K)] = lab                 # the label twice among the candidates
                        if rs.rand() < 0.15:
                            row[rs.randint(0, K)] = 5
                            row[rs.randint(0, K)] = 6
                        row.insert(rs.randint(0, K + 1), lab)            # the label at any rank
                    else:
                        n_valid = rs.randint(0, top_n + 1)
                        row = others[:n_valid] + [0] * (top_n - n_valid)
                        if n_valid and rs.rand() < 0.7:
                            row[rs.randint(0, n_valid)] = lab           # present, else absent
                    preds[b, t] = row[:width]
            for mt in metrics:
                if isinstance(mt, mod.ItemCoverage):
                    mt.add(preds, labels, clicked)
                elif isinstance(mt, (mod.ExpectedRankSensitiveNovelty, mod.ExpectedRankRelevanceSensitiveNovelty)):
                    mt.add(preds, labels, pop[preds])
                else:
                    mt.add(preds, labels)
            for k, mt in zip(('ndcg', 'coverage', 'esi-r', 'esi-rr', 'eild-r', 'eild-rr'), metrics):
                res[k].append(mt.result())
            res['recommended'].append(len(metrics[1].recommended_items))
            res['clicked'].append(len(metrics[1].clicked_items))
            out[pre + 'b%d/preds' % batch] = preds
            out[pre + 'b%d/labels' % batch] = labels
            out[pre + 'b%d/clicked' % batch] = clicked
        out[pre + 'acr'] = acr
        out[pre + 'pop'] = pop
        out[pre + 'buffer'] = buffer
        for k, v in res.items():
            out[pre + k] = np.asarray(v)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'eval_metrics_golden.npz'), **out)
print({k: v for k, v in out.items() if k.endswith(('/ndcg', '/coverage', '/eild-r'))})
