"""The list-metrics oracle (oracle/eval_metrics_ref.py) against the reference's own streaming metric classes
(tests/golden/eval_metrics_golden.npz, made by make_eval_metrics_golden.py): NDCG, item coverage, ESI-R / ESI-RR and
EILD-R / EILD-RR after every batch, for model-shaped and baseline-shaped lists at top_n 2, 3 and 10.  EILD is compared
to 1e-6: the reference's cosines are float32, the oracle's fp64."""
import os

import numpy as np
import pytest

from oracle.eval_metrics_ref import EvalMetricsRef

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'eval_metrics_golden.npz'))
CASES = [(n, s) for n in (2, 3, 10) for s in ('model', 'baseline')]


@pytest.mark.parametrize('top_n,shape', CASES)
def test_oracle_matches_reference(top_n, shape):
    pre = 'n%d_%s/' % (top_n, shape)
    g = {k[len(pre):]: GOLDEN[k] for k in GOLDEN.files if k.startswith(pre)}
    ref = EvalMetricsRef(1, top_n, g['acr'], 0.1)
    ref.begin(g['buffer'])
    for b in range(4):
        preds, labels = g['b%d/preds' % b], g['b%d/labels' % b]
        ref.add_lists(0, preds.reshape(-1, preds.shape[2]), labels.reshape(-1), g['pop'])
        ref.add_clicks(g['b%d/clicked' % b], labels)
        r = ref.results(0)
        for k in ('ndcg', 'esi-r', 'esi-rr'):
            assert abs(r[k] - g[k][b]) <= 1e-12 * max(1.0, abs(g[k][b])), (k, b, r[k], g[k][b])
        for k in ('eild-r', 'eild-rr'):
            assert abs(r[k] - float(g[k][b])) <= 1e-6, (k, b, r[k], g[k][b])
        assert r['recommended'] == g['recommended'][b] and r['clicked'] == g['clicked'][b], b
        assert r['coverage'] == g['coverage'][b], b


def test_fixture_covers_the_edge_cases():
    for n, s in CASES:
        pre = 'n%d_%s/' % (n, s)
        assert 0 in GOLDEN[pre + 'buffer']                                  # padding in the buffer
        acr = GOLDEN[pre + 'acr']
        assert not acr[0].any() and np.array_equal(acr[5], acr[6])
        assert (GOLDEN[pre + 'pop'] == np.float32(1.0 / 500)).any()
        ranks, absent, zeros = set(), 0, 0
        for b in range(4):
            preds, labels = GOLDEN[pre + 'b%d/preds' % b], GOLDEN[pre + 'b%d/labels' % b]
            assert (labels == 0).any()
            for lst, lab in zip(preds.reshape(-1, preds.shape[2]), labels.reshape(-1)):
                if lab == 0:
                    continue
                hit = np.flatnonzero(lst[:n] == lab)
                ranks.update(hit[:1].tolist())
                absent += hit.size == 0
                zeros += (lst == 0).any()
        assert ranks == set(range(min(n, preds.shape[2]))), (n, s, ranks)
        assert zeros > 0
        if s == 'baseline' or n < 8:
            assert absent > 0
