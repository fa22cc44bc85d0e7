"""The by-position oracle (oracle/by_position_ref.py) against the reference's own HitRateBySessionPosition, update_metrics
and compute_metrics_results (tests/golden/by_position_golden.npz, made by make_by_position_golden.py) after every batch,
for model-shaped and baseline-shaped lists at top_n 1, 3 and 10: every key, hit rates and counts exactly, the mean label
popularity bit for bit as float32.  Also the switch's params: off by default, and the default params dict unchanged."""
import os

import numpy as np
import pytest

from oracle.by_position_ref import ByPositionRef

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'by_position_golden.npz'))
CASES = [(n, s) for n in (1, 3, 10) for s in ('model', 'baseline')]
T = 6


def _case(top_n, shape):
    pre = 'n%d_%s/' % (top_n, shape)
    return {k[len(pre):]: GOLDEN[k] for k in GOLDEN.files if k.startswith(pre)}


@pytest.mark.parametrize('top_n,shape', CASES)
def test_oracle_matches_reference(top_n, shape):
    g = _case(top_n, shape)
    model = shape == 'model'
    ref = ByPositionRef(1, top_n)
    ref.begin()
    for b in range(4):
        preds, labels = g['b%d/preds' % b], g['b%d/labels' % b]
        ref.add(0, preds.reshape(-1, preds.shape[2]), labels.reshape(-1), T, pop=g['pop'] if model else None)
        got = ref.results(0, '' if model else 'v-sknn')
        want = {str(k).replace('_chameleon', ''): v for k, v in zip(g['b%d/keys' % b], g['b%d/values' % b])}
        assert sorted(got) == sorted(want), b
        for k, v in want.items():
            if k.startswith('avg_norm_pop_by_pos'):
                assert v == np.float64(np.float32(v)), k                       # the reference's value is a float32
                assert np.float32(got[k]).view(np.int32) == np.float32(v).view(np.int32), (b, k, got[k], v)
            else:
                assert got[k] == v, (b, k, got[k], v)


def test_fixture_covers_the_edge_cases():
    for n, s in CASES:
        g = _case(n, s)
        ranks, absent, holes, per_pos = set(), 0, 0, np.zeros(T, np.int64)
        for b in range(4):
            preds, labels = g['b%d/preds' % b], g['b%d/labels' % b]
            lens = T - np.argmax((labels != 0)[:, ::-1], axis=1)
            holes += int(((labels == 0) & (np.arange(T)[None, :] < lens[:, None])).sum())
            per_pos += (labels != 0).sum(axis=0)
            for lst, lab in zip(preds.reshape(-1, preds.shape[2]), labels.reshape(-1)):
                if lab:
                    hit = np.flatnonzero(lst[:n] == lab)
                    ranks.update(hit[:1].tolist())
                    absent += hit.size == 0
        assert ranks == set(range(min(n, preds.shape[2]))), (n, s, ranks)
        assert holes > 0, (n, s)
        if s == 'baseline' or n < preds.shape[2]:                # top_n 10 reads all 8 model candidates: always a hit
            assert absent > 0, (n, s)
        assert per_pos[-1] < per_pos[0] / 2 and per_pos[-1] > 0, (n, s, per_pos)     # late positions: few queries
    # the popularity sums depend on their order: summed in fp64, or sessions reversed, some position rounds otherwise
    for n in (1, 3, 10):
        g = _case(n, 'model')
        labels = np.stack([g['b%d/labels' % b] for b in range(4)]).reshape(-1, T)
        differs = False
        for t in range(T):
            v = g['pop'][labels[labels[:, t] != 0, t]]
            fwd = rev = np.float32(0)
            for x in v:
                fwd = np.float32(fwd + x)
            for x in v[::-1]:
                rev = np.float32(rev + x)
            differs |= fwd != rev or fwd != np.float32(v.astype(np.float64).sum())
        assert differs, n


def test_switch_defaults_off_and_params_dict_unchanged():
    from chameleon_recsys_b200.hparams import NARHParams
    args = ({}, {'article_id': {}}, {}, np.zeros((2, 2), np.float32))
    assert NARHParams().eval_metrics_by_session_position is False
    default = NARHParams().to_params(*args)
    assert default['eval_metrics_by_session_position'] is False
    on = NARHParams(eval_metrics_by_session_position=True).to_params(*args)
    assert on['eval_metrics_by_session_position'] is True
    assert set(on) == set(default)
    assert all(on[k] is default[k] or np.array_equal(on[k], default[k]) for k in default
               if k != 'eval_metrics_by_session_position')
