"""oracle/session_logs_ref.py and the nar_trainer writers against tests/golden/session_logs_golden.npz: the lists the
reference hook's own logging block filled over 3 batches, and the files the reference trainer's own writers made of them
(tests/golden/make_session_logs_golden.py)."""
import json
import os

import numpy as np
import pytest

from chameleon_recsys_b200 import nar_trainer
from oracle.session_logs_ref import scatter_compact, session_logs_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'session_logs_golden.npz')
REC_KEYS = ['session_id', 'next_click_labels', 'predicted_item_ids', 'predicted_item_probs', 'predicted_item_norm_pop']


@pytest.fixture(scope='module')
def golden():
    g = np.load(GOLDEN)
    return g, json.loads(str(g['neg_log_json'])), json.loads(str(g['rec_log_json']))


def _bits(rows):
    return [np.asarray(r, dtype=np.float64).astype(np.float32).view(np.uint32).tolist() for r in rows]


def _batches(g):
    for b in range(3):
        yield b, {k: g['b%d/%s' % (b, k)] for k in ('labels', 'neg', 'ids', 'probs', 'pop', 'sids', 'lens')}


@pytest.mark.parametrize('pop_dtype', [np.float64, np.float32])
def test_oracle_matches_reference_hook_after_every_batch(golden, pop_dtype):
    g, want_neg, want_rec = golden
    B = int(g['cfg'][1])
    got_neg, got_rec = [], []
    for b, a in _batches(g):
        neg, rec = session_logs_ref(a['sids'], a['labels'], a['neg'], a['ids'], a['probs'], a['pop'].astype(pop_dtype))
        got_neg += neg
        got_rec += rec
        n = int(g['entries_after_batch'][b])
        assert len(got_neg) == len(got_rec) == n == (b + 1) * B
        assert got_neg == want_neg[:n]                               # keys, nesting, lengths, ids
        for got, want in zip(got_rec, want_rec[:n]):
            assert list(got) == list(want) == REC_KEYS                # key order
            for k in REC_KEYS[:3]:
                assert got[k] == want[k], k
            assert len(got['predicted_item_probs']) == len(want['next_click_labels'])
            # a float32 widens exactly: equal doubles and equal float32 bit patterns
            assert got['predicted_item_probs'] == want['predicted_item_probs']
            assert _bits(got['predicted_item_probs']) == _bits(want['predicted_item_probs'])
            gp, wp = np.asarray(got['predicted_item_norm_pop']), np.asarray(want['predicted_item_norm_pop'])
            assert gp.shape == wp.shape
            if pop_dtype is np.float64:
                assert got['predicted_item_norm_pop'] == want['predicted_item_norm_pop']
            elif gp.size:
                assert np.abs(gp - wp).max() <= 1e-7
    assert len(want_neg) == len(got_neg)


def test_fixture_covers_the_hard_cases(golden):
    g, want_neg, want_rec = golden
    lens = np.concatenate([a['lens'] for _, a in _batches(g)])
    T = int(g['cfg'][2])
    assert set(lens.tolist()) == set(range(T + 1))                    # sessions without a query up to full ones
    assert any(len(e['negative_items']) == 0 for e in want_neg)
    hole = [(a['labels'] == 0) & (np.arange(T)[None, :] < a['lens'][:, None]) for _, a in _batches(g)]
    assert sum(int(h.sum()) for h in hole) == 1                       # one label-0 hole inside a session
    assert any(len(e['session_id']) == 17 for e in want_rec)
    probs = np.concatenate([a['probs'][a['labels'] != 0].reshape(-1) for _, a in _batches(g)])
    x = probs * np.float32(1e7)
    assert x.dtype == np.float32
    assert ((x - np.floor(x)) == 0.5).sum() >= 10                     # ties of the rounding
    assert ((probs > 0) & (probs < 5e-8)).any() and (probs == 0).any() and (probs == 1).any()
    assert ((probs > 0) & (probs < np.finfo(np.float32).tiny)).any()  # a denormal
    pops = np.concatenate([a['pop'] for _, a in _batches(g)])
    assert (pops == pops.min()).mean() > 0.5                          # most articles sit at the floor


def test_compact_rows_give_the_same_logs(golden):
    g, _, _ = golden
    for _, a in _batches(g):
        B, T = a['labels'].shape
        pos_idx = np.flatnonzero((np.arange(T)[None, :] < a['lens'][:, None]).reshape(-1)).astype(np.int32)
        ids_c, probs_c = a['ids'].reshape(B * T, -1)[pos_idx], a['probs'].reshape(B * T, -1)[pos_idx]
        assert np.array_equal(scatter_compact(ids_c, pos_idx, B, T), a['ids'])
        want = session_logs_ref(a['sids'], a['labels'], a['neg'], a['ids'], a['probs'], a['pop'])
        assert session_logs_ref(a['sids'], a['labels'], a['neg'], ids_c, probs_c, a['pop'], pos_idx=pos_idx) == want
        assert session_logs_ref(a['sids'], a['labels'], a['neg']) == (want[0], None)
        assert session_logs_ref(a['sids'], a['labels'], None, a['ids'], a['probs'], a['pop']) == (None, want[1])


def test_float32_rounding_steps_are_ndarray_round():
    """ndarray.round(decimals=7) on float32 = multiply, round half to even, divide, each in float32: the three steps the
    pack kernel takes (__fmul_rn, rintf, __fdiv_rn)."""
    g = np.load(GOLDEN)
    rs = np.random.RandomState(5)
    x = np.concatenate([rs.rand(200000).astype(np.float32), (rs.rand(50000) * 1e-5).astype(np.float32),
                        np.concatenate([g['b%d/probs' % b].reshape(-1) for b in range(3)]),
                        ((np.arange(4000) + 0.5) / 1e7).astype(np.float32)])
    scale = np.float32(1e7)
    steps = np.rint(x * scale) / scale
    assert steps.dtype == np.float32
    assert np.array_equal(steps.view(np.uint32), x.round(decimals=7).view(np.uint32))


def test_writers_reproduce_the_reference_files(golden, tmp_path):
    g, want_neg, want_rec = golden
    nar_trainer.save_sessions_negative_items(str(tmp_path), want_neg)
    nar_trainer.save_sessions_chameleon_recommendations_log(str(tmp_path), want_rec, 3)
    assert (tmp_path / 'eval_sessions_negative_samples.json').read_text() == str(g['neg_file_text'])
    assert (tmp_path / 'eval_chameleon_recommendations_log.json').read_text() == str(g['rec_file_text'])
    # appended to, never truncated
    nar_trainer.save_sessions_negative_items(str(tmp_path), want_neg[:2])
    assert (tmp_path / 'eval_sessions_negative_samples.json').read_text().count('\n') == len(want_neg) + 2


def test_writers_on_the_float32_popularity_lists(golden, tmp_path):
    """The lists as this project fills them (popularity gathered from the float32 array the model was fed): every line
    equals the reference's except the popularity field, compared parsed, to 1e-7."""
    g, _, _ = golden
    neg, rec = [], []
    for _, a in _batches(g):
        n, r = session_logs_ref(a['sids'], a['labels'], a['neg'], a['ids'], a['probs'], a['pop'].astype(np.float32))
        neg += n
        rec += r
    nar_trainer.save_sessions_negative_items(str(tmp_path), neg)
    nar_trainer.save_sessions_chameleon_recommendations_log(str(tmp_path), rec, 3)
    assert (tmp_path / 'eval_sessions_negative_samples.json').read_text() == str(g['neg_file_text'])
    got = (tmp_path / 'eval_chameleon_recommendations_log.json').read_text().splitlines()
    want = str(g['rec_file_text']).splitlines()
    assert len(got) == len(want)
    for gl, wl in zip(got, want):
        gd, wd = json.loads(gl), json.loads(wl)
        assert list(gd) == list(wd) == ['eval_hour_id'] + REC_KEYS
        gp, wp = np.asarray(gd.pop('predicted_item_norm_pop')), np.asarray(wd.pop('predicted_item_norm_pop'))
        assert gd == wd and gp.shape == wp.shape and (gp.size == 0 or np.abs(gp - wp).max() <= 1e-7)
        assert json.dumps(gd) == json.dumps(wd)
