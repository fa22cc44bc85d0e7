"""ClickedItemsState / datasets / plan (host logic) against fixtures generated from the reference's own
classes (tests/golden/make_state_golden.py) and against the reference's documented semantics.  Both the product
class (one C pass in libnar_b200) and the numpy specification (oracle/clicked_items_state_ref.py) are pinned to the
reference's outputs."""
import os

import numpy as np
import pytest

from chameleon_recsys_b200.clicked_items_state import ClickedItemsState, batch_clicks_for_state_update
from chameleon_recsys_b200.datasets import OutOfRangeError, parse_sequence_example, prepare_dataset_iterator
from chameleon_recsys_b200.harness import make_problem
from chameleon_recsys_b200.hparams import get_embedding_size, workload

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize('which', ['product_c_pass', 'numpy_spec'])
def test_state_matches_reference_golden(which):
    from oracle.clicked_items_state_ref import ClickedItemsStateRef
    cls = ClickedItemsState if which == 'product_c_pass' else ClickedItemsStateRef
    g = np.load(os.path.join(HERE, 'golden', 'state_golden.npz'))
    for ci in range(3):
        hours, max_size, n_norm, V = g['c%d_cfg' % ci]
        st = cls(float(hours), int(max_size), int(n_norm), int(V))
        for step in range(6):
            st.update_items_state(g['c%d_items_%d' % (ci, step)], g['c%d_ts_%d' % (ci, step)])
            assert np.array_equal(st.pop_recent_clicks_buffer, g['c%d_buffer_%d' % (ci, step)])
            assert np.array_equal(st.get_articles_recent_pop(), g['c%d_recent_pop_%d' % (ci, step)])
            assert np.array_equal(st.get_articles_recent_pop_norm(), g['c%d_pop_norm_%d' % (ci, step)])
            assert np.array_equal(st.get_articles_pop(), g['c%d_pop_%d' % (ci, step)])


def test_state_invariants():
    st = ClickedItemsState(1.0, 50, 10, 100)
    assert st.get_recent_clicks_buffer().shape == (50,) and not st.get_recent_clicks_buffer().any()
    assert np.all(st.get_articles_recent_pop_norm() == 0.1)
    t0 = 1_000_000_000
    st.update_items_state(np.array([5, 6, 7]), np.array([t0, t0 + 1, t0 + 2]))
    assert list(st.get_recent_clicks_buffer()[:4]) == [7, 6, 5, 0]            # newest first
    st.update_items_state(np.array([8]), np.array([t0 + 2 * 3600 * 1000]))     # two hours later: old clicks dropped
    assert list(st.get_recent_clicks_buffer()[:2]) == [8, 0]
    assert st.get_articles_recent_pop_norm().min() >= 1.0 / 10
    st.save_state_checkpoint()
    st.update_items_state(np.array([9]), np.array([t0 + 2 * 3600 * 1000 + 5]))
    st.restore_state_checkpoint()
    assert list(st.get_recent_clicks_buffer()[:2]) == [8, 0]


def test_batch_clicks_for_state_update():
    items = np.array([[3, 4, 0], [5, 0, 0]]); ts = np.array([[10, 20, 0], [30, 0, 0]]); last = np.array([[9], [8]])
    i, t = batch_clicks_for_state_update(items, ts, last)
    assert list(i) == [3, 4, 9, 5, 8]
    assert list(t) == [10, 20, 20, 30, 30]          # last label inherits the session's max timestamp (:1641-1643)


def test_parse_sequence_example_labels_and_truncation():
    cfg = {'single_features': {'session_size': {'dtype': 'int'}, 'user_id': {'dtype': 'int'}},
           'sequence_features': {'item_clicked': {'dtype': 'int'}, 'event_timestamp': {'dtype': 'int'},
                                 'x': {'dtype': 'float'}}}
    ex = {'session_size': 6, 'user_id': 3, 'item_clicked': [1, 2, 3, 4, 5, 6], 'event_timestamp': [10, 20, 30, 40, 50, 60],
          'x': [.1, .2, .3, .4, .5, .6]}
    p = parse_sequence_example(ex, cfg, truncate_sequence_length=4)
    assert p['session_size'] == 4
    assert list(p['item_clicked']) == [1, 2, 3] and list(p['label_next_item']) == [2, 3, 4] and list(p['label_last_item']) == [4]
    assert p['x'].dtype == np.float32 and p['item_clicked'].dtype == np.int64
    it = prepare_dataset_iterator([ex, dict(ex, session_size=2, item_clicked=[7, 8], event_timestamp=[1, 2], x=[1., 2.])],
                                  cfg, batch_size=2, truncate_session_length=4)
    f, l = it.get_next()
    assert f['item_clicked'].tolist() == [[1, 2, 3], [7, 0, 0]] and l['label_next_item'].tolist() == [[2, 3, 4], [8, 0, 0]]
    assert l['label_last_item'].tolist() == [[4], [8]] and f['session_size'].tolist() == [4, 2]
    with pytest.raises(OutOfRangeError):
        it.get_next()


def test_plan_and_layout_roundtrip():
    assert get_embedding_size(46034) == 117 and get_embedding_size(461) == 37 and get_embedding_size(1000) == 44
    for prof, F in (('A', 1 + 250 + 117), ('B', 71 + 37 + 250 + 117 + 2)):
        pb = make_problem(workload('g1', prof), batch_size=4)
        assert pb.plan.F == F and pb.plan.Fp % 4 == 0
        for s in pb.plan.segments:
            if s.name in ('acr', 'item_emb'):
                assert s.int_col % 4 == 0
        assert sorted(pb.plan.int2log[pb.plan.int2log >= 0].tolist()) == list(range(F))
        if prof == 'B':       # the item table is large; check the round trip on the small profile only once
            continue
        logical = pb.layout.init_logical(1)
        flat = pb.layout.to_internal(logical)
        back = pb.layout.to_logical(flat)
        for k in logical:
            assert np.array_equal(logical[k], back[k]), k
        # padding stays zero
        total_logical = sum(v.size for v in logical.values())
        assert np.count_nonzero(flat) <= total_logical
    pbt = make_problem('tiny', profile='B')
    names = pbt.layout.logical_names()
    assert 'main/RNN/rnn/multi_rnn_cell/cell_0/ugrnn_cell/kernel' in names
    lg = pbt.layout.init_logical(3)
    assert lg['main/RNN/rnn/multi_rnn_cell/cell_0/ugrnn_cell/kernel'].shape == (64 + 64, 128)
    assert np.array_equal(pbt.layout.to_logical(pbt.layout.to_internal(lg))['main/RNN/rnn/multi_rnn_cell/cell_0/ugrnn_cell/kernel'],
                          lg['main/RNN/rnn/multi_rnn_cell/cell_0/ugrnn_cell/kernel'])


def test_checkpoint_file_roundtrip(tmp_path):
    """checkpoint.py: logical tensors, Adam slots, step and ClickedItemsState survive save -> load -> restore; the
    latest file is picked by step number, not by name order."""
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState

    class FakeEngine:
        def __init__(self, seed):
            r = np.random.RandomState(seed)
            self.sd = {'params': {'a/kernel': r.randn(3, 4).astype(np.float32), 'a/bias': r.randn(4).astype(np.float32)},
                       'adam_m': {'a/kernel': r.randn(3, 4).astype(np.float32), 'a/bias': r.randn(4).astype(np.float32)},
                       'adam_v': {'a/kernel': r.rand(3, 4).astype(np.float32), 'a/bias': r.rand(4).astype(np.float32)},
                       'global_step': 7 + seed}

        def state_dict(self):
            return self.sd

        def load_state_dict(self, sd):
            self.sd = sd

    st = ClickedItemsState(1.0, 50, 20, 30)
    st.update_items_state(np.array([3, 4, 4, 9]), np.array([1000, 2000, 3000, 4000]))
    e = FakeEngine(2)
    d = str(tmp_path)
    ckpt.save(ckpt.checkpoint_path(d, 9), e, st)
    ckpt.save(ckpt.checkpoint_path(d, 10), FakeEngine(3), st)
    assert ckpt.latest_checkpoint(d).endswith('model.ckpt-10.npz')       # 10 > 9 numerically
    e2, st2 = FakeEngine(5), ClickedItemsState(1.0, 50, 20, 30)
    step = ckpt.restore(ckpt.checkpoint_path(d, 9), e2, st2)
    assert step == 9 and e2.sd['global_step'] == 9
    for g in ('params', 'adam_m', 'adam_v'):
        for k in e.sd[g]:
            assert np.array_equal(e2.sd[g][k], e.sd[g][k])
    assert np.array_equal(st2.get_recent_clicks_buffer(), st.get_recent_clicks_buffer())
    assert np.array_equal(st2.get_articles_recent_pop_norm(), st.get_articles_recent_pop_norm())
    assert ckpt.latest_checkpoint(str(tmp_path / 'missing')) is None


def test_acr_resource_loaders(tmp_path):
    """nar_utils: G1 csv + pickle and the Adressa tuple pickle; row normalisation equals sklearn's Normalizer."""
    import pickle
    import pandas as pd
    from sklearn.preprocessing import Normalizer
    from chameleon_recsys_b200 import nar_utils
    rs = np.random.RandomState(0)
    emb = rs.randn(6, 5).astype(np.float32); emb[0] = 0
    df = pd.DataFrame({'article_id': np.arange(6), 'category_id': rs.randint(0, 9, 6), 'created_at_ts': rs.randint(1, 10 ** 9, 6)})
    df.to_csv(tmp_path / 'meta.csv', index=False)
    pickle.dump(emb, open(tmp_path / 'emb.pickle', 'wb'))
    pickle.dump(({'category_id': {'a': 1}}, df, emb), open(tmp_path / 'acr.pickle', 'wb'))
    d2, e2 = nar_utils.load_acr_module_resources(str(tmp_path / 'meta.csv'), str(tmp_path / 'emb.pickle'))
    assert np.array_equal(e2, emb) and list(d2.columns) == list(df.columns)
    enc, d3, e3 = nar_utils.load_acr_module_resources_adressa(str(tmp_path / 'acr.pickle'))
    assert enc == {'category_id': {'a': 1}} and np.array_equal(e3, emb) and d3.equals(df)
    meta = nar_utils.process_articles_metadata(d2, {'category_id': {}, 'created_at_ts': {}})
    assert meta['category_id'].dtype == np.int64 and np.array_equal(meta['created_at_ts'], df['created_at_ts'].values)
    got = nar_utils.normalize_content_embeddings(emb, 2.0)
    want = Normalizer(norm='l2').fit_transform(emb) * 2.0
    assert np.allclose(got, want, atol=1e-6) and not got[0].any()


def test_native_state_update_equals_numpy_spec():
    """libnar_b200's nar_host_state_update (C, host) against the numpy restatement, step by step on a stream that
    exercises the hour cut-off, the clip at max size, padding and repeated ids."""
    from chameleon_recsys_b200 import _lib
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from oracle.clicked_items_state_ref import ClickedItemsStateRef
    _lib.load()                                                   # the library must be there: build() made it
    rs = np.random.RandomState(1)
    a = ClickedItemsState(0.5, 300, 50, 400)
    b = ClickedItemsStateRef(0.5, 300, 50, 400)
    t = 1_500_000_000_000
    for step in range(60):
        n = int(rs.randint(1, 90))
        items = rs.randint(1, 400, n).astype(np.int64)
        t += int(rs.randint(0, 600_000))                         # up to 10 min between batches, 30 min window
        ts = (t + rs.randint(-200_000, 200_000, n)).astype(np.int64)
        a.update_items_state(items, ts)                           # native
        b.update_items_state(items, ts)                           # spec
        assert np.array_equal(a.get_recent_clicks_buffer(), b.get_recent_clicks_buffer()), step
        assert np.array_equal(a.pop_recent_clicks_buffer, b.pop_recent_clicks_buffer), step
        assert np.array_equal(a.get_articles_recent_pop(), b.get_articles_recent_pop())
        assert a.get_articles_recent_pop_norm().dtype == np.float64
        assert np.array_equal(a.get_articles_recent_pop_norm(), b.get_articles_recent_pop_norm())   # bit-exact float64
        assert np.array_equal(a.get_articles_pop(), b.get_articles_pop())
    with pytest.raises(ValueError):
        a.update_items_state(np.array([400]), np.array([t]))      # id outside [0, num_items)


def test_native_update_from_batch_equals_hook_spec():
    """update_from_batch (one C pass over the padded batch) == batch_clicks_for_state_update + numpy update."""
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from oracle import clicked_items_state_ref as ref
    pb = make_problem('tiny', profile='B')
    it = pb.input_fn()
    a = ClickedItemsState(1.0, 400, 100, pb.plan.num_items)
    b = ref.ClickedItemsStateRef(1.0, 400, 100, pb.plan.num_items)
    for step in range(12):
        f, l = it.get_next()
        a.update_from_batch(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
        items, ts = ref.batch_clicks_for_state_update(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
        i2, t2 = batch_clicks_for_state_update(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
        assert np.array_equal(items, i2) and np.array_equal(ts, t2)
        b.update_items_state(items, ts)
        assert np.array_equal(a.pop_recent_clicks_buffer, b.pop_recent_clicks_buffer), step
        assert np.array_equal(a.get_articles_recent_pop_norm(), b.get_articles_recent_pop_norm())
        assert np.array_equal(a.get_articles_pop(), b.get_articles_pop())
    z = np.zeros_like(f['item_clicked'])
    before = a.pop_recent_clicks_buffer.copy()
    a.update_from_batch(z, z, np.zeros_like(l['label_last_item']))          # all padding: state untouched
    assert np.array_equal(before, a.pop_recent_clicks_buffer)


def test_shard_bounds_balanced_and_complete():
    """dp.shard_bounds / shard_sessions: the shards are contiguous, disjoint, cover every session, never empty, are the same
    on every rank, and hold (nearly) equal numbers of valid positions; the union of the ranks' position lists is the
    single-rank list (so the summed loss / gradients are those of the global batch whatever the split)."""
    from chameleon_recsys_b200.dp import shard_bounds, shard_sessions
    rng = np.random.default_rng(5)
    T = 20
    for world in (1, 2, 3, 8):
        for Bg in (world, 17, 256, 2048):
            if Bg < world:
                continue
            size = rng.geometric(0.35, Bg) + 1                         # session_size incl. the label click
            size[rng.random(Bg) < 0.1] = 1                             # sessions without a valid position
            lens = np.clip(size - 1, 0, T)
            b = shard_bounds(lens, world)
            assert b[0] == 0 and b[-1] == Bg and (np.diff(b) >= 1).all()
            full = shard_sessions(size, T, 1, 0)
            parts = [shard_sessions(size, T, world, r) for r in range(world)]
            assert [p['s0'] for p in parts] == list(b[:-1]) and [p['per'] for p in parts] == list(np.diff(b))
            assert np.array_equal(np.concatenate([p['pos_idx'] for p in parts]), full['pos_idx'])
            assert sum(p['L'] for p in parts) == full['L'] == parts[0]['L_global']
            for p in parts:
                assert p['sess_off'][-1] == p['L'] and len(p['sess_off']) == p['per'] + 1
            if Bg >= 256:
                Ls = np.array([p['L'] for p in parts], dtype=np.float64)
                assert Ls.max() <= Ls.mean() + T                       # within one session of the mean
    # equal-count split on request (and its divisibility rule)
    assert list(shard_bounds(np.ones(8, np.int64), 4, balance=False)) == [0, 2, 4, 6, 8]
    with pytest.raises(ValueError):
        shard_bounds(np.ones(9, np.int64), 4, balance=False)
    with pytest.raises(ValueError):
        shard_bounds(np.ones(3, np.int64), 4)
    assert list(shard_bounds(np.zeros(5, np.int64), 2)) == [0, 2, 5]    # nothing to balance: near-equal counts


def test_hook_matches_reference_hook():
    """ItemsStateUpdaterHook.before_run / after_run + ClickedItemsState (the product's C pass) against the REFERENCE hook
    and state class run over the same training batches (tests/golden/make_hook_golden.py: nar_model.py:1435-1470 feed,
    :1635-1650 flattening of [clicked | last label] with the label click borrowing the session's last timestamp)."""
    from chameleon_recsys_b200.hparams import ModeKeys
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'hook_golden.npz'))
    for ci in range(2):
        hours, max_size, n_norm, V = d['c%d_cfg' % ci]
        state = ClickedItemsState(float(hours), int(max_size), int(n_norm), int(V))
        hook = ItemsStateUpdaterHook(ModeKeys.TRAIN, None, 3, state)
        hook.begin()
        for step in range(5):
            feed = hook.before_run(None)
            assert np.array_equal(feed['pop_recent_items_buffer'], d['c%d_feed_buffer_%d' % (ci, step)])
            assert np.array_equal(np.asarray(feed['articles_recent_pop_norm']), d['c%d_feed_pop_norm_%d' % (ci, step)])
            hook.after_run(None, {'clicked_items': d['c%d_item_clicked_%d' % (ci, step)],
                                  'clicked_timestamps': d['c%d_event_timestamp_%d' % (ci, step)],
                                  'last_item_label': d['c%d_label_last_item_%d' % (ci, step)]})
            assert np.array_equal(state.pop_recent_clicks_buffer, d['c%d_buffer_%d' % (ci, step)]), (ci, step)
            assert np.array_equal(state.get_articles_recent_pop(), d['c%d_recent_pop_%d' % (ci, step)])
            assert np.array_equal(state.get_articles_recent_pop_norm(), d['c%d_pop_norm_%d' % (ci, step)])      # float64, bit-exact
            assert np.array_equal(state.get_articles_pop(), d['c%d_pop_%d' % (ci, step)])
        hook.end()


def test_checkpoint_accepts_tf_variable_names(tmp_path):
    """checkpoint.load maps the names TensorFlow gives the shared Dense layers (scope of their first call; observed by running
    the reference model code, tests/golden/model_golden.npz) onto plan.ParamLayout's names."""
    from chameleon_recsys_b200 import checkpoint as ckpt
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'model_golden.npz'))
    from oracle.golden_sampling import preset_variables
    tf_names = [str(n) for n in d['train64/var_names']]
    pb = make_problem('tiny', profile='B')
    ours = set(pb.layout.init_logical(1).keys())
    assert set(ckpt.layout_name(n + ':0') for n in tf_names) == ours
    assert any(ckpt.layout_name(n) != n for n in tf_names)
    path = str(tmp_path / 'model.ckpt-7.npz')
    values = preset_variables(d, 'train64')
    np.savez(path, global_step=np.int64(7), **{'params/' + n: values[n] for n in tf_names})
    ck = ckpt.load(path)
    assert set(ck['params'].keys()) == ours and ck['global_step'] == 7


def test_feature_config_builders_match_reference_trainer():
    """hparams.get_*_features_config against the reference trainer's builders (nar_trainer_gcom.py:99-231, run by
    tests/golden/make_model_fn_golden.py) under three flag settings.  The one documented difference: this repo always sets
    the article_id / item_clicked cardinality to the catalogue size (the gcom trainer hard-codes 364047 for item_clicked and
    forgets article_id, which nar_model.py:183 reads)."""
    import json
    from chameleon_recsys_b200.hparams import (get_articles_features_config, get_internal_enabled_features_config,
                                               get_session_features_config)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'model_fn_golden.json')) as f:
        g = json.load(f)['feature_configs']
    assert len(g) == 3
    for c in g:
        clicks, arts, internal = c['flags']
        ours_s = get_session_features_config(364047, clicks)
        assert ours_s == c['session']
        assert list(ours_s['sequence_features']) == list(c['session']['sequence_features'])      # order = feature column order
        ours_a = get_articles_features_config(1000, arts)
        ref_a = dict(c['articles'])
        ref_a['article_id'] = dict(ref_a['article_id'], cardinality=1000)
        assert ours_a == ref_a and list(ours_a) == list(ref_a)
        assert get_internal_enabled_features_config(internal) == c['internal']
