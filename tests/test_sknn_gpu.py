"""Session-based kNN baselines on the H100 (csrc/sknn.cu, chameleon_recsys_b200/sknn.py) against the plain-Python oracle
(oracle/sknn_ref.py): the ring and its live bits after many updates, top-n ids and the accumulator bit for bit at small
and G1 shapes, and Estimator.train + evaluate end to end (ring restored, the other baselines and the model's numbers
unchanged, checkpoint round trip).  The parameter checks need no GPU."""
import numpy as np
import pytest

from oracle.baselines_ref import SUFFIXES
from oracle.sknn_ref import SknnRef

gpu = pytest.mark.gpu
KNN_ALL = [{'recommender': s, 'params': {}} for s in SUFFIXES] + [{'recommender': 'v-sknn', 'params': {}}]


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sessions(rs, B, T1, V, min_len=1):
    ai = np.zeros((B, T1), dtype=np.int64)
    for b in range(B):
        n = int(rs.randint(min_len, T1 + 1))
        ai[b, :n] = rs.zipf(1.3, n) % (V - 1) + 1
    return ai


def _ids(rs, step, B):
    """Ascending by batch, jittered within it (so the buffer's binary search misses some)."""
    return 1000 * (step * B + np.arange(B, dtype=np.int64)) + rs.randint(0, 2500, size=B)


def _tables(V, params, suffix='v-sknn'):
    from chameleon_recsys_b200.baselines import BaselineTables
    return BaselineTables([{'recommender': suffix, 'params': params}], V)


def _ref(p, suffix='v-sknn'):
    return SknnRef(p.get('sessions_buffer_size', 3000), p.get('candidate_sessions_sample_size', 1000),
                   p.get('nearest_neighbor_session_for_scoring', 500), p.get('similarity', 'cosine'),
                   p.get('first_session_clicks_decay', 'div' if suffix == 'v-sknn' else 'same'))


def _check_ring(tab, ref, suffix):
    got, want = tab.export_knn(suffix), ref.export()
    np.testing.assert_array_equal(got['ids'], want['ids'])
    np.testing.assert_array_equal(got['lens'], want['lens'])
    W = want['items'].shape[1]
    np.testing.assert_array_equal(got['items'][:, :W], want['items'])
    assert not got['items'][:, W:].any()
    np.testing.assert_array_equal(got['live'][:, :W], want['live'])
    return bool((want['items'] > 0).sum() > want['live'].sum())       # some pair was discarded by a twin's eviction


@gpu
@pytest.mark.parametrize('S,B', [(40, 16), (16, 16), (200, 24)])
def test_ring_matches_oracle(S, B):
    rs = np.random.RandomState(S + B)
    V, T1 = 30, 9
    p = {'sessions_buffer_size': S}
    tab, ref = _tables(V, p), _ref(p)
    prev, dead = None, False
    for step in range(14):
        if step in (4, 9) and prev is not None:
            sid, ai = prev                                          # the same sessions trained twice
        elif step == 6:
            sid, ai = 500 - 10 * np.arange(B, dtype=np.int64), _sessions(rs, B, T1, V)   # ids going backwards
        else:
            sid, ai = _ids(rs, step, B), _sessions(rs, B, T1, V)
        tab.update(_dev(ai), session_ids=sid)
        ref.update(sid, ai)
        prev = (sid, ai)
        dead |= _check_ring(tab, ref, 'v-sknn')
    assert dead
    tab.snapshot()
    ref.snapshot()
    for step in range(3):
        sid, ai = _ids(rs, 20 + step, B), _sessions(rs, B, T1, V)
        tab.update(_dev(ai), session_ids=sid)
        ref.update(sid, ai)
    tab.restore()
    ref.restore()
    _check_ring(tab, ref, 'v-sknn')


def _score_case(B, T, K, V, top_n, seed, params, suffix, n_train):
    import torch
    rs = np.random.RandomState(seed)
    tab, ref = _tables(V, params, suffix), _ref(params, suffix)
    for step in range(n_train):
        sid, ai = _ids(rs, step, B), _sessions(rs, B, T + 1, V, min_len=2)
        tab.update(_dev(ai), session_ids=sid)
        ref.update(sid, ai)
    ai = _sessions(rs, B, T + 1, V, min_len=2)
    ic, ln = ai[:, :T].copy(), ai[:, 1:].copy()
    ln[ic == 0] = 0
    neg = rs.randint(1, V, size=(B, T, K)).astype(np.int64)
    neg[rs.rand(B, T, K) < 0.1] = 0
    rows = tab.n_rows
    metrics = torch.zeros(rows, 3, dtype=torch.float64, device='cuda')
    out = torch.zeros(rows, B * T, top_n, dtype=torch.int64, device='cuda')
    tab.score(_dev(ic), _dev(ln), _dev(neg), None, None, top_n, metrics, out_ids=out)
    tab.check_errors()
    row = len(SUFFIXES) + ('v-sknn', 'sknn').index(suffix)
    return out.cpu().numpy()[row], metrics.cpu().numpy()[row], ref.score(ic, ln, neg, top_n)


SMALL = [
    ('v-sknn', {'sessions_buffer_size': 30, 'candidate_sessions_sample_size': 12, 'nearest_neighbor_session_for_scoring': 6}),
    ('sknn', {'sessions_buffer_size': 30, 'candidate_sessions_sample_size': 12, 'nearest_neighbor_session_for_scoring': 6,
              'similarity': 'jaccard'}),
    ('v-sknn', {'sessions_buffer_size': 30, 'candidate_sessions_sample_size': 0, 'nearest_neighbor_session_for_scoring': 8,
                'similarity': 'jaccard'}),
    ('sknn', {'sessions_buffer_size': 50, 'candidate_sessions_sample_size': 0, 'nearest_neighbor_session_for_scoring': 50}),
]


@gpu
@pytest.mark.parametrize('case', range(len(SMALL)))
def test_scoring_matches_oracle_small(case):
    suffix, params = SMALL[case]
    got, m, want = _score_case(8, 6, 7, 25, 5, case, params, suffix, n_train=6)
    np.testing.assert_array_equal(got, want['ids'])
    assert m.tolist() == [want['hits'], want['rr'], want['count']]
    assert want['hits'] > 0


@gpu
def test_scoring_matches_oracle_g1():
    """G1 shapes with the reference parameters: B 256, T 20, K 50, 13 batches (3 328 sessions) folded into 3 000 slots."""
    got, m, want = _score_case(256, 20, 50, 5000, 10, 7, {}, 'v-sknn', n_train=13)
    np.testing.assert_array_equal(got, want['ids'])
    assert m.tolist() == [want['hits'], want['rr'], want['count']]
    assert want['hits'] > 0


def test_knn_parameters_are_checked():
    from chameleon_recsys_b200.baselines import parse_classifiers
    p = parse_classifiers(['v-sknn', {'recommender': 'sknn', 'params': {'similarity': 'jaccard'}}])
    assert p['v-sknn']['first_session_clicks_decay'] == 'div' and p['v-sknn']['sessions_buffer_size'] == 3000
    assert p['sknn']['first_session_clicks_decay'] == 'same' and p['sknn']['similarity'] == 'jaccard'
    with pytest.raises(NotImplementedError, match='v-sknn'):
        parse_classifiers(['vsknn'])
    for bad in ({'sampling_strategy': 'random'}, {'first_session_clicks_decay': 'log'},
                {'first_session_clicks_decay': 'linear'}, {'first_session_clicks_decay': 'same'},
                {'similarity': 'dice'}, {'sessions_buffer_size': 4097}, {'sessions_buffer_size': 0},
                {'nearest_neighbor_session_for_scoring': -1}):
        with pytest.raises(ValueError):
            parse_classifiers([{'recommender': 'v-sknn', 'params': bad}])


@gpu
def test_knn_update_errors():
    tab = _tables(30, {'sessions_buffer_size': 8})
    ai = _dev(np.ones((9, 4), dtype=np.int64))
    with pytest.raises(ValueError):
        tab.update(ai)                                              # no session ids
    with pytest.raises(ValueError):
        tab.update(ai, session_ids=np.arange(9))                    # more sessions than the buffer holds


def _problem():
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 2)
    return pb


def _est(pb, d, state, benchmarks):
    from chameleon_recsys_b200.estimator import build_estimator
    hp = pb.hp.copy(eval_benchmarks=tuple(benchmarks))
    return build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                           pb.session_features_config, hp, state, device=0)


@gpu
@pytest.mark.parametrize('device_state', ['1', '0'])
def test_estimator_with_knn(device_state, tmp_path, monkeypatch):
    """Runs without baselines (twice: the control spread), with the five others, with all six and with V-SkNN alone, on
    the same batches: the engine launches are the same, the model's numbers within the control spread, the five others'
    numbers unchanged by V-SkNN, V-SkNN's numbers those of the oracle, its ring restored after evaluate, and a fresh
    Estimator on model_dir reproduces them."""
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    monkeypatch.setenv('NAR_DEVICE_STATE', device_state)
    five = [{'recommender': s, 'params': {}} for s in SUFFIXES]
    runs = {}
    for name, bench in (('off', []), ('control', []), ('five', five), ('six', KNN_ALL),
                        ('knn', [{'recommender': 'v-sknn', 'params': {}}])):
        pb = _problem()
        it = pb.input_fn()
        train_batches = [it.get_next() for _ in range(6)]
        eval_batches = [it.get_next() for _ in range(3)]
        d = str(tmp_path / name)
        est = _est(pb, d, pb.clicked_items_state, bench)
        losses = []
        for i in range(3):
            est.train(lambda i=i: iter(train_batches[2 * i:2 * i + 2]))
            losses.append(est.last_loss)
        launches = est.model.engine.launches
        tables = pb.clicked_items_state.baselines
        before = tables.export_knn('v-sknn') if tables is not None and tables.knn else None
        ev = est.evaluate(lambda: iter(eval_batches))
        if before is not None:
            after = tables.export_knn('v-sknn')
            for k in before:
                np.testing.assert_array_equal(after[k], before[k], err_msg=k)
        runs[name] = (losses, ev, launches, pb, d, train_batches, eval_batches)
    off = runs['off']
    for name in ('control', 'five', 'six', 'knn'):
        run = runs[name]
        assert run[2] == off[2], name
        for a, b in zip(run[0] + [run[1]['loss']], off[0] + [off[1]['loss']]):
            assert abs(a - b) <= 1e-5 * abs(b), (name, a, b)
        for k in ('hitrate_at_n', 'mrr_at_n'):
            assert abs(run[1][k] - off[1][k]) <= 1.0 / 100, (name, k)
    for s in SUFFIXES:
        for m in ('hitrate', 'mrr'):
            k = '%s_at_n_%s' % (m, s)
            assert runs['six'][1][k] == runs['five'][1][k], k
    for m in ('hitrate', 'mrr'):
        k = '%s_at_n_v-sknn' % m
        assert runs['six'][1][k] == runs['knn'][1][k], k
    assert set(runs['six'][1]) - set(off[1]) == {'%s_at_n_%s' % (m, s) for m in ('hitrate', 'mrr')
                                                 for s in SUFFIXES + ('v-sknn',)}

    _, ev, _, pb, d, train_batches, eval_batches = runs['knn']
    assert ev['hitrate_at_n_v-sknn'] > 0

    # checkpoint round trip: a fresh Estimator on model_dir reproduces the V-SkNN metrics
    st = pb.clicked_items_state
    saved = ckpt.load(ckpt.latest_checkpoint(d))
    assert saved['baselines']['sknn_v-sknn_ids'].size > 0
    fresh_state = ClickedItemsState(st.recent_clicks_buffer_hours, st.recent_clicks_buffer_max_size,
                                    st.recent_clicks_for_normalization, st.num_items)
    for f in ckpt.STATE_FIELDS:
        setattr(fresh_state, f, np.array(saved['state'][f]))
    fresh = _est(pb, d, fresh_state, [{'recommender': 'v-sknn', 'params': {}}])
    ev2 = fresh.evaluate(lambda: iter(eval_batches))
    for k in ('hitrate_at_n_v-sknn', 'mrr_at_n_v-sknn'):
        assert ev2[k] == ev[k], k


@gpu
def test_estimator_knn_matches_oracle(monkeypatch):
    """V-SkNN's numbers from Estimator.evaluate equal the oracle's over the same batches and the negatives the engine
    drew (recorded in the hook)."""
    import torch
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    est = _est(pb, None, pb.clicked_items_state, [{'recommender': 'v-sknn', 'params': {}}])
    est.train(lambda: iter(train_batches))
    seen = []
    orig = ItemsStateUpdaterHook.after_run

    def spy(self, run_context, run_values):
        if 'eval_batch_negative_items' in run_values:
            seen.append(run_values['eval_batch_negative_items'].cpu().numpy().copy())
        return orig(self, run_context, run_values)
    monkeypatch.setattr(ItemsStateUpdaterHook, 'after_run', spy)
    ev = est.evaluate(lambda: iter(eval_batches))
    ref = SknnRef()
    for f, l in train_batches:
        ref.update(f['session_id'], np.concatenate([f['item_clicked'], l['label_last_item'].reshape(-1, 1)], axis=1))
    h = rr = n = 0.0
    for (f, l), neg in zip(eval_batches, seen):
        r = ref.score(f['item_clicked'], l['label_next_item'], neg, pb.hp.eval_metrics_top_n)
        h += r['hits']; rr += r['rr']; n += r['count']
        ref.update(f['session_id'], np.concatenate([f['item_clicked'], l['label_last_item'].reshape(-1, 1)], axis=1))
    assert ev['hitrate_at_n_v-sknn'] == h / n and ev['mrr_at_n_v-sknn'] == rr / n
    torch.cuda.synchronize()
