"""Baseline recommenders on the H100 (csrc/baselines.cu, chameleon_recsys_b200/baselines.py) against the numpy oracle
(oracle/baselines_ref.py): pair tables (with growth), scoring / ranking / metrics, and Estimator.train + evaluate end
to end (NAR numbers unchanged, tables restored after evaluation, checkpoint round trip)."""
import numpy as np
import pytest

from oracle.baselines_ref import SUFFIXES, BaselinesRef

pytestmark = pytest.mark.gpu
ALL = [{'recommender': s, 'params': {}} for s in SUFFIXES]


def _batch(rs, B, T, V, min_len=1):
    ai = np.zeros((B, T + 1), dtype=np.int64)
    for b in range(B):
        n = int(rs.randint(min_len, T + 2))
        ai[b, :n] = rs.zipf(1.3, n) % (V - 1) + 1
    return ai


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize('capacity', [16, 1 << 16])
def test_tables_match_oracle(capacity):
    from chameleon_recsys_b200.baselines import BaselineTables
    rs = np.random.RandomState(3)
    V = 300
    tab = BaselineTables(['coocurrent', 'sr'], V, capacity=capacity)
    ref = BaselinesRef(V)
    for _ in range(12):
        ai = _batch(rs, 24, 12, V)
        tab.update(_dev(ai))
        ref.update(ai)
    got, want = tab.export(), ref.export()
    if capacity == 16:
        assert tab.cap >= 8 * 16                                   # grew several times
    for k in ('keys', 'cooc', 'sr_w', 'sr_first'):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


def _score_case(B, T, K, V, top_n, seed, n_train=6):
    import torch
    from chameleon_recsys_b200.baselines import BaselineTables
    rs = np.random.RandomState(seed)
    acr = rs.randn(V, 24).astype(np.float32)
    acr[0] = 0.0
    acr_d = _dev(np.pad(acr, ((0, 0), (0, 8))))                      # leading dimension > dim
    tab = BaselineTables(ALL, V, acr=acr_d, acr_dim=24, capacity=64)
    ref = BaselinesRef(V, acr=acr.astype(np.float64))
    for _ in range(n_train):
        ai = _batch(rs, B, T, V, min_len=2)
        tab.update(_dev(ai))
        ref.update(ai)
    ic = _batch(rs, B, T - 1, V, min_len=2)
    ln = np.zeros((B, T), dtype=np.int64)
    ln[:, :-1] = ic[:, 1:]
    ic = ic[:, :T]
    ln[ic == 0] = 0
    neg = rs.randint(1, V, size=(B, T, K)).astype(np.int64)
    neg[rs.rand(B, T, K) < 0.1] = 0
    buf = np.where(rs.rand(4 * B) < 0.8, rs.zipf(1.3, 4 * B) % (V - 1) + 1, 0).astype(np.int64)
    pop = rs.randint(0, 50, size=V).astype(np.int64)
    metrics = torch.zeros(5, 3, dtype=torch.float64, device='cuda')
    out = torch.zeros(5, B * T, top_n, dtype=torch.int64, device='cuda')
    tab.score(_dev(ic), _dev(ln), _dev(neg), buf, pop, top_n, metrics, out_ids=out)
    tab.check_errors()
    want = ref.score(ic, ln, neg, buf, pop, top_n)
    return out.cpu().numpy(), metrics.cpu().numpy(), want, ref, (ic, ln, neg, buf, pop)


@pytest.mark.parametrize('shape', [(8, 6, 7, 40, 5), (256, 20, 50, 5000, 10)], ids=['small', 'g1'])
def test_scoring_matches_oracle(shape):
    B, T, K, V, top_n = shape
    got, m, want, ref, (ic, ln, neg, buf, pop) = _score_case(B, T, K, V, top_n, seed=B)
    for i, sfx in enumerate(SUFFIXES):
        w = want[sfx]
        if sfx != 'cb':
            np.testing.assert_array_equal(got[i], w['ids'], err_msg=sfx)
            assert m[i].tolist() == [w['hits'], w['rr'], w['count']], sfx
            continue
        # cb: equal except where two candidates' fp64 cosines lie within 1e-6
        for q in np.flatnonzero(ln.reshape(-1)):
            sc = ref.candidate_scores('cb', ic.reshape(-1)[q], [ln.reshape(-1)[q]] + neg.reshape(B * T, K)[q].tolist(), buf, pop)
            v = np.sort(np.array(list(sc.values())))
            if np.any(np.diff(v) < 1e-6):
                continue
            np.testing.assert_array_equal(got[i][q], w['ids'][q])
        assert m[i][2] == w['count']


def test_unsupported_requests_raise():
    from chameleon_recsys_b200.baselines import parse_classifiers
    with pytest.raises(NotImplementedError):
        parse_classifiers([{'recommender': 'vsknn', 'params': {}}])
    with pytest.raises(ValueError):
        parse_classifiers([{'recommender': 'sr', 'params': {'dist_between_clicks_decay': 'linear'}}])
    with pytest.raises(ValueError):
        parse_classifiers([{'recommender': 'sr', 'params': {'max_clicks_dist': 21}}])
    with pytest.raises(ValueError):
        parse_classifiers(['gru4rec'])


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


@pytest.mark.parametrize('device_state', ['1', '0'])
def test_nar_numbers_unchanged(device_state, monkeypatch):
    """Training and evaluation with the baselines on launch exactly the engine work of a run with them off, and give the
    model's numbers of such a run.  The engine's training is not bit-reproducible run to run (float32 atomics in the loss
    and gradient reductions): a second run with the baselines off is the control, and on H100 it differs from the first
    in the last bits of the losses and, through near-tied logits, by a rank of one query in MRR.  So the losses are
    compared to 1e-5 relative and HR / MRR to one query's worth (1 / queries)."""
    monkeypatch.setenv('NAR_DEVICE_STATE', device_state)
    res = {}
    for name, on in (('off', False), ('control', False), ('on', True)):
        pb = _problem()
        est = _est(pb, None, pb.clicked_items_state, ALL if on else [])
        losses = []
        for _ in range(3):
            est.train(pb.input_fn, steps=2)
            losses.append(est.last_loss)
        launches = est.model.engine.launches
        ev = est.evaluate(pb.input_fn, steps=2)
        res[name] = (losses, ev, launches)
    off = res['off']
    for name in ('control', 'on'):
        run = res[name]
        assert run[2] == off[2], name                                   # the same engine launches
        for a, b in zip(run[0] + [run[1]['loss']], off[0] + [off[1]['loss']]):
            assert abs(a - b) <= 1e-5 * abs(b), (name, a, b)
        assert run[1]['global_step'] == off[1]['global_step']
        for k in ('hitrate_at_n', 'mrr_at_n'):
            assert abs(run[1][k] - off[1][k]) <= 1.0 / 100, (name, k)    # < 1 / queries (153 here)
    assert set(res['on'][1]) - set(off[1]) == {'%s_at_n_%s' % (m, s) for m in ('hitrate', 'mrr') for s in SUFFIXES}


def test_estimator_end_to_end(tmp_path, monkeypatch):
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    pb = _problem()
    st = pb.clicked_items_state
    est = _est(pb, str(tmp_path), st, ALL)
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(5)]
    eval_batches = [it.get_next() for _ in range(3)]
    est.train(lambda: iter(train_batches))
    tables = st.baselines
    before = tables.export()

    seen = []
    orig = ItemsStateUpdaterHook.after_run

    def spy(self, run_context, run_values):
        if 'eval_batch_negative_items' in run_values:
            seen.append((run_values['eval_batch_negative_items'].cpu().numpy().copy(),
                         self.clicked_items_state.get_recent_clicks_buffer().copy(),
                         self.clicked_items_state.get_articles_pop().copy()))
        return orig(self, run_context, run_values)
    monkeypatch.setattr(ItemsStateUpdaterHook, 'after_run', spy)
    ev = est.evaluate(lambda: iter(eval_batches))
    after = tables.export()
    for k in before:
        np.testing.assert_array_equal(after[k], before[k], err_msg=k)

    # the oracle over the same batches and the negatives the engine drew
    V = pb.wl.num_items
    ref = BaselinesRef(V, acr=pb.content_article_embeddings_matrix)
    for f, l in train_batches:
        ref.update(np.concatenate([f['item_clicked'], l['label_last_item'].reshape(-1, 1)], axis=1))
    tot = {s: [0.0, 0.0, 0.0] for s in SUFFIXES}
    for (f, l), (neg, buf, pop) in zip(eval_batches, seen):
        r = ref.score(f['item_clicked'], l['label_next_item'], neg, buf, pop, pb.hp.eval_metrics_top_n)
        for s in SUFFIXES:
            for i, k in enumerate(('hits', 'rr', 'count')):
                tot[s][i] += r[s][k]
        ref.update(np.concatenate([f['item_clicked'], l['label_last_item'].reshape(-1, 1)], axis=1))
    for s in SUFFIXES:
        h, rr, n = tot[s]
        if s == 'cb':
            assert abs(ev['hitrate_at_n_cb'] - h / n) <= 2.0 / n and abs(ev['mrr_at_n_cb'] - rr / n) <= 2.0 / n
        else:
            assert ev['hitrate_at_n_' + s] == h / n and ev['mrr_at_n_' + s] == rr / n, s

    # checkpoint round trip: a fresh Estimator on model_dir reproduces the baseline metrics
    monkeypatch.setattr(ItemsStateUpdaterHook, 'after_run', orig)
    path = ckpt.latest_checkpoint(str(tmp_path))
    saved = ckpt.load(path)
    assert saved['baselines'] and np.array_equal(saved['baselines']['keys'], before['keys'])
    fresh_state = ClickedItemsState(st.recent_clicks_buffer_hours, st.recent_clicks_buffer_max_size,
                                    st.recent_clicks_for_normalization, st.num_items)
    for f in ckpt.STATE_FIELDS:
        setattr(fresh_state, f, np.array(saved['state'][f]))
    fresh = _est(pb, str(tmp_path), fresh_state, ALL)
    ev2 = fresh.evaluate(lambda: iter(eval_batches))
    for k, v in ev.items():
        if '_at_n_' in k:
            assert ev2[k] == v, k
    torch.cuda.synchronize()


def test_data_parallel_raises():
    from types import SimpleNamespace
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.hparams import ModeKeys
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    model = SimpleNamespace(engine=SimpleNamespace(world=2))
    with pytest.raises(NotImplementedError):
        ItemsStateUpdaterHook(ModeKeys.EVAL, model, 5, ClickedItemsState(1.0, 10, 10, 10), eval_benchmark_classifiers=ALL)
