"""The per-session evaluation logs on the H100 (csrc/session_logs.cu nar_eval_session_logs_pack, session_logs.SessionLogs)
against the oracle (oracle/session_logs_ref.py): the kernel at tiny and G1 shapes bit for bit - rounded probabilities on
ties, below 5e-8, denormal, 0 and 1 -, each log alone and both, sessions without queries, a label-0 hole, out-of-range
ids, run-to-run bit identity; Estimator.evaluate end to end with all seven baselines and both metric switches; and
nar_trainer.run_train_eval_loop on TFRecord hour files.  The parameter checks need no GPU."""
import itertools
import json

import numpy as np
import pytest

from oracle.baselines_ref import SUFFIXES
from oracle.session_logs_ref import session_logs_ref

gpu = pytest.mark.gpu
KNN = ('v-sknn', 'sknn')
ALL7 = [{'recommender': s, 'params': {}} for s in SUFFIXES + KNN]


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _special_probs():
    ties = [np.float32((n + 0.5) / 1e7) for n in list(range(64)) + [12345, 99999, 250000, 1048574]]
    ties = [x for x in ties if (np.float32(x * np.float32(1e7)) % 1) == 0.5]
    assert len(ties) > 30
    return np.array(ties + [0.0, 1.0, 3e-8, 4.9999999e-8, 5.0000001e-8, 1e-30, 1e-40, 1.4e-45, 0.99999994, 0.33333334],
                    dtype=np.float32)


def _batch(rs, V, B, T, K, mean_len, holes=0.05, first_sid=1500000000):
    """Sessions of lengths 0 .. T (one of each end), labels [B, T] with holes (0 inside a session), the compacted rows as
    dp.shard_sessions makes them, eval negatives [B, T, K] (zero-padded in places), ranked candidates [L, 1 + K] = a
    permutation of label + negatives, probabilities with the rounding's hard cases mixed in, and float32 popularity over
    four decades with a fifth of the articles at a floor."""
    lens = np.minimum(rs.geometric(1.0 / mean_len, size=B) - 1, T)
    lens[rs.randint(0, B // 2)] = T
    lens[B // 2 + rs.randint(0, B - B // 2)] = 0
    valid = np.arange(T)[None, :] < lens[:, None]
    labels = np.where(valid, rs.randint(1, V, size=(B, T)), 0).astype(np.int64)
    labels[valid & (rs.rand(B, T) < holes)] = 0
    sess_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pos_idx = (np.arange(B)[:, None] * T + np.arange(T)[None, :])[valid].astype(np.int32)
    L = pos_idx.size
    neg = rs.randint(1, V, size=(B, T, K)).astype(np.int64)
    neg[rs.rand(B, T) < 0.2, K // 2:] = 0
    neg[~valid] = 0
    cand = np.concatenate([labels.reshape(-1)[pos_idx][:, None], neg.reshape(B * T, K)[pos_idx]], axis=1)
    order = np.argsort(rs.rand(L, 1 + K), axis=1)
    ids = np.take_along_axis(cand, order, axis=1)
    probs = -np.sort(-rs.dirichlet(np.ones(1 + K), size=L).astype(np.float32), axis=1)
    special = _special_probs()
    m = rs.rand(L, 1 + K) < 0.3
    probs[m] = rs.choice(special, size=int(m.sum()))
    pop = (rs.rand(V) * 10.0 ** rs.uniform(-4, 0, size=V)).astype(np.float32)
    pop[rs.rand(V) < 0.2] = np.float32(1.0 / 500)
    sids = (first_sid + np.arange(B)).astype(np.int64)
    sids[0] = 15436781234567890
    return dict(lens=lens, labels=labels, sess_off=sess_off, pos_idx=pos_idx, L=L, neg=neg, cand=cand, ids=ids,
                probs=np.ascontiguousarray(probs), pop=pop, sids=sids)


def _add(sl, b, V):
    sl.add(b['sids'], _dev(b['labels']), _dev(b['pos_idx'] if b['L'] else np.zeros(1, np.int32)), _dev(b['sess_off']), b['L'],
           negatives=_dev(b['neg']), pred_ids=_dev(b['ids']) if b['L'] else None,
           pred_probs=_dev(b['probs']) if b['L'] else None, cand=_dev(b['cand']) if b['L'] else None,
           cand_stride=b['cand'].shape[1], pop=_dev(b['pop']))


def _run(batches, V, neg_on=True, rec_on=True):
    import torch
    from chameleon_recsys_b200.session_logs import SessionLogs
    neg_log, rec_log = ([] if neg_on else None), ([] if rec_on else None)
    sl = SessionLogs(V, torch.device('cuda', 0), neg_log, rec_log)
    sl.begin()
    for b in batches:
        _add(sl, b, V)
    sl.end()
    torch.cuda.synchronize()
    return neg_log, rec_log, sl


def _want(batches, neg_on=True, rec_on=True):
    neg_log, rec_log = [], []
    for b in batches:
        n, r = session_logs_ref(b['sids'], b['labels'], b['neg'] if neg_on else None, b['ids'] if rec_on else None,
                                b['probs'], b['pop'], pos_idx=b['pos_idx'])
        neg_log += n or []
        rec_log += r or []
    return (neg_log if neg_on else None), (rec_log if rec_on else None)


def _float_bits(log, key):
    return [np.asarray(row, dtype=np.float64).astype(np.float32).view(np.uint32).tolist() for e in log for row in e[key]]


SHAPES = {'tiny': dict(V=60, B=8, T=6, K=7, mean_len=3.0), 'odd_k': dict(V=300, B=33, T=5, K=4, mean_len=2.5),
          'g1': dict(V=46034, B=256, T=19, K=50, mean_len=2.9)}


@gpu
@pytest.mark.parametrize('shape', sorted(SHAPES))
@pytest.mark.parametrize('neg_on,rec_on', [(True, True), (True, False), (False, True)])
def test_kernel_matches_oracle(shape, neg_on, rec_on):
    cfg = SHAPES[shape]
    rs = np.random.RandomState(sum(map(ord, shape)))
    batches = [_batch(rs, **cfg, first_sid=1500000000 + 1000 * i) for i in range(3)]
    if shape == 'g1':
        assert 350 < sum(int(np.count_nonzero(b['labels'])) for b in batches) / 3 < 650
    assert any(((b['labels'] == 0) & (np.arange(cfg['T'])[None, :] < b['lens'][:, None])).any() for b in batches)   # holes
    neg_log, rec_log, _ = _run(batches, cfg['V'], neg_on, rec_on)
    want_neg, want_rec = _want(batches, neg_on, rec_on)
    assert neg_log == want_neg
    assert rec_log == want_rec
    if rec_on:
        for key in ('predicted_item_probs', 'predicted_item_norm_pop'):
            assert _float_bits(rec_log, key) == _float_bits(want_rec, key)
        assert len(rec_log) == 3 * cfg['B'] and any(not e['next_click_labels'] for e in rec_log)
        assert list(rec_log[0]) == ['session_id', 'next_click_labels', 'predicted_item_ids', 'predicted_item_probs',
                                    'predicted_item_norm_pop']
        assert rec_log[0]['session_id'] == '15436781234567890'
        json.dumps(rec_log[:4])
    if neg_on:
        assert len(neg_log) == 3 * cfg['B'] and list(neg_log[0]) == ['session_id', 'negative_items']


@gpu
def test_batch_without_a_valid_position_and_all_holes():
    rs = np.random.RandomState(3)
    b0 = _batch(rs, 60, 8, 6, 7, 3.0)
    empty = _batch(rs, 60, 8, 6, 7, 3.0)
    empty.update(lens=np.zeros(8, np.int64), labels=np.zeros((8, 6), np.int64), sess_off=np.zeros(9, np.int32),
                 pos_idx=np.zeros(0, np.int32), L=0, ids=np.zeros((0, 8), np.int64), probs=np.zeros((0, 8), np.float32),
                 cand=np.zeros((0, 8), np.int64))
    holes = _batch(rs, 60, 8, 6, 7, 3.0)
    holes['labels'][:] = 0                                    # valid positions, no query at all: Q = 0 < L
    holes['cand'][:, 0] = 0
    batches = [b0, empty, holes, b0]
    neg_log, rec_log, _ = _run(batches, 60)
    assert (neg_log, rec_log) == _want(batches)
    assert all(e['negative_items'] == [] for e in neg_log[8:24]) and rec_log[8]['predicted_item_probs'] == []


@gpu
def test_two_runs_are_bit_identical():
    import torch
    cfg = SHAPES['g1']
    rs = np.random.RandomState(11)
    batches = [_batch(rs, **cfg) for _ in range(2)]
    a_neg, a_rec, a = _run(batches, cfg['V'])
    b_neg, b_rec, b = _run(batches, cfg['V'])
    assert a_neg == b_neg and a_rec == b_rec
    assert a.d2h_bytes == b.d2h_bytes > 0
    assert torch.equal(a.packed[:a.d2h_bytes], b.packed[:b.d2h_bytes])


@gpu
def test_copy_is_sized_from_the_valid_positions():
    cfg = SHAPES['g1']
    b = _batch(np.random.RandomState(2), **cfg, holes=0.0)
    _, _, sl = _run([b], cfg['V'])
    B, K, L = cfg['B'], cfg['K'], b['L']
    assert L == int(np.count_nonzero(b['labels']))
    payload = L * (K * 8 + 8 + (K + 1) * (8 + 4 + 4))             # what ends up in the two files
    assert payload < sl.d2h_bytes <= payload + 16 + 4 * B + 16 + L * (8 + 4 + 4) + 32    # + header, one pad column


@gpu
@pytest.mark.parametrize('bad', [-1, 60, 2 ** 40])
def test_out_of_range_id_raises(bad):
    rs = np.random.RandomState(4)
    b = _batch(rs, 60, 8, 6, 7, 3.0, holes=0.0)
    b['ids'][b['L'] // 2, 3] = bad
    with pytest.raises(ValueError, match='outside'):
        _run([b], 60)
    neg_log, _, _ = _run([b], 60, rec_on=False)                   # the negatives log gathers nothing
    assert neg_log == _want([b], rec_on=False)[0]


def test_parameter_checks():
    from types import SimpleNamespace
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.hparams import ModeKeys
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    state = ClickedItemsState(1.0, 100, 50, 60)
    two = SimpleNamespace(engine=SimpleNamespace(world=2))
    for kw in ({'sessions_negative_items_log': []}, {'sessions_chameleon_recommendations_log': []}):
        with pytest.raises(NotImplementedError):
            ItemsStateUpdaterHook(ModeKeys.EVAL, two, 3, state, **kw)
        hook = ItemsStateUpdaterHook(ModeKeys.TRAIN, two, 3, state, **kw)           # EVAL only
        assert not hook.session_logs_on
    hook = ItemsStateUpdaterHook(ModeKeys.EVAL, two, 3, state)
    assert not hook.session_logs_on and hook.session_logs is None


def _problem():
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 2)
    return pb


def _est(pb, d, state, **extra):
    from chameleon_recsys_b200.estimator import build_estimator
    hp = pb.hp.copy(eval_benchmarks=tuple(ALL7), eval_extended_metrics=True, eval_metrics_by_session_position=True)
    return build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                           pb.session_features_config, hp, state, device=0, **extra)


@gpu
def test_estimator_matches_oracle(monkeypatch):
    """Train, then evaluate with both logs, all seven baselines and both metric switches on: the two lists equal the
    oracle applied to the arrays the same evaluate exposes to its hook - ranked ids, probabilities, negatives and the
    staged float32 popularity the batch was fed with."""
    import torch
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    neg_log, rec_log = [], []
    est = _est(pb, None, pb.clicked_items_state, sessions_negative_items_log=neg_log,
               sessions_chameleon_recommendations_log=rec_log)
    est.train(lambda: iter(train_batches))
    seen = []
    orig_after = ItemsStateUpdaterHook.after_run

    def spy_after(self, run_context, run_values):
        st = run_values['stage']
        cp = (lambda x: x.cpu().numpy().copy())
        seen.append(dict(ids=cp(run_values['predicted_item_ids']), probs=cp(run_values['predicted_item_probs']),
                         neg=cp(run_values['eval_batch_negative_items']), pop=cp(st['t']['pop_norm']),
                         pos=cp(st['t']['pos_idx'])[:st['L']], sids=np.asarray(run_values['session_ids']).copy(),
                         fed=self.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32).copy()))
        return orig_after(self, run_context, run_values)
    monkeypatch.setattr(ItemsStateUpdaterHook, 'after_run', spy_after)
    ev = est.evaluate(lambda: iter(eval_batches))
    torch.cuda.synchronize()
    hook = est._eval_spec.evaluation_hooks[0]
    assert hook.session_logs is not None and hook.session_logs.pending is None
    want_neg, want_rec = [], []
    for (f, l), s in zip(eval_batches, seen):
        assert np.array_equal(s['pop'], s['fed']) and np.array_equal(s['sids'], f['session_id'])
        n, r = session_logs_ref(f['session_id'], l['label_next_item'], s['neg'], s['ids'], s['probs'], s['pop'],
                                pos_idx=s['pos'])
        want_neg += n
        want_rec += r
    assert neg_log == want_neg and rec_log == want_rec
    queries = sum(int(np.count_nonzero(l['label_next_item'])) for _, l in eval_batches)
    assert sum(len(e['next_click_labels']) for e in rec_log) == queries > 0
    assert len(rec_log) == sum(len(f['session_id']) for f, _ in eval_batches)
    # the cross-file invariant: each query's ranked ids are a permutation of its label + its negatives
    for n, r in zip(neg_log, rec_log):
        assert n['session_id'] == r['session_id']
        for lab, negs, ids in zip(r['next_click_labels'], n['negative_items'], r['predicted_item_ids']):
            assert sorted(ids) == sorted([lab] + negs)
    # a second evaluate appends again (the lists are the caller's to empty)
    est.evaluate(lambda: iter(eval_batches[:1]))
    assert len(neg_log) == len(want_neg) + len(eval_batches[0][0]['session_id'])
    assert 'hitrate_at_n_by_pos_01' in ev and 'ndcg_at_n' in ev


@gpu
def test_logs_change_no_key_of_evaluate(tmp_path):
    """From one checkpoint: every key evaluate returns has the same value with the logs on - bit for bit, except the loss
    and the model's MRR, which the existing evaluation kernels sum with float atomics and which are held to the rounding
    bound of their summation order (DESIGN.md section 10).  With the logs off the hook owns no SessionLogs object."""
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    d = str(tmp_path)
    _est(pb, d, pb.clicked_items_state).train(lambda: iter(train_batches))
    saved = ckpt.load(ckpt.latest_checkpoint(d))
    st = pb.clicked_items_state
    runs, hooks = {}, {}
    for name in ('off', 'on'):
        fresh = ClickedItemsState(st.recent_clicks_buffer_hours, st.recent_clicks_buffer_max_size,
                                  st.recent_clicks_for_normalization, st.num_items)
        for f in ckpt.STATE_FIELDS:
            setattr(fresh, f, np.array(saved['state'][f]))
        extra = {'sessions_negative_items_log': [], 'sessions_chameleon_recommendations_log': []} if name == 'on' else {}
        est = _est(pb, d, fresh, **extra)
        runs[name] = est.evaluate(lambda: iter(eval_batches))
        hooks[name] = est._eval_spec.evaluation_hooks[0]
    off, on = runs['off'], runs['on']
    assert hooks['off'].session_logs is None and not hooks['off'].session_logs_on
    assert hooks['on'].session_logs is not None and len(hooks['on'].sessions_negative_items_log) > 0
    assert list(on) == list(off)
    positions = max(np.asarray(f['item_clicked']).size for f, _ in eval_batches)
    queries = sum(int(np.count_nonzero(l['label_next_item'])) for _, l in eval_batches)
    tol = {'loss': 2 * (positions - 1) * 2.0 ** -24, 'mrr_at_n': 2 * queries * 2.0 ** -53}
    for k, v in off.items():
        if k in tol:
            assert abs(on[k] - v) <= tol[k] * abs(v), (k, on[k], v)
        else:
            assert on[k] == v, (k, on[k], v)
    torch.cuda.synchronize()


@gpu
def test_train_eval_loop_on_tfrecord_hour_files(tmp_path):
    from chameleon_recsys_b200 import nar_trainer, tfrecords
    pb = _problem()
    stream = iter(pb.stream)
    per_file = 3 * pb.hp.batch_size // 2                       # one full batch and a half one per hour file
    files = []
    for h in range(5):
        path = str(tmp_path / ('sessions_hour_%03d.tfrecord.gz' % h))
        tfrecords.write_sequence_examples(path, itertools.islice(stream, per_file), pb.session_features_config)
        files.append(path)
    out = tmp_path / 'out'
    out.mkdir()
    est = _est(pb, None, pb.clicked_items_state)
    log = nar_trainer.run_train_eval_loop(est, files, pb.session_features_config, pb.hp, train_files_from=0,
                                          train_files_up_to=4, training_hours_for_each_eval=2, save_results_each_n_evals=1,
                                          model_output_dir=str(out), save_eval_sessions_negative_samples=True,
                                          save_eval_sessions_recommendations=True)
    assert len(log) == 2 and all('hitrate_at_n' in m and 'ndcg_at_n_pop_recent' in m for m in log)
    assert sorted(p.name for p in out.iterdir()) == ['eval_chameleon_recommendations_log.json', 'eval_sessions_negative_samples.json',
                                                    'eval_stats_benchmarks.csv']
    rec = [json.loads(l) for l in (out / 'eval_chameleon_recommendations_log.json').read_text().splitlines()]
    neg = [json.loads(l) for l in (out / 'eval_sessions_negative_samples.json').read_text().splitlines()]
    assert len(rec) == len(neg) == 2 * per_file                  # every session of both evaluated hours
    assert [r['eval_hour_id'] for r in rec] == [0] * per_file + [1] * per_file
    n_queries = 0
    for n, r in zip(neg, rec):
        assert n['session_id'] == r['session_id']
        assert len(n['negative_items']) == len(r['next_click_labels']) == len(r['predicted_item_ids'])
        for lab, negs, ids, probs, pops in zip(r['next_click_labels'], n['negative_items'], r['predicted_item_ids'],
                                               r['predicted_item_probs'], r['predicted_item_norm_pop']):
            assert sorted(ids) == sorted([lab] + negs) and len(probs) == len(pops) == len(ids)
            assert probs == sorted(probs, reverse=True)
            n_queries += 1
    assert n_queries > 0
    rows = (out / 'eval_stats_benchmarks.csv').read_text().splitlines()
    assert len(rows) == 3 and rows[0].startswith('index,loss,') and rows[0].endswith(',hour,day')
    assert rows[1].endswith(',2,0') and rows[2].endswith(',4,0')
    assert est.params['sessions_negative_items_log'] == []
