"""Hit rate by session position on the H100 (csrc/eval_metrics.cu nar_eval_by_position, eval_metrics.ByPosition) against
the oracle (oracle/by_position_ref.py): the kernel at tiny and G1 shapes (counts exact, the float32 popularity sums
bit for bit), run-to-run bit identity, out-of-range ids, and Estimator.evaluate end to end with the model and all seven
baselines - its keys against the oracle, its per-position counts against the existing hit-rate counts, and every other
key unchanged by the switch.  The parameter checks need no GPU."""
import numpy as np
import pytest

from oracle.baselines_ref import SUFFIXES
from oracle.by_position_ref import ByPositionRef

gpu = pytest.mark.gpu
KNN = ('v-sknn', 'sknn')
ALL7 = [{'recommender': s, 'params': {}} for s in SUFFIXES + KNN]
PREFIXES = ('hitrate_at_n_by_pos_', 'clicks_at_pos_', 'avg_norm_pop_by_pos_')


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pop(rs, V):
    """float32 over four decades, so that the order of a float32 sum changes its rounding"""
    pop = (rs.rand(V) * 10.0 ** rs.uniform(-4, 0, size=V)).astype(np.float32)
    pop[rs.rand(V) < 0.2] = np.float32(1.0 / 500)
    return pop


def _batch(rs, V, B, T, K, n, bl_rows, mean_len):
    """One batch: sessions of lengths 0 .. T (one of length T), labels [B*T] with a few holes (0 inside a session); the
    model's compacted rows (pos_idx, sess_off as dp.shard_sessions makes them) with ranked candidate lists [L, 1+K]
    whose column 0 of the candidate ids is the label; baseline lists [bl_rows, B*T, n] (0-padded, label at any rank or
    absent; cells without a label hold out-of-range garbage, which must be ignored)."""
    lens = np.minimum(rs.geometric(1.0 / mean_len, size=B) - 1, T)
    lens[rs.randint(0, B)] = T
    valid = np.arange(T)[None, :] < lens[:, None]
    labels = np.where(valid, rs.randint(1, V, size=(B, T)), 0).astype(np.int64)
    labels[valid & (rs.rand(B, T) < 0.05)] = 0
    labels = labels.reshape(-1)
    sess_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pos_idx = (np.arange(B)[:, None] * T + np.arange(T)[None, :])[valid].astype(np.int32)
    model = rs.randint(1, V, size=(pos_idx.size, 1 + K)).astype(np.int64)
    model[rs.rand(*model.shape) < 0.05] = 0
    for i, p in enumerate(pos_idx):
        model[i, rs.randint(0, 1 + K)] = labels[p] if labels[p] else rs.randint(1, V)
    cand = np.zeros_like(model)
    cand[:, 0] = labels[pos_idx]
    bl = rs.choice([-7, V + 3], size=(bl_rows, B * T, n)).astype(np.int64)
    for r in range(bl_rows):
        for p in np.flatnonzero(labels):
            k = rs.randint(0, n + 1)
            row = [int(x) for x in rs.randint(1, V, size=k)] + [0] * (n - k)
            if k and rs.rand() < 0.6:
                row[rs.randint(0, k)] = labels[p]
            bl[r, p] = row
    return labels, pos_idx, sess_off, model, cand, bl


def _run(seed, V, B, T, K, n, bl_rows, mean_len, batches, bl_mask):
    import torch
    from chameleon_recsys_b200.eval_metrics import ByPosition
    rs = np.random.RandomState(seed)
    pop = _pop(rs, V)
    pop_d = _dev(pop)
    bp = ByPosition(1 + bl_rows, V, n, 'cuda')
    ref = ByPositionRef(1 + bl_rows, n)
    bp.begin()
    ref.begin()
    for _ in range(batches):
        labels, pos_idx, sess_off, model, cand, bl = _batch(rs, V, B, T, K, n, bl_rows, mean_len)
        bp.add(_dev(model), _dev(cand).view(-1), T, pos_idx=_dev(pos_idx), sess_off=_dev(sess_off), pop=pop_d,
               label_stride=1 + K)
        bp.add(_dev(bl), _dev(labels), T, row0=1, row_mask=bl_mask)
        ref.add(0, model, cand[:, 0], T, pos=pos_idx, pop=pop)
        for r in range(bl_rows):
            if (bl_mask >> r) & 1:
                ref.add(1 + r, bl[r], labels, T)
    torch.cuda.synchronize()
    return bp, ref


def _compare(bp, ref, T):
    names = [(r, '' if r == 0 else 'bl%d' % r) for r in range(bp.rows)]
    got = bp.results(names)
    want = {}
    for r, s in names:
        want.update(ref.results(r, s))
    assert got == want
    counts = bp.counts.cpu().numpy()
    for r in range(bp.rows):
        assert all(counts[0, r, p - 1] == ref.hits[r][p] and counts[1, r, p - 1] == ref.total[r][p] for p in range(1, T + 1))
        assert not counts[:, r, T:].any()
    sums = bp.norm_pop.cpu().numpy()
    assert np.array_equal(sums[:T].view(np.int32), np.array([ref.norm_pop[0][p] for p in range(1, T + 1)],
                                                            dtype=np.float32).view(np.int32))
    return got


@gpu
def test_kernel_matches_oracle_tiny():
    """top_n 3 out of 1 + K = 8 candidates; baseline row 2 masked out (its garbage ids must be ignored)."""
    bp, ref = _run(1, 60, 8, 6, 7, 3, 3, 3.0, 4, bl_mask=0b101)
    got = _compare(bp, ref, 6)
    assert not any(k.startswith('hitrate_at_n_by_pos_bl2_') for k in got)
    assert 'hitrate_at_n_by_pos_06' in got and 'avg_norm_pop_by_pos_06' in got


@gpu
def test_kernel_matches_oracle_top_n_one():
    bp, ref = _run(2, 60, 8, 6, 5, 1, 2, 3.0, 3, bl_mask=0b11)
    _compare(bp, ref, 6)


@gpu
def test_kernel_matches_oracle_g1():
    """G1 shapes: V 46 034, B 256 x T 20 with about 500 queries per batch, K 50, top_n 10, the model and 7 baseline rows,
    3 batches (the float32 sums carry across them)."""
    bp, ref = _run(3, 46034, 256, 20, 50, 10, 7, 3.0, 3, bl_mask=0x7f)
    assert 1000 < sum(ref.total[0].values()) < 2500
    _compare(bp, ref, 20)


@gpu
def test_runs_are_bit_identical():
    import torch
    runs = [_run(4, 46034, 256, 20, 50, 10, 7, 3.0, 3, bl_mask=0x7f)[0] for _ in range(2)]
    assert torch.equal(runs[0].counts, runs[1].counts)
    assert torch.equal(runs[0].norm_pop.view(torch.int32), runs[1].norm_pop.view(torch.int32))


@gpu
def test_out_of_range_ids_raise():
    from chameleon_recsys_b200.eval_metrics import ByPosition
    for ids, labels in (([[3, 25]], [3]), ([[3, 4]], [-2])):
        bp = ByPosition(1, 20, 2, 'cuda')
        bp.begin()
        bp.add(_dev(np.array(ids, dtype=np.int64)), _dev(np.array(labels, dtype=np.int64)), 1)
        with pytest.raises(ValueError):
            bp.results([(0, '')])


def test_parameters_are_checked():
    from types import SimpleNamespace
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.hparams import ModeKeys
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    state = ClickedItemsState(1.0, 10, 10, 10)
    model = SimpleNamespace(engine=SimpleNamespace(world=1))
    for top_n in (0, -1, 65):
        with pytest.raises(ValueError):
            ItemsStateUpdaterHook(ModeKeys.EVAL, model, top_n, state, eval_metrics_by_session_position=True)
    ItemsStateUpdaterHook(ModeKeys.EVAL, model, 1, state, eval_metrics_by_session_position=True)
    ItemsStateUpdaterHook(ModeKeys.EVAL, model, 0, state)                                     # switch off
    with pytest.raises(NotImplementedError):
        ItemsStateUpdaterHook(ModeKeys.EVAL, SimpleNamespace(engine=SimpleNamespace(world=2)), 3, state,
                              eval_metrics_by_session_position=True)


def test_empty_evaluate_adds_no_keys():
    from chameleon_recsys_b200.estimator import Estimator
    est = Estimator(None, {'eval_metrics_by_session_position': True, 'eval_benchmarks': ['cb', 'v-sknn']})
    ev = est.evaluate(lambda: iter(()))
    assert not [k for k in ev if k.startswith(PREFIXES)]


def _problem():
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 2)
    return pb


def _est(pb, d, state, on, top_n=None):
    from chameleon_recsys_b200.estimator import build_estimator
    hp = pb.hp.copy(eval_benchmarks=tuple(ALL7), eval_metrics_by_session_position=on)
    if top_n is not None:
        hp.eval_metrics_top_n = top_n
    return build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                           pb.session_features_config, hp, state, device=0)


@gpu
def test_bad_top_n_raises_in_evaluate():
    pb = _problem()
    est = _est(pb, None, pb.clicked_items_state, True, top_n=65)
    est.train(pb.input_fn, steps=1)
    with pytest.raises(ValueError, match='eval_metrics_by_session_position'):
        est.evaluate(pb.input_fn, steps=1)


@gpu
def test_estimator_matches_oracle(monkeypatch):
    """Train with all seven baselines, evaluate with the switch on: the by-position keys equal the oracle applied to the
    model's ranked candidates (with the popularity the batch was fed with) and to the baselines' top-n lists.  Summed
    over positions, each recommender's hits and queries are exactly the counts behind its hitrate_at_n."""
    import torch
    from chameleon_recsys_b200.baselines import BaselineTables
    from chameleon_recsys_b200.eval_metrics import ByPosition
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    est = _est(pb, None, pb.clicked_items_state, True)
    est.train(lambda: iter(train_batches))
    fed, calls = [], []
    orig_after, orig_add = ItemsStateUpdaterHook.after_run, ByPosition.add

    def spy_after(self, run_context, run_values):
        fed.append(self.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32).copy())
        return orig_after(self, run_context, run_values)

    def spy_add(self, ids, labels, T, pos_idx=None, sess_off=None, pop=None, row0=0, row_mask=None, label_stride=1):
        cp = (lambda x: None if x is None else x.cpu().numpy().copy())
        calls.append(dict(ids=cp(ids), labels=cp(labels)[::label_stride], T=T, pos=cp(pos_idx), pop=cp(pop), row0=row0,
                          sess_off=cp(sess_off)))
        return orig_add(self, ids, labels, T, pos_idx=pos_idx, sess_off=sess_off, pop=pop, row0=row0,
                        row_mask=row_mask, label_stride=label_stride)
    monkeypatch.setattr(ItemsStateUpdaterHook, 'after_run', spy_after)
    monkeypatch.setattr(ByPosition, 'add', spy_add)
    ev = est.evaluate(lambda: iter(eval_batches))
    torch.cuda.synchronize()
    hook = est._eval_spec.evaluation_hooks[0]

    n = pb.hp.eval_metrics_top_n
    names = ('',) + SUFFIXES + KNN
    rows = {s: (0 if not s else 1 + BaselineTables.row(s)) for s in names}
    ref = ByPositionRef(1 + hook.baselines.n_rows, n)
    ref.begin()
    assert len(calls) == 2 * len(eval_batches)
    for (f, l), pop, model, bls in zip(eval_batches, fed, calls[0::2], calls[1::2]):
        ln = np.asarray(l['label_next_item']).reshape(-1)
        B, T = np.asarray(f['item_clicked']).shape
        assert model['row0'] == 0 and bls['row0'] == 1 and model['T'] == bls['T'] == T
        L = model['ids'].shape[0]
        assert np.array_equal(model['labels'], ln[model['pos'][:L]]) and np.array_equal(bls['labels'], ln)
        assert np.array_equal(model['pop'], pop)                          # the popularity the batch was fed with
        assert np.array_equal(np.diff(model['sess_off']), np.bincount(model['pos'][:L] // T, minlength=B))
        ref.add(0, model['ids'], model['labels'], T, pos=model['pos'][:L], pop=pop)
        for s in SUFFIXES + KNN:
            ref.add(rows[s], bls['ids'][rows[s] - 1], ln, T)
    want = {}
    for s in names:
        want.update(ref.results(rows[s], s))
    got = {k: v for k, v in ev.items() if k.startswith(PREFIXES)}
    assert got == want
    assert 'hitrate_at_n_by_pos_01' in got and 'hitrate_at_n_by_pos_v-sknn_01' in got

    # the invariant: per recommender, the by-position counts add up to the hit-rate counts
    counts = hook.by_position.counts.cpu().numpy()
    queries = sum(int(np.count_nonzero(l['label_next_item'])) for _, l in eval_batches)
    hits, total = int(counts[0, 0].sum()), int(counts[1, 0].sum())
    assert total == queries and hits / float(total) == ev['hitrate_at_n']
    bench = hook.bench_metrics.cpu().numpy()
    for s in SUFFIXES + KNN:
        r = BaselineTables.row(s)
        assert counts[1, 1 + r].sum() == bench[r, 2] == queries, s
        assert counts[0, 1 + r].sum() == bench[r, 0], s


@gpu
def test_switch_changes_no_other_key(tmp_path):
    """From one checkpoint: every key evaluate returns with the switch off has the same value with it on - bit for bit,
    except the loss and the model's MRR, which the existing evaluation kernels sum with float atomics (their last bits
    differ between any two runs, the switch on or off) and which are held to the rounding bound of their summation order
    (as in test_eval_metrics_gpu.test_switch_changes_no_other_key)."""
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    d = str(tmp_path)
    _est(pb, d, pb.clicked_items_state, False).train(lambda: iter(train_batches))
    saved = ckpt.load(ckpt.latest_checkpoint(d))
    st = pb.clicked_items_state
    runs = {}
    for name in ('off', 'on'):
        fresh = ClickedItemsState(st.recent_clicks_buffer_hours, st.recent_clicks_buffer_max_size,
                                  st.recent_clicks_for_normalization, st.num_items)
        for f in ckpt.STATE_FIELDS:
            setattr(fresh, f, np.array(saved['state'][f]))
        runs[name] = _est(pb, d, fresh, name == 'on').evaluate(lambda: iter(eval_batches))
    off, on = runs['off'], runs['on']
    new = set(on) - set(off)
    assert new and all(k.startswith(PREFIXES) for k in new) and not [k for k in off if k.startswith(PREFIXES)]
    positions = max(np.asarray(f['item_clicked']).size for f, _ in eval_batches)
    queries = sum(int(np.count_nonzero(l['label_next_item'])) for _, l in eval_batches)
    tol = {'loss': 2 * (positions - 1) * 2.0 ** -24, 'mrr_at_n': 2 * queries * 2.0 ** -53}
    for k, v in off.items():
        if k in tol:
            assert abs(on[k] - v) <= tol[k] * abs(v), (k, on[k], v)
        else:
            assert on[k] == v, (k, on[k], v)
    torch.cuda.synchronize()
