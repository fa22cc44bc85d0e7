"""NDCG, item coverage, ESI-R / ESI-RR and EILD-R / EILD-RR on the H100 (csrc/eval_metrics.cu,
chameleon_recsys_b200/eval_metrics.py) against the oracle (oracle/eval_metrics_ref.py): the kernels at tiny and G1
shapes with every edge case of the reference fixture, run-to-run bit identity, and Estimator.evaluate end to end with the
model and all seven baselines.  The parameter checks need no GPU."""
import numpy as np
import pytest

from oracle.baselines_ref import SUFFIXES, BaselinesRef
from oracle.eval_metrics_ref import VALUES, EvalMetricsRef
from oracle.sknn_ref import SknnRef

gpu = pytest.mark.gpu
KNN = ('v-sknn', 'sknn')
ALL7 = [{'recommender': s, 'params': {}} for s in SUFFIXES + KNN]
NORM = 500


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _tables(rs, V, dim):
    acr = rs.randn(V, dim).astype(np.float32)
    acr[0] = 0.0                                                    # norm 0: cosine 0, distance 0.5
    acr[6] = acr[5]                                                 # identical rows: distance 0
    pop = (rs.randint(1, 40, size=V) / NORM).astype(np.float32)
    pop[rs.rand(V) < 0.4] = np.float32(1.0 / NORM)                  # the normalisation floor
    buf = np.zeros(400, dtype=np.int64)
    buf[:300] = rs.randint(1, V, size=300)                          # padding at the end
    return acr, pop, buf


def _batch(rs, V, B, T, K, n, bl_rows, valid):
    """One batch: labels [B*T] (about `valid` of them nonzero), the model's ranked candidate lists [Q, 1+K] (label at any
    rank, repeated ids, zero padding, rows 5 / 6 together), baseline lists [bl_rows, B*T, n] (0-padded, label at any rank
    or absent; positions without a label hold out-of-range garbage, which must be ignored) and clicks [B*T]."""
    labels = rs.randint(1, V, size=B * T).astype(np.int64)
    labels[rs.rand(B * T) >= valid] = 0
    q = np.flatnonzero(labels)
    model = np.zeros((q.size, 1 + K), dtype=np.int64)
    for i, lab in enumerate(labels[q]):
        row = list(rs.randint(1, V, size=K))
        if rs.rand() < 0.3:
            s = rs.randint(K // 2, K)
            row[s:] = [0] * (K - s)
        if rs.rand() < 0.15:
            row[rs.randint(0, K)] = lab
        if rs.rand() < 0.15:
            row[rs.randint(0, K)], row[rs.randint(0, K)] = 5, 6
        row.insert(rs.randint(0, K + 1), lab)
        model[i] = row
    cand = np.zeros_like(model)
    cand[:, 0] = labels[q]
    bl = rs.choice([-7, V + 3], size=(bl_rows, B * T, n)).astype(np.int64)
    for r in range(bl_rows):
        for p in q:
            k = rs.randint(0, n + 1)
            row = [int(x) for x in rs.randint(1, V, size=k)] + [0] * (n - k)
            if k and rs.rand() < 0.7:
                row[rs.randint(0, k)] = labels[p]
            bl[r, p] = row
    clicks = np.where(rs.rand(B * T) < 0.7, rs.randint(1, V, size=B * T), 0).astype(np.int64)
    return labels, model, cand, bl, clicks


def _run(seed, V, dim, B, T, K, n, bl_rows, valid, batches, bl_mask):
    import torch
    from chameleon_recsys_b200.eval_metrics import EvalMetrics
    rs = np.random.RandomState(seed)
    acr, pop, buf = _tables(rs, V, dim)
    acr_d = _dev(np.pad(acr, ((0, 0), (0, 6))))                     # leading dimension > dim
    em = EvalMetrics(1 + bl_rows, V, acr_d, dim, n, 0.1)
    ref = EvalMetricsRef(1 + bl_rows, n, acr, 0.1)
    em.begin(buf)
    ref.begin(buf)
    pop_d, pop64 = _dev(pop), pop.astype(np.float64)
    for _ in range(batches):
        labels, model, cand, bl, clicks = _batch(rs, V, B, T, K, n, bl_rows, valid)
        em.add_lists(_dev(model), _dev(cand).view(-1), pop_d, label_stride=1 + K)
        em.add_lists(_dev(bl), _dev(labels), pop_d, row0=1, row_mask=bl_mask)
        em.add_clicks(_dev(clicks), _dev(labels))
        ref.add_lists(0, model, cand[:, 0], pop64)
        for r in range(bl_rows):
            if (bl_mask >> r) & 1:
                ref.add_lists(1 + r, bl[r], labels, pop64)
        ref.add_clicks(clicks, labels)
    got = em.results()
    torch.cuda.synchronize()
    return got, ref, em


def _compare(got, ref):
    from chameleon_recsys_b200.eval_metrics import COVERAGE_KEY, KEYS
    for r, g in enumerate(got):
        w = ref.results(r)
        assert g['queries'] == ref.count[r] and g['recommended'] == w['recommended'] and g['clicked'] == w['clicked'], r
        if not ref.count[r]:
            assert all(np.isnan(g[k]) for k in KEYS) and g[COVERAGE_KEY] == 0.0
            continue
        for k, v in zip(KEYS, VALUES):
            assert abs(g[k] * g['queries'] - ref.sums[r, VALUES.index(v)]) <= 1e-9 * abs(ref.sums[r, VALUES.index(v)]), \
                (r, k, g[k], w[v])
        assert g[COVERAGE_KEY] == w['coverage'], r


@gpu
def test_kernels_match_oracle_tiny():
    """top_n 3 out of 1 + K = 8 candidates; baseline row 2 masked out (its garbage ids must be ignored)."""
    got, ref, _ = _run(1, 60, 12, 8, 6, 7, 3, 3, 0.7, 4, bl_mask=0b101)
    _compare(got, ref)
    assert got[2]['queries'] == 0 and got[2]['recommended'] == 0


@gpu
def test_kernels_match_oracle_top_n_beyond_list():
    """top_n 10 with 1 + K = 6: the model's lists are scored whole (m = 6)."""
    got, ref, _ = _run(2, 60, 12, 8, 6, 5, 10, 2, 0.7, 3, bl_mask=0b11)
    _compare(got, ref)


@gpu
def test_kernels_match_oracle_g1():
    """G1 shapes: V 46 034, ACR 250, B 256 x T 20 positions with about 480 queries, K 50, top_n 10, the model and 7
    baseline rows, 2 batches."""
    got, ref, _ = _run(3, 46034, 250, 256, 20, 50, 10, 7, 480 / 5120, 2, bl_mask=0x7f)
    assert 800 < got[0]['queries'] < 1200
    _compare(got, ref)


@gpu
def test_runs_are_bit_identical():
    import torch
    accs = []
    for _ in range(2):
        _, _, em = _run(4, 46034, 250, 256, 20, 50, 10, 7, 480 / 5120, 2, bl_mask=0x7f)
        accs.append(em.acc.clone())
    assert torch.equal(accs[0].view(torch.int64), accs[1].view(torch.int64))


@gpu
def test_out_of_range_ids_raise():
    from chameleon_recsys_b200.eval_metrics import EvalMetrics
    acr = _dev(np.ones((20, 4), dtype=np.float32))
    em = EvalMetrics(1, 20, acr, 4, 2, 0.1)
    em.begin(np.zeros(3, dtype=np.int64))
    em.add_lists(_dev(np.array([[3, 25]], dtype=np.int64)), _dev(np.array([3], dtype=np.int64)),
                 _dev(np.full(20, 0.5, dtype=np.float32)))
    with pytest.raises(ValueError):
        em.results()


def test_parameters_are_checked():
    from types import SimpleNamespace
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.hparams import ModeKeys, NARHParams
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    state = ClickedItemsState(1.0, 10, 10, 10)
    model = SimpleNamespace(engine=SimpleNamespace(world=1))
    for top_n, rel in ((1, 0.1), (3, 0.0), (3, -1.0), (3, None)):
        with pytest.raises(ValueError):
            ItemsStateUpdaterHook(ModeKeys.EVAL, model, top_n, state, eval_negative_sample_relevance=rel,
                                  eval_extended_metrics=True)
    ItemsStateUpdaterHook(ModeKeys.EVAL, model, 1, state, eval_negative_sample_relevance=0.1)        # switch off
    with pytest.raises(NotImplementedError):
        ItemsStateUpdaterHook(ModeKeys.EVAL, SimpleNamespace(engine=SimpleNamespace(world=2)), 3, state,
                              eval_negative_sample_relevance=0.1, eval_extended_metrics=True)
    args = ({}, {'article_id': {}}, {}, np.zeros((2, 2), np.float32))
    assert 'eval_extended_metrics' not in NARHParams().to_params(*args)
    assert NARHParams(eval_extended_metrics=True).to_params(*args)['eval_extended_metrics'] is True


def _problem():
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 2)
    return pb


def _est(pb, d, state, extended, top_n=None):
    from chameleon_recsys_b200.estimator import build_estimator
    hp = pb.hp.copy(eval_benchmarks=tuple(ALL7), eval_extended_metrics=extended)
    if top_n is not None:
        hp.eval_metrics_top_n = top_n
    return build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                           pb.session_features_config, hp, state, device=0)


@gpu
def test_top_n_one_raises_in_evaluate():
    pb = _problem()
    est = _est(pb, None, pb.clicked_items_state, True, top_n=1)
    est.train(pb.input_fn, steps=1)
    with pytest.raises(ValueError):
        est.evaluate(pb.input_fn, steps=1)


@gpu
def test_estimator_matches_oracle(monkeypatch):
    """Train with all seven baselines, evaluate with the switch on: the model's keys equal the oracle applied to its
    ranked candidates, each baseline's the oracle applied to its top-n lists, and those lists are the baselines oracles'
    (cb: where its fp64 cosines are not within 1e-6 of a tie)."""
    import torch
    from chameleon_recsys_b200.baselines import BaselineTables
    from chameleon_recsys_b200.eval_metrics import COVERAGE_KEY, KEYS, EvalMetrics
    from chameleon_recsys_b200.nar_model import ItemsStateUpdaterHook
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    est = _est(pb, None, pb.clicked_items_state, True)
    est.train(lambda: iter(train_batches))
    seen, lists = [], []
    orig_after, orig_add = ItemsStateUpdaterHook.after_run, EvalMetrics.add_lists

    def spy_after(self, run_context, run_values):
        st = run_values['stage']
        pred = run_values['predicted_item_ids']
        cand = self.model.engine.buffer(st, 'row_item').view(-1)[st['L']:].view(pred.shape)
        s = self.clicked_items_state
        seen.append((run_values['eval_batch_negative_items'].cpu().numpy().copy(), s.get_recent_clicks_buffer().copy(),
                     s.get_articles_pop().copy(), s.get_articles_recent_pop_norm().astype(np.float32).astype(np.float64),
                     pred.cpu().numpy().copy(), cand[:, 0].cpu().numpy().copy()))
        return orig_after(self, run_context, run_values)

    def spy_add(self, ids, labels, pop, row0=0, row_mask=None, label_stride=1):
        if row0 == 1:
            lists.append(ids.cpu().numpy().copy())
        return orig_add(self, ids, labels, pop, row0=row0, row_mask=row_mask, label_stride=label_stride)
    monkeypatch.setattr(ItemsStateUpdaterHook, 'after_run', spy_after)
    monkeypatch.setattr(EvalMetrics, 'add_lists', spy_add)
    ev = est.evaluate(lambda: iter(eval_batches))
    torch.cuda.synchronize()

    n, V = pb.hp.eval_metrics_top_n, pb.wl.num_items
    acr = pb.content_article_embeddings_matrix
    bref = BaselinesRef(V, acr=acr)
    kref = {'v-sknn': SknnRef(), 'sknn': SknnRef(first_session_clicks_decay='same')}
    for f, l in train_batches:
        ai = np.concatenate([f['item_clicked'], l['label_last_item'].reshape(-1, 1)], axis=1)
        bref.update(ai)
        for r in kref.values():
            r.update(f['session_id'], ai)
    names = ('',) + SUFFIXES + KNN
    ref = EvalMetricsRef(len(names), n, acr, 0.1)
    ref.begin(seen[0][1])
    for (f, l), (neg, buf, apop, pop, pred, labels), dev_ids in zip(eval_batches, seen, lists):
        ic, ln = f['item_clicked'], l['label_next_item']
        assert np.array_equal(np.sort(labels), np.sort(ln[ln != 0]))
        want = bref.score(ic, ln, neg, buf, apop, n)
        for s in KNN:
            want[s] = kref[s].score(ic, ln, neg, n)
        B, T = ic.shape
        for s in SUFFIXES + KNN:
            got = dev_ids[BaselineTables.row(s)]
            for q in np.flatnonzero(ln.reshape(-1)):
                if s == 'cb':
                    sc = bref.candidate_scores('cb', ic.reshape(-1)[q], [ln.reshape(-1)[q]] + neg.reshape(B * T, -1)[q].tolist(),
                                               buf, apop)
                    if np.any(np.diff(np.sort(np.array(list(sc.values())))) < 1e-6):
                        continue
                np.testing.assert_array_equal(got[q], want[s]['ids'][q], err_msg=s)
        ref.add_lists(0, pred, labels, pop)
        for i, s in enumerate(SUFFIXES + KNN):
            ref.add_lists(1 + i, dev_ids[BaselineTables.row(s)], ln.reshape(-1), pop)
        ref.add_clicks(ic, ln)
        ai = np.concatenate([ic, l['label_last_item'].reshape(-1, 1)], axis=1)
        bref.update(ai)
        for r in kref.values():
            r.update(f['session_id'], ai)
    for row, s in enumerate(names):
        w = ref.results(row)
        sfx = '_' + s if s else ''
        for k, v in zip(KEYS, VALUES):
            assert abs(ev[k + sfx] - w[v]) <= 1e-9 * abs(w[v]), (k + sfx, ev[k + sfx], w[v])
        assert ev[COVERAGE_KEY + sfx] == w['coverage'], s
    assert ev['ndcg_at_n'] > 0 and ev['item_coverage_at_n'] > 0


@gpu
def test_switch_changes_no_other_key(tmp_path):
    """From one checkpoint: every key evaluate returns with the switch off has the same value with it on - bit for bit,
    except two sums whose order of addition the existing evaluation kernels leave to the hardware, so that they differ in
    the last bits between any two runs, the switch on or off:
    * ``loss``: per-position float32 cross-entropy terms (positive) added with atomics (and the far smaller L2 term).  Two orders of n positive terms
      differ by at most 2 (n - 1) 2^-24 relative; n <= B * T per batch (on H100 two runs differed by ~3e-8).
    * ``mrr_at_n``: the model's reciprocal ranks added to an fp64 accumulator with atomics (nar_rank_candidates); all
      terms positive, so any two orders differ by at most 2 n 2^-53 relative over the n queries of the call.
    Every other key - HR (integer counts in fp64), each baseline's keys (fixed-order sums), global_step - is exact."""
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.eval_metrics import metric_names
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
    assert set(on) - set(off) == {k for s in ('',) + SUFFIXES + KNN for k in metric_names(s)}
    positions = max(np.asarray(f['item_clicked']).size for f, _ in eval_batches)
    queries = sum(int(np.count_nonzero(l['label_next_item'])) for _, l in eval_batches)
    tol = {'loss': 2 * (positions - 1) * 2.0 ** -24, 'mrr_at_n': 2 * queries * 2.0 ** -53}
    for k, v in off.items():
        if k in tol:
            assert abs(on[k] - v) <= tol[k] * abs(v), (k, on[k], v)
        else:
            assert on[k] == v, (k, on[k], v)
    torch.cuda.synchronize()


def test_empty_evaluate_returns_nan():
    from chameleon_recsys_b200.estimator import Estimator
    from chameleon_recsys_b200.eval_metrics import metric_names
    est = Estimator(None, {'eval_extended_metrics': True, 'eval_benchmarks': ['cb', 'v-sknn']})
    ev = est.evaluate(lambda: iter(()))
    for s in ('', 'cb', 'v-sknn'):
        for k in metric_names(s):
            assert np.isnan(ev[k]), k
