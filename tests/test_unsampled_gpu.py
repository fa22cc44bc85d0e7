"""The unsampled evaluation on the H100 (DESIGN.md section 13): nar_rank_labels against numpy bit for bit, NarEngine.
rank_labels against the sampled EVAL step's ranks and the fp64 oracle (oracle/unsampled_ref.py), block-size invariance,
the switch changing nothing else in Estimator.evaluate, and a G1-shaped evaluate."""
import copy
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _order_key(x):
    """topn_kernel's order_key: -0 -> +0, every NaN -> the canonical 0x7fffffff (above +inf), then the order-preserving
    map to uint32."""
    x = np.asarray(x, dtype=np.float32)
    b = x.view(np.uint32).copy()
    b[x == 0] = 0
    b[np.isnan(x)] = 0x7fffffff
    return np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)


def _rank_numpy(lg, cand, label_next, all_items, q_pos, T, top_n):
    Q, N = lg.shape
    rank = np.full(Q, -1, np.int32)
    hist = np.zeros(top_n + 2, np.int64)
    keys = _order_key(lg)
    for q in range(Q):
        b = q_pos[q] // T
        lab = label_next.reshape(-1)[q_pos[q]]
        j = np.flatnonzero(cand == lab)
        if lab == 0 or j.size == 0:
            continue
        comp = ~np.isin(cand, all_items[b])
        comp[j[0]] = False
        rank[q] = np.count_nonzero(keys[q, comp] > keys[q, j[0]])
        if rank[q] < top_n:
            hist[rank[q]] += 1
        hist[top_n] += 1
        hist[top_n + 1] += comp.sum()
    return rank, hist


def _kernel_case(name):
    rs = np.random.RandomState(len(name))
    if name == 'ties_zero_nan':
        Q, N, T = 9, 37, 6
    elif name == 'n1':
        Q, N, T = 4, 1, 3
    elif name == 'wide':
        Q, N, T = 700, 5000, 8
    else:                                              # 'max_row': the longest session row the kernel takes
        Q, N, T = 6, 900, 1023
    cand = np.sort(rs.choice(np.arange(1, 4 * N + 10), N, replace=False)).astype(np.int64)
    B = Q
    lg = rs.randn(Q, N).astype(np.float32)
    label_next = np.zeros((B, T), np.int64)
    all_items = rs.randint(1, 4 * N + 10, size=(B, T + 1)).astype(np.int64)
    q_pos = (np.arange(Q) * T + rs.randint(0, T, Q)).astype(np.int32)
    lab_j = rs.randint(0, N, Q)
    label_next.reshape(-1)[q_pos] = cand[lab_j]
    if name == 'ties_zero_nan':
        lg = np.round(lg * 2).astype(np.float32) / 2              # a handful of values: ties with the label
        lg[0, lab_j[0]] = -0.0; lg[0, ::3] = 0.0                  # -0 label, +0 competitors: ties
        lg[1, lab_j[1]] = 0.0; lg[1, 1::4] = -0.0
        lg[2, ::5] = np.nan                                       # NaN competitors order above everything
        lg[3, lab_j[3]] = np.nan                                  # a NaN label: nothing above it
        lg[4, ::7] = -np.float32(np.nan); lg[4, 2] = np.inf
        lg[5, lab_j[5]] = np.inf; lg[5, 3] = np.inf
        label_next.reshape(-1)[q_pos[6]] = 0                      # label 0: not ranked
        label_next.reshape(-1)[q_pos[7]] = 4 * N + 20             # a label outside the candidates: not ranked
        all_items[8] = cand[rs.randint(0, N, T + 1)]              # a row of candidates, the label among them
        all_items[8, 0] = cand[lab_j[8]]
    if name == 'n1':
        all_items[1, 0] = cand[0]
    if name == 'max_row':
        for q in range(Q):
            row = np.concatenate([cand[rs.randint(0, N, 600)], np.zeros(100, np.int64), rs.randint(1, 9 * N, 324)])
            all_items[q] = row[rs.permutation(T + 1)]             # duplicates, padding zeros, ids outside the candidates
        others = np.setdiff1d(cand, [cand[lab_j[0]]])
        all_items[0, :others.size] = others                       # every competitor of query 0 excluded: rank 0
        all_items[0, others.size:] = 0
    return lg, cand, label_next, all_items, q_pos, T


@pytest.mark.parametrize('case', ['max_row', 'n1', 'ties_zero_nan', 'wide'])
def test_rank_kernel_matches_numpy(case):
    import torch
    from chameleon_recsys_b200 import ops
    lg, cand, label_next, all_items, q_pos, T = _kernel_case(case)
    Q, N = lg.shape
    for top_n in (1, 5, 20):
        rank = torch.full((Q,), -7, dtype=torch.int32, device='cuda')
        hist = torch.zeros(top_n + 2, dtype=torch.int64, device='cuda')
        args = (_dev(lg), _dev(cand), Q, N, _dev(label_next), _dev(all_items), _dev(q_pos), T, top_n, rank, hist)
        ops.rank_labels(*args)
        ops.rank_labels(*args)                                   # the histogram accumulates
        want_r, want_h = _rank_numpy(lg, cand, label_next, all_items, q_pos, T, top_n)
        assert np.array_equal(rank.cpu().numpy(), want_r), (case, top_n)
        assert np.array_equal(hist.cpu().numpy(), 2 * want_h), (case, top_n)
        if case == 'max_row':
            assert want_r[0] == 0 and want_h[top_n + 1] > 0
        if case == 'ties_zero_nan':
            assert want_r[3] == 0 and (want_r[6], want_r[7]) == (-1, -1)       # a NaN label: nothing orders above it


def test_rank_kernel_rejects_a_longer_row():
    import torch
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import NarError
    T = 1024
    rank = torch.empty(1, dtype=torch.int32, device='cuda')
    hist = torch.zeros(3, dtype=torch.int64, device='cuda')
    with pytest.raises(NarError):
        ops.rank_labels(_dev(np.zeros((1, 4), np.float32)), _dev(np.arange(1, 5)), 1, 4, _dev(np.ones((1, T), np.int64)),
                        _dev(np.zeros((1, T + 1), np.int64)), _dev(np.zeros(1, np.int32)), T, 1, rank, hist)


def _setup(name='tiny', warm=5, oracle=False, **hp):
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools.gpu_step_check import make_engine, make_oracle
    pb = make_problem(name, profile='B', **hp)
    warm_state(pb, warm)
    eng = make_engine(pb)
    logical = pb.layout.init_logical(pb.hp.init_seed)
    eng.set_params(logical)
    orc = None
    if oracle:
        orc = make_oracle(pb, torch.float64)
        orc.set_params(logical)
    feats, labels = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    return pb, eng, orc, feats, labels, buf, pop


def test_engine_rejects_a_longer_session():
    pb, eng, _, feats, labels, buf, pop = _setup(warm=2)
    T = np.asarray(feats['item_clicked']).shape[1]
    wide = {k: (np.pad(v, ((0, 0), (0, 1024 - T))) if np.ndim(v) == 2 and np.shape(v)[1] == T else v) for k, v in feats.items()}
    lab = dict(labels, label_next_item=np.pad(labels['label_next_item'], ((0, 0), (0, 1024 - T))))
    st = eng.stage(wide, lab, buf, pop, slot='eval')
    with pytest.raises(ValueError):
        eng.rank_labels(st, eng.unsampled_pool(wide['item_clicked'], lab['label_last_item'], buf), 5)


@pytest.mark.parametrize('name,ranking', [('tiny', 'mlp'), ('tiny', 'cosine'), ('g1', 'mlp')])
def test_consistent_with_the_sampled_eval_rank(name, ranking):
    """With the candidates restricted to one query's label and its logged eval negatives, the unsampled rank is the EVAL
    step's rank of that query, except where a negative's logit lies within the recorded PP-vs-PC+PI gap (1e-4 of the
    largest logit, DESIGN.md section 8) of the label's: those are counted and reported."""
    pb, eng, _, feats, labels, buf, pop = _setup(name, warm=20 if name == 'g1' else 5, ranking=ranking)
    out = eng.eval_step(feats, labels, buf, pop, top_n=3)
    st = out['stage']
    L, n_cand = st['L'], eng.K + 1
    lg = out['logits'].cpu().numpy().reshape(L, n_cand)
    ids = eng.buffer(st, 'row_item').view(-1)[L:L + L * n_cand].cpu().numpy().reshape(L, n_cand)
    pred = out['predicted_item_ids'].cpu().numpy()
    gap = 1e-4 * np.abs(lg).max()
    rs = np.random.RandomState(3)
    picks = rs.choice(L, min(L, 12), replace=False)
    close = 0
    for q in picks:
        if ids[q, 0] == 0 or not ids[q, 1:].all():     # (a zero-padded negative is ranked in EVAL, not a candidate here)
            continue
        negs = ids[q, 1:][ids[q, 1:] != 0]
        sampled = int(np.flatnonzero(pred[q] == ids[q, 0])[0])
        r = eng.rank_labels(st, np.concatenate([[ids[q, 0]], negs]), 3)['rank'].cpu().numpy()
        if np.any(np.abs(lg[q, 1:][ids[q, 1:] != 0] - lg[q, 0]) <= gap):
            close += 1
            continue
        assert r[q] == sampled, (q, r[q], sampled)
    print('queries with a negative within the PP-vs-PC+PI gap of the label: %d of %d' % (close, len(picks)))
    assert close < len(picks)


@pytest.mark.parametrize('cell', ['ugrnn', 'gru', 'lstm'])
def test_against_the_fp64_oracle(cell):
    import torch
    from oracle.unsampled_ref import unsampled
    pb, eng, orc, feats, labels, buf, pop = _setup(oracle=True, rnn_cell=cell, batch_size=24)
    top_n = pb.hp.eval_metrics_top_n
    out = eng.eval_step(feats, labels, buf, pop, top_n=top_n)
    res = eng.rank_labels(out['stage'], eng.unsampled_pool(feats['item_clicked'], labels['label_last_item'], buf), top_n)
    rank = res['rank'].cpu().numpy()
    ref = unsampled(orc, feats, labels, buf, pop, top_n)
    assert np.array_equal(res['candidates'], ref['candidates'])
    got = rank[rank >= 0]
    assert got.size == ref['rank'].size > 0
    bar = 1e-3 * np.abs(ref['scores']).max()
    close = ref['gap'] < bar
    assert np.array_equal(got[~close], ref['rank'][~close]), cell
    from chameleon_recsys_b200.eval_metrics import unsampled_results
    mine = unsampled_results(res['hist'].cpu().numpy(), top_n)
    Q = got.size
    for k in ('unsampled_hitrate_at_n', 'unsampled_mrr_at_n', 'unsampled_ndcg_at_n'):
        assert abs(mine[k] - ref[k]) <= close.sum() / Q + 1e-12, (k, mine[k], ref[k])
    assert mine['unsampled_candidates_per_query'] == ref['unsampled_candidates_per_query']
    torch.cuda.synchronize()


@pytest.mark.parametrize('ranking', ['mlp', 'cosine'])
def test_blocking_is_bit_identical(ranking):
    pb, eng, _, feats, labels, buf, pop = _setup(ranking=ranking)
    top_n = pb.hp.eval_metrics_top_n
    out = eng.eval_step(feats, labels, buf, pop, top_n=top_n)
    pool = eng.unsampled_pool(feats['item_clicked'], labels['label_last_item'], buf)
    from chameleon_recsys_b200._lib import NarError
    full = eng.rank_labels(out['stage'], pool, top_n)
    want_r, want_h = full['rank'].cpu().numpy(), full['hist'].cpu().numpy()
    blocks = set()
    for budget in range(2 << 20, 0, -(64 << 10)):       # down to the smallest workspace that holds one query x one candidate
        try:
            small = eng.rank_labels(out['stage'], pool, top_n, ws_budget=budget)
        except NarError:
            break
        blocks.add((small['q_block'], small['n_block']))
        assert np.array_equal(small['rank'].cpu().numpy(), want_r), budget
        assert np.array_equal(small['hist'].cpu().numpy(), want_h), budget
    assert any(q < out['stage']['L'] for q, _ in blocks) and any(n < pool.size for _, n in blocks), blocks


def _problem():
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 2)
    return pb


def test_the_switch_changes_nothing_else(tmp_path):
    """From one checkpoint, evaluate with the switch off and on, with every other evaluation extension on: every key of
    the off run has the same value - bit for bit, except the loss and the model's MRR, which the existing evaluation
    kernels sum with float atomics and which are held to the rounding bound of their summation order (DESIGN.md
    section 10) -, the negatives log is the same, and so is the ClickedItemsState afterwards."""
    import torch
    from chameleon_recsys_b200 import checkpoint as ckpt
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.eval_metrics import UNSAMPLED_KEYS
    from oracle.baselines_ref import SUFFIXES
    pb = _problem()
    it = pb.input_fn()
    train_batches = [it.get_next() for _ in range(6)]
    eval_batches = [it.get_next() for _ in range(3)]
    d = str(tmp_path)
    all7 = tuple({'recommender': s, 'params': {}} for s in SUFFIXES + ('v-sknn', 'sknn'))

    def est(state, on, **extra):
        hp = pb.hp.copy(eval_benchmarks=all7, eval_extended_metrics=True, eval_metrics_by_session_position=True,
                        eval_unsampled_metrics=on)
        return build_estimator(d, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                               pb.session_features_config, hp, state, device=0, **extra)
    est(pb.clicked_items_state, False).train(lambda: iter(train_batches))
    saved = ckpt.load(ckpt.latest_checkpoint(d))
    st = pb.clicked_items_state
    runs, logs, states = {}, {}, {}
    for name, on in (('off', False), ('on', True)):
        fresh = ClickedItemsState(st.recent_clicks_buffer_hours, st.recent_clicks_buffer_max_size,
                                  st.recent_clicks_for_normalization, st.num_items)
        for f in ckpt.STATE_FIELDS:
            setattr(fresh, f, np.array(saved['state'][f]))
        logs[name] = []
        runs[name] = est(fresh, on, sessions_negative_items_log=logs[name]).evaluate(lambda: iter(eval_batches))
        states[name] = {f: copy.deepcopy(getattr(fresh, f)) for f in ckpt.STATE_FIELDS}
    off, on = runs['off'], runs['on']
    assert set(on) - set(off) == set(UNSAMPLED_KEYS)
    assert all(np.isfinite(on[k]) for k in UNSAMPLED_KEYS)
    positions = max(np.asarray(f['item_clicked']).size for f, _ in eval_batches)
    queries = sum(int(np.count_nonzero(l['label_next_item'])) for _, l in eval_batches)
    tol = {'loss': 2 * (positions - 1) * 2.0 ** -24, 'mrr_at_n': 2 * queries * 2.0 ** -53}
    for k, v in off.items():
        if k in tol:
            assert abs(on[k] - v) <= tol[k] * abs(v), (k, on[k], v)
        else:
            assert on[k] == v or (np.isnan(v) and np.isnan(on[k])), (k, on[k], v)
    assert logs['on'] == logs['off'] and len(logs['on']) > 0
    for f in ckpt.STATE_FIELDS:
        assert np.array_equal(np.asarray(states['on'][f]), np.asarray(states['off'][f])), f
    torch.cuda.synchronize()


def test_g1_estimator_evaluate():
    """A G1-shaped batch through Estimator.evaluate: finite keys, and the mean competitor count is the oracle's for the
    same batch and state."""
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from oracle.unsampled_ref import competitor_sets, queries
    pb = make_problem('g1', profile='B')
    warm_state(pb, 20)
    it = pb.input_fn()
    train = [it.get_next() for _ in range(2)]
    batch = it.get_next()
    hp = pb.hp.copy(eval_unsampled_metrics=True)
    est = build_estimator(None, pb.content_article_embeddings_matrix, pb.articles_metadata, pb.articles_features_config,
                          pb.session_features_config, hp, pb.clicked_items_state, device=0)
    est.train(lambda: iter(train))
    f, l = batch
    sets = competitor_sets(f['item_clicked'], l['label_last_item'], pb.clicked_items_state.get_recent_clicks_buffer())
    qs, _ = queries(f, l)
    want = float(sum(sets[b].size for b in qs)) / qs.size
    ev = est.evaluate(lambda: iter([batch]))
    for k in ('unsampled_hitrate_at_n', 'unsampled_mrr_at_n', 'unsampled_ndcg_at_n', 'unsampled_candidates_per_query'):
        assert np.isfinite(ev[k]), k
    assert ev['unsampled_candidates_per_query'] == want
    print('G1 batch: %d queries, %.1f competitors per query, unsampled HR@n %.4f vs sampled %.4f'
          % (qs.size, want, ev['unsampled_hitrate_at_n'], ev['hitrate_at_n']))
