"""Data-parallel prediction == one-process prediction, bit for bit (NarEngine.recommend and Estimator.predict).

Every rank of the process group builds the same problem, runs recommend on a data-parallel engine (the group) and on a
one-process engine with the same weights, and compares the six arrays of the two dicts byte for byte: positions 'last' /
'all', candidates None / 'catalog' / an id array, with and without the exclusion of the session's clicks, on the tiny
workload, an empty recent-clicks buffer, batches where some or all ranks have no query, a G1-shaped batch of 64 and an
LSTM residual stack.  Then Estimator.predict with params['process_group'] against a one-process Estimator, both serving
the checkpoint a one-process run wrote to ``model_dir``.  Weights, Adam slots, global_step and ClickedItemsState must be
unchanged afterwards.  Raises AssertionError at the first difference.

tests/test_predict_dp_gpu.py runs run_checks in 2 and 3 processes sharing cuda:0 over gloo.  Launched by torchrun
(one rank per GPU, NCCL) this script runs the same checks and prints one line 'PREDICT_DP_CHECK {json}' on rank 0:
  torchrun --nproc-per-node 2 tools/predict_dp_check.py <model_dir>
"""
from __future__ import annotations

import copy
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chameleon_recsys_b200 import checkpoint as ckpt  # noqa: E402
from chameleon_recsys_b200.estimator import build_estimator  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from tools.gpu_step_check import make_engine  # noqa: E402

KEYS = ('query_session', 'query_position', 'candidates', 'predicted_item_ids', 'predicted_item_scores',
        'predicted_item_probs')


def same_bits(a: dict, b: dict, what):
    for k in KEYS:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape, (what, k, x.dtype, y.dtype, x.shape, y.shape)
        assert x.tobytes() == y.tobytes(), (what, k, 'first differing row',
                                            int(np.flatnonzero((x != y).reshape(x.shape[0], -1).any(1))[0]) if x.size else -1)


def _snapshot(eng):
    return [t.clone() for t in (eng.params, eng.adam_m, eng.adam_v)] + [eng.global_step]


def _unchanged(eng, snap, what):
    now = _snapshot(eng)
    assert all(torch.equal(a, b) for a, b in zip(now[:3], snap[:3])) and now[3] == snap[3], (what, 'engine state changed')


def _engines(pb, pg, device):
    logical = pb.layout.init_logical(pb.hp.init_seed)
    dp = make_engine(pb, process_group=pg, device=device)
    one = make_engine(pb, device=device)
    for e in (dp, one):
        e.set_params(logical)
    return dp, one


def _compare(dp, one, feats, buf, pop, cases, tag):
    snap = _snapshot(dp)
    n_queries = []
    for positions, cands, excl in cases:
        what = (tag, positions, cands if cands is None or isinstance(cands, str) else 'ids[%d]' % len(cands), excl)
        kw = dict(candidates=cands, positions=positions, exclude_session_clicks=excl)
        a = dp.recommend(feats, buf, pop, 10, **kw)
        b = one.recommend(feats, buf, pop, 10, **kw)
        same_bits(a, b, what)
        n_queries.append(int(a['query_session'].size))
    _unchanged(dp, snap, tag)
    return n_queries


def check_engines(pg, rank: int, world: int, device: int) -> dict:
    res = {}
    # ---- tiny: the whole matrix, then an empty buffer (the clicked rows' normalisation comes from the batch itself)
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 5)
    dp, one = _engines(pb, pg, device)
    feats, _ = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    ids = np.random.RandomState(1).choice(np.arange(1, pb.wl.num_items), 300, replace=False)
    cases = [(p, c, e) for p in ('last', 'all') for c in (None, 'catalog', ids) for e in (True, False)]
    res['tiny'] = _compare(dp, one, feats, buf, pop, cases, 'tiny')
    empty = np.zeros_like(buf)
    res['empty_buffer'] = _compare(dp, one, feats, empty, pop, [(p, c, True) for p in ('last', 'all') for c in ('catalog', ids)],
                                   'empty buffer')
    # ---- sessions without a valid position (session_size <= 1): one session keeps its queries, so every other rank
    # has none; then none at all (no rank gathers)
    lone = {k: np.array(v, copy=True) for k, v in feats.items()}
    keep = int(np.flatnonzero(np.asarray(feats['session_size']) > 2)[0])
    drop = np.arange(lone['item_clicked'].shape[0]) != keep
    lone['session_size'][drop] = np.where(np.arange(drop.sum()) % 2 == 0, 1, 0)
    lone['item_clicked'][drop, 1:] = 0
    res['one_session'] = _compare(dp, one, lone, buf, pop, [(p, c, True) for p in ('last', 'all') for c in (None, ids)],
                                  'one session with queries')
    assert res['one_session'][0] == 1
    none = {k: np.array(v, copy=True) for k, v in lone.items()}
    none['session_size'][keep] = 1
    res['no_session'] = _compare(dp, one, none, buf, pop, [('last', None, True), ('all', 'catalog', False)], 'no query')
    assert res['no_session'] == [0, 0]
    del dp, one
    # ---- LSTM residual stack
    pb = make_problem('tiny', profile='B', rnn_cell='lstm', rnn_residual_connections=True)
    warm_state(pb, 5)
    dp, one = _engines(pb, pg, device)
    feats, _ = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    res['lstm_residual'] = _compare(dp, one, feats, buf, pop, [('last', None, True), ('all', 'catalog', True)], 'lstm residual')
    del dp, one
    # ---- G1-shaped batch of 64 (46 033 articles, C = 1024)
    pb = make_problem('g1', profile='B', batch_size=64)
    warm_state(pb, 5)
    dp, one = _engines(pb, pg, device)
    feats, _ = pb.input_fn().get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
    ids = np.random.RandomState(2).choice(np.arange(1, pb.wl.num_items), 2000, replace=False)
    res['g1'] = _compare(dp, one, feats, buf, pop, [('last', None, True), ('all', None, False), ('last', 'catalog', True),
                                                    ('all', ids, True)], 'g1')
    del dp, one
    torch.cuda.synchronize()
    return res


def check_estimator(pg, rank: int, world: int, device: int, model_dir: str) -> dict:
    """Estimator.predict over the group == one-process Estimator.predict, from a checkpoint a one-process run wrote."""
    def est_for(pb, state, **kw):
        return build_estimator(model_dir, pb.content_article_embeddings_matrix, pb.articles_metadata,
                               pb.articles_features_config, pb.session_features_config, pb.hp, state, device=device, **kw)
    if rank == 0:                                     # the one-process training run (its own problem and stream)
        pt = make_problem('tiny', profile='B')
        warm_state(pt, 3)
        est_for(pt, pt.clicked_items_state).train(pt.input_fn, steps=3)
    dist.barrier(group=pg)
    latest = ckpt.latest_checkpoint(model_dir)
    assert latest is not None
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 4)
    batches = [pb.input_fn().get_next() for _ in range(2)]
    state = pb.clicked_items_state
    buf0, pop0 = state.get_recent_clicks_buffer().copy(), state.get_articles_recent_pop_norm().copy()
    dp = est_for(pb, state, process_group=pg)
    one = est_for(pb, copy.deepcopy(state))
    ids = np.random.RandomState(3).choice(np.arange(1, pb.wl.num_items), 200, replace=False)
    n = []
    for kw in (dict(), dict(positions='all', candidates='catalog'), dict(candidates=ids, exclude_session_clicks=False, top_n=7)):
        a = list(dp.predict(lambda: iter(batches), **kw))
        b = list(one.predict(lambda: iter(batches), **kw))
        assert len(a) == len(b) == sum(f['item_clicked'].shape[0] for f, _ in batches)
        for i, (x, y) in enumerate(zip(a, b)):
            assert sorted(x) == sorted(y) and np.array_equal(x['session_id'], y['session_id']), i
            for k in ('predicted_item_ids', 'predicted_item_scores', 'predicted_item_probs'):
                assert x[k].dtype == y[k].dtype and x[k].shape == y[k].shape and x[k].tobytes() == y[k].tobytes(), (kw, i, k)
        n.append(len(a))
    # weights, Adam slots and step are the checkpoint's; the state is what it was
    eng = dp._predict_spec.model.engine
    assert eng.world == world
    ck, sd = ckpt.load(latest), eng.state_dict()
    for g in ('params', 'adam_m', 'adam_v'):
        for name in eng.layout.logical_names():
            assert np.array_equal(sd[g][name], np.asarray(ck[g][name])), (g, name)
    assert sd['global_step'] == ck['global_step'] == 3
    assert np.array_equal(state.get_recent_clicks_buffer(), buf0)
    assert np.array_equal(state.get_articles_recent_pop_norm(), pop0)
    return {'estimator_sessions': n}


def run_checks(pg, rank: int, world: int, device: int, model_dir: str) -> dict:
    res = check_engines(pg, rank, world, device)
    res.update(check_estimator(pg, rank, world, device, model_dir))
    return res


def main():
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    try:
        res = run_checks(dist.group.WORLD, rank, world, local, sys.argv[1])
        if rank == 0:
            print('PREDICT_DP_CHECK ' + json.dumps(dict(res, world=world, backend='nccl')))
            sys.stdout.flush()
    finally:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
