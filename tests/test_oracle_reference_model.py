"""The float path of the oracle (oracle/nar_oracle.py) against outputs of the REFERENCE's own model code.

tests/golden/model_golden.npz was produced by importing /root/reference/nar_module/nar/nar_model.py unmodified and running
NARModuleModel's constructor on an eager stand-in for the TF-1.x API (tests/golden/tf1_shim.py; generator:
tests/golden/make_model_golden.py).  So the WIRING compared here is the reference's: feature order, embedding / one-hot
choice, recency and novelty normalisation (incl. the float32 cast of the millisecond timestamps before they are
subtracted and the cold-start branch), gamma / beta, the shared CAR layers, UGRNN over masked sequences, FC1 / FC2,
the product + 4-layer scorer, temperature, masked mean of the cross-entropy, WHICH variables are L2-regularised, the
novelty regulariser, multi-layer RNN, and in EVAL mode the ranking and the recall@n / MRR@n batch values.  Per-op TF
kernel semantics are the shim's restatement of the TF documentation (see its docstring) - that part stays unpinned.

The oracle gets the reference's variables (by TF name), the batch, the state arrays and the negatives the reference's
own sampler drew, and must reproduce logits, loss, every intermediate the reference exposes as a histogram, every
gradient and the first Adam step."""
import os

import numpy as np
import pytest
import torch

from chameleon_recsys_b200.harness import make_problem
from oracle.golden_sampling import preset_variables, sample_index
from tools.gpu_step_check import make_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'model_golden.npz')


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def _tf_name_to_layout(n: str) -> str:
    """tf.layers.Dense creates its variables under the scope of its FIRST call; plan.ParamLayout names the two shared layers
    by the scope they are constructed in.  Everything else carries the TF name."""
    n = n.replace('main/user_personalized_contextual_article_embedding/input/CAR_representation', 'main/CAR/CAR_representation')
    return n.replace('main/recommendations_ranking/cos_sim_positive/', 'main/recommendations_ranking/')


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _sampled(a, ref):
    """`a` at the entries make_model_golden.py kept of the same tensor (`ref`: the stored sample)."""
    a = np.asarray(a).reshape(-1)
    return a[sample_index(a.size, np.asarray(ref).size)]


def _load(d, case, hp_over, dtype):
    P = case + '/'
    pb = make_problem('tiny', profile='B', **hp_over)
    orc = make_oracle(pb, dtype)
    # the variables THIS case's graph created, with the values the reference graph ran with
    tf_vars = preset_variables(d, case)
    orc.set_params({_tf_name_to_layout(n): v for n, v in tf_vars.items()})
    assert set(_tf_name_to_layout(n) for n in tf_vars) == set(pb.layout.init_logical(1).keys())      # same variable set, same shapes
    for n, v in tf_vars.items():
        assert pb.layout.init_logical(1)[_tf_name_to_layout(n)].shape == v.shape, n
    f = {k[len(P) + 5:]: d[k] for k in d.files if k.startswith(P + 'feat/')}
    lab = {k[len(P) + 6:]: d[k] for k in d.files if k.startswith(P + 'label/')}
    return pb, orc, f, lab, d[P + 'negatives'], d[P + 'buffer'], d[P + 'pop_norm'], tf_vars


CASES = [('train64', {}, torch.float64, 1e-7), ('train32', {}, torch.float32, 2e-5), ('cold64', {}, torch.float64, 1e-7),
         ('nov64', {'novelty_reg_factor': 0.3}, torch.float64, 1e-7), ('layers2_64', {'rnn_num_layers': 2}, torch.float64, 1e-7),
         ('featoff64', {'enabled_internal_features': ['recency', 'article_content_embeddings']}, torch.float64, 1e-7),
         # the reference code with the stand-in's GRUCell in place of UGRNNCell (= un-commenting nar_model.py:1315): pins where
         # the oracle's GRU branch sits in the graph; the cell formula itself is the TF documentation's, restated twice
         ('gru64', {'rnn_num_layers': 2, 'rnn_cell': 'gru'}, torch.float64, 1e-7)]


@pytest.mark.parametrize('case,hp_over,dtype,tol', CASES, ids=[c[0] for c in CASES])
def test_train_graph_matches_reference_code(golden, case, hp_over, dtype, tol):
    d = golden
    P = case + '/'
    pb, orc, f, lab, neg, buf, pop, tf_vars = _load(d, case, hp_over, dtype)
    if case == 'cold64':
        assert not buf.any()                               # empty recent-clicks buffer: statistics come from the batch
    o = orc.forward(f, lab, neg, buf, pop)
    mask = o['mask'].numpy().astype(bool)
    assert mask.sum() > 100
    # loss and (temperature-scaled) logits
    assert abs(float(o['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) < tol
    assert _rel(_sampled(o['logits'].detach().numpy()[mask], d[P + 'logits_sample']), d[P + 'logits_sample']) < tol
    # which variables the reference regularises: Dense kernels, embeddings, gamma / beta - no bias, no RNN weight
    reg_ref = sorted(_tf_name_to_layout(str(n)) for n in d[P + 'reg_names'])
    assert reg_ref == sorted(n for n in orc.params if not (n.endswith('/bias') or '/RNN/' in n))
    reg = sum(float((tf_vars[str(n)].astype(np.float64) ** 2).sum()) / 2 for n in d[P + 'reg_names']) * pb.hp.reg_l2
    assert abs(float(o['reg_loss'].detach()) - reg) / reg < max(tol, 1e-6 if dtype == torch.float32 else 0)
    # intermediates the reference exposes as histograms (valid positions)
    if (P + 'hist/input_user_items_features') in d.files:
        H = lambda n: d[P + 'hist/' + n]      # noqa: E731
        rows = sample_index(int(mask.sum()), H('input_user_items_features').shape[0])      # the valid positions kept
        V = lambda t: t.detach().numpy()[mask][rows]      # noqa: E731
        assert _rel(V(o['x_in']), H('input_user_items_features')) < tol      # (recency column: f32 division)
        n_ctx = H('user_context_features').shape[1]
        # x = concat(user context, item features) * gamma + beta   (nar_model.py:332-333, :997)
        g = tf_vars['main/user_items_contextual_features/input_features_center_scale/gamma_scale'].astype(np.float64)
        b = tf_vars['main/user_items_contextual_features/input_features_center_scale/beta_center'].astype(np.float64)
        cat_pos = np.concatenate([H('user_context_features'), H('positive_items_features')], axis=1)
        assert n_ctx + H('positive_items_features').shape[1] == g.shape[0]
        assert _rel(V(o['x_pos']), cat_pos * g + b) < tol
        assert _rel(V(o['e_in']), H('input_contextual_item_embedding')) < tol
        assert _rel(V(o['e_pos']), H('positive_contextual_item_embedding')) < tol
        assert _rel(V(o['rnn_out']), H('rnn/outputs')) < tol
        assert _rel(V(o['pred']), H('predicted_contextual_item_embedding')) < tol
    # gradients of total_loss w.r.t. every variable (the last bias has an analytically zero gradient: absolute scale)
    grads = orc.compute_gradients(o)
    gmax = max(float(np.abs(d[k]).max()) for k in d.files if k.startswith(P + 'grad/'))
    for n_tf in tf_vars:
        g_ref = d[P + 'grad/' + n_tf]
        g_orc = _sampled(grads[_tf_name_to_layout(n_tf)].detach().numpy(), g_ref)
        assert float(np.abs(g_orc - g_ref).max()) < max(tol, 2e-7) * gmax * 10, n_tf
        if np.abs(g_ref).max() > 1e-6 * gmax:
            assert _rel(g_orc, g_ref) < max(tol * 50, 1e-5), n_tf
    # the one AdamOptimizer step of the constructor (first case): entries whose gradient is not rounding noise
    if (P + 'adam_delta/main/CAR/PreCAR_representation/bias') in d.files:
        before = orc.get_params()
        orc.apply_gradients(grads)
        after = orc.get_params()
        for n_tf in tf_vars:
            n = _tf_name_to_layout(n_tf)
            ref = d[P + 'adam_delta/' + n_tf].astype(np.float64)
            delta = _sampled(after[n].astype(np.float64) - before[n].astype(np.float64), ref)
            gr = d[P + 'grad/' + n_tf].astype(np.float64)          # sampled at the same entries
            sel = np.abs(gr) > 1e-9 * gmax
            if not sel.any():                                 # matching_dense_layer_4/bias: the softmax is shift invariant
                continue
            assert float(np.abs(delta - ref)[sel].max()) < 2e-3 * pb.hp.learning_rate, n_tf


def test_eval_graph_matches_reference_code(golden):
    d = golden
    P = 'eval64/'
    pb, orc, f, lab, neg, buf, pop, _ = _load(d, 'eval64', {}, torch.float64)
    o = orc.forward(f, lab, neg, buf, pop)
    mask = o['mask'].numpy().astype(bool)
    assert abs(float(o['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) < 1e-7
    assert _rel(o['logits'].detach().numpy()[mask], d[P + 'logits_scaled'][mask]) < 1e-7
    top_n = pb.hp.eval_metrics_top_n
    ids, probs, hits, rr, cnt = orc.rank_and_metrics(o, lab, neg, top_n)
    assert np.array_equal(np.asarray(ids)[mask], d[P + 'predicted_item_ids'][mask])           # rank_items_by_predicted_prob
    assert _rel(np.asarray(probs)[mask], d[P + 'predicted_item_probs'][mask]) < 1e-7
    assert cnt == mask.sum()
    assert abs(hits / cnt - float(d[P + 'recall_at_n'])) < 1e-12                              # sparse_recall_at_top_k
    assert abs(rr / cnt - float(d[P + 'mrr_at_n'])) < 1e-12                                   # define_mrr_metric


def test_reference_sampler_output_has_the_properties_the_oracle_sampler_guarantees(golden):
    """The negatives in the golden file were drawn by the reference's TF sampler code (nar_model.py:1239-1300) on the shim.
    TF's shuffles cannot be reproduced, so the product's sampler is defined by oracle/sampler_ref.py's counter-based RNG; what
    both must share are the reference's structural guarantees: zeros at padded clicks, K distinct ids per real click, none
    of them clicked in that session (label included), all from batch clicks + recent-clicks buffer."""
    from oracle import sampler_ref
    d = golden
    for case in ('train64', 'cold64', 'eval64'):
        P = case + '/'
        neg = d[P + 'negatives']
        clicked, last = d[P + 'feat/item_clicked'], d[P + 'label/label_last_item']
        buf = d[P + 'buffer']
        allc = np.concatenate([clicked, last], axis=1)
        B, T, K = neg.shape
        assert (B, T) == clicked.shape
        pool = set(allc[allc != 0].tolist()) | set(buf[buf != 0].tolist())
        ours = sampler_ref.sample_negatives(allc, buf, K, 300, 42, 1)
        assert ours.shape == neg.shape
        for arr in (neg, ours):
            for b in range(B):
                sess = set(allc[b].tolist())
                for t in range(T):
                    row = arr[b, t]
                    if clicked[b, t] == 0:
                        assert not row.any()
                        continue
                    nz = row[row != 0]
                    assert len(set(nz.tolist())) == len(nz)
                    assert not (set(nz.tolist()) & sess)
                    assert set(nz.tolist()) <= pool
                    assert not row[len(nz):].any()            # padding (pool exhausted) only at the end


def test_dropout_sites_match_reference_code(golden):
    """keep_prob 0.8, two RNN layers: the reference code ran with the stand-in's random masks; the SAME masks are handed to
    the oracle (mask_override), which must then reproduce loss, logits and gradients - i.e. dropout sits at the same five
    sites (input / positive / negative feature rows after gamma-beta, every cell's OUTPUT but not its state, FC1) with the
    same 1 / keep_prob scaling.  (The product's own masks are defined by oracle/dropout_ref.py's counter-based RNG.)"""
    d = golden
    P = 'drop64/'
    hp_over = {'dropout_keep_prob': 0.8, 'rnn_num_layers': 2}
    pb, orc, f, lab, neg, buf, pop, tf_vars = _load(d, 'drop64', hp_over, torch.float64)

    def unpack(n):
        shp = tuple(int(v) for v in d[P + 'mask_shape/' + n])
        return np.unpackbits(d[P + 'mask/' + n])[:int(np.prod(shp))].reshape(shp).astype(bool)

    rnn = unpack('rnn')                                      # [T, layers, B, H]
    over = {1: unpack('in'), 2: unpack('pos'), 3: unpack('neg'), 4: unpack('fc1')}
    for t in range(rnn.shape[0]):
        for i in range(rnn.shape[1]):
            over[(8 + i, t)] = rnn[t, i]
    assert 0.75 < over[3].mean() < 0.85
    orc.mask_override = over
    o = orc.forward(f, lab, neg, buf, pop, train_step=1)
    mask = o['mask'].numpy().astype(bool)
    assert abs(float(o['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) < 1e-7
    assert _rel(_sampled(o['logits'].detach().numpy()[mask], d[P + 'logits_sample']), d[P + 'logits_sample']) < 1e-7
    grads = orc.compute_gradients(o)
    gmax = max(float(np.abs(d[k]).max()) for k in d.files if k.startswith(P + 'grad/'))
    for n_tf in tf_vars:
        g_ref = d[P + 'grad/' + n_tf]
        g_orc = _sampled(grads[_tf_name_to_layout(n_tf)].detach().numpy(), g_ref)
        assert float(np.abs(g_orc - g_ref).max()) < 2e-6 * gmax, n_tf
    # and without the masks the result differs (the check above is not vacuous)
    orc.mask_override = None
    o2 = orc.forward(f, lab, neg, buf, pop, train_step=1)
    assert abs(float(o2['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) > 1e-4


def test_reference_model_fn_accepts_this_repos_params(golden):
    """tests/golden/make_model_fn_golden.py called the REFERENCE's nar_module_model_fn (nar_trainer_gcom.py:234-332) with the
    params dict NARHParams.to_params builds (what this repo's build_estimator passes to its own model_fn): it accepted the
    dict in TRAIN and EVAL and produced exactly the losses of the direct-constructor golden cases, i.e. key names, the
    train / eval choice of sampling sizes and keep_prob = 1 in EVAL line up with the reference's trainer."""
    import json
    with open(os.path.join(os.path.dirname(GOLDEN), 'model_fn_golden.json')) as f:
        g = json.load(f)
    for mode in ('train', 'eval'):
        assert abs(g[mode]['loss'] - float(golden[g[mode]['golden_case'] + '/total_loss'])) < 1e-12
    assert g['eval']['eval_metric_ops'] == ['hitrate_at_n', 'mrr_at_n']
    pb = make_problem('tiny', profile='B')
    params = pb.hp.to_params(pb.session_features_config, pb.articles_features_config, pb.articles_metadata,
                             pb.content_article_embeddings_matrix)
    assert sorted(params) == g['train']['params_keys_passed']                 # the dict has not drifted since
