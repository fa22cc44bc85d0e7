"""Generate tests/golden/model_golden.npz: outputs of the REFERENCE model code
(/root/reference/nar_module/nar/nar_model.py, class NARModuleModel, imported unmodified) executed on the eager TF-1.x
stand-in tests/golden/tf1_shim.py (TensorFlow 1.12 itself cannot be installed here).  See the shim's docstring for what
this pins (the model's wiring - the reference's own code ran) and what it does not (per-op TF kernel semantics, which are
the shim's restatement of the TF documentation).

Per case the file holds: the batch (features, labels), the state arrays fed to the placeholders, the mean / std of the
reference's initializer and the shape of every variable (the graph runs with oracle/golden_sampling.preset_variable values), the negatives the reference's sampler drew (the oracle takes them as an input: TF's shuffles are not
reproducible), the tensors the reference itself sends to tf.summary.histogram (plot_histograms=True), the scaled logits
(input of the first tf.nn.softmax), total_loss, d(total_loss)/d(variable) for every variable, and the variables after
the one AdamOptimizer step of the constructor.  EVAL cases hold predicted_item_ids / predicted_item_probs and the batch
values of the recall@n / MRR@n streaming metrics.  Gradients, Adam deltas, TRAIN logits and the intermediates (first case
only) are kept at a fixed seeded sample of their entries / rows (oracle/golden_sampling.sample_index): the file stays < 1 MB.

Run once in the build container (python tests/golden/make_model_golden.py); the .npz is committed."""
import importlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import tf1_shim as shim  # noqa: E402  (registers itself as `tensorflow` in sys.modules)

import pandas  # noqa: E402,F401  (before the pytz stub: pandas probes pytz as an optional dependency)

# the reference's utils.py imports two preprocessing-only packages that are not installed here
sys.modules.setdefault('pytz', types.ModuleType('pytz'))
_ua = types.ModuleType('ua_parser')
_ua.user_agent_parser = types.ModuleType('ua_parser.user_agent_parser')
sys.modules.setdefault('ua_parser', _ua)
sys.modules.setdefault('ua_parser.user_agent_parser', _ua.user_agent_parser)

REF_DIR = '/root/reference/nar_module/nar'
pkg = types.ModuleType('refnar')
pkg.__path__ = [REF_DIR]
sys.modules['refnar'] = pkg
ref = importlib.import_module('refnar.nar_model')

import torch  # noqa: E402

torch.set_num_threads(1)      # float32 scatter-add order (embedding gradients) would otherwise vary run to run at 1e-7
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from oracle.golden_sampling import preset_variable, sample_index  # noqa: E402


def build(pb, feats, labels, buf, pop, mode, float64, preset, seed, **over):
    hp = pb.hp
    shim.configure(float64=float64, seed=seed, preset=preset, feeds={
        'articles_metadata': [pb.articles_metadata[k] for k in pb.articles_metadata],
        'content_article_embeddings_matrix': pb.content_article_embeddings_matrix,
        'articles_recent_pop_norm': np.asarray(pop, dtype=np.float32),
        'pop_recent_items_buffer': np.asarray(buf, dtype=np.int64)})
    inputs = {k: shim._t(np.asarray(v)) for k, v in feats.items()}
    labs = {k: shim._t(np.asarray(v)) for k, v in labels.items()}
    train = mode == 'train'
    kw = dict(session_features_config=pb.session_features_config, articles_features_config=pb.articles_features_config,
              batch_size=hp.batch_size, lr=hp.learning_rate, keep_prob=hp.dropout_keep_prob,
              negative_samples=hp.train_total_negative_samples if train else hp.eval_total_negative_samples,
              negative_sample_from_buffer=hp.train_negative_samples_from_buffer if train else hp.eval_negative_samples_from_buffer,
              content_article_embeddings_matrix=pb.content_article_embeddings_matrix, rnn_num_layers=hp.rnn_num_layers,
              softmax_temperature=hp.softmax_temperature, reg_weight_decay=hp.reg_l2,
              recent_clicks_buffer_hours=hp.recent_clicks_buffer_hours,
              recent_clicks_buffer_max_size=hp.recent_clicks_buffer_max_size,
              recent_clicks_for_normalization=hp.recent_clicks_for_normalization, articles_metadata=pb.articles_metadata,
              plot_histograms=True, metrics_top_n=hp.eval_metrics_top_n,
              elapsed_days_smooth_log_base=hp.elapsed_days_smooth_log_base,
              popularity_smooth_log_base=hp.popularity_smooth_log_base, CAR_embedding_size=hp.CAR_embedding_size,
              rnn_units=hp.rnn_units, max_cardinality_for_ohe=hp.max_cardinality_for_ohe,
              novelty_reg_factor=hp.novelty_reg_factor, diversity_reg_factor=0.0,
              internal_features_config=pb.internal_features_config, eval_cold_start=False)
    kw.update(over)
    model = ref.NARModuleModel(mode, inputs, labs, **kw)
    return model


GRAD_SAMPLE = 256        # entries kept per gradient / Adam delta
LOGIT_SAMPLE = 512       # TRAIN logits kept (valid positions)
HIST_ROWS = 48           # valid positions kept per intermediate


def _sample(a, k):
    a = np.asarray(a).reshape(-1)
    return np.ascontiguousarray(a[sample_index(a.size, k)])


def run_case(name, mode='train', float64=True, warm=5, seed=3, hp_over=None, steps_skip=0, keep_adam=False, keep_hist=False,
             gru=False):
    # gru: the cell nar_model.py:1315 keeps commented out (north_star's "session GRU").  The reference file is not edited:
    # the stand-in hands out its GRUCell when the code asks for tf.contrib.rnn.UGRNNCell - the effect of un-commenting :1315
    shim.tf.contrib.rnn.UGRNNCell = shim.GRUCell if gru else shim.UGRNNCell
    pb = make_problem('tiny', profile='B', **(hp_over or {}))
    if warm:
        warm_state(pb, warm)
    it = pb.input_fn()
    for _ in range(steps_skip):
        it.get_next()
    feats, labels = it.get_next()
    buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
    pop = pb.clicked_items_state.get_articles_recent_pop_norm().astype(np.float32)
    # pass 1: discover the variables (names, shapes, the reference's initializers)
    build(pb, feats, labels, buf, pop, mode, float64, None, seed)
    preset, stats = {}, {}
    for n, v in shim.S.vars.items():
        a = v.detach().numpy().astype(np.float64)
        stats[n] = np.array([a.mean(), a.std()])
        preset[n] = preset_variable(n, a.shape, *stats[n])   # float32 values, as a TF checkpoint would hold
    # pass 2: same sampler seed (-> same negatives), preset variables
    model = build(pb, feats, labels, buf, pop, mode, float64, preset, seed)
    S = shim.S
    out = {}
    for k, v in feats.items():
        out['feat/' + k] = np.asarray(v)
    for k, v in labels.items():
        out['label/' + k] = np.asarray(v)
    out['buffer'] = buf
    out['pop_norm'] = pop
    for n, v in S.vars.items():
        assert np.array_equal(preset[n].astype(np.float64), v.detach().numpy().astype(np.float64))
    out['reg_names'] = np.array(sorted(S.regs.keys()))
    out['var_names'] = np.array(list(S.vars.keys()))
    # row i: variable var_names[i] - initializer mean / std, shape (rank <= 2; -1 pads a rank-1 shape)
    out['var_stats'] = np.array([stats[n] for n in S.vars])
    out['var_shapes'] = np.array([list(v.shape) + [-1] * (2 - len(v.shape)) for v in S.vars.values()], dtype=np.int64)
    out['negatives'] = model.batch_negative_items.numpy()
    out['total_loss'] = np.asarray(model.total_loss.detach().numpy())
    mask = (np.arange(feats['item_clicked'].shape[1])[None, :] < (np.asarray(feats['session_size']) - 1)[:, None])
    if mode == 'train':
        out['logits_sample'] = _sample(S.softmax_inputs[0].numpy()[mask], LOGIT_SAMPLE)
    else:
        out['logits_scaled'] = S.softmax_inputs[0].numpy()
    first = {}
    for hname, t in S.hist:
        first.setdefault(hname, t)
    for hname in (KEEP_HIST if keep_hist else []):            # valid positions only (the rest never reaches the loss)
        if hname in first and first[hname].shape[:2] == mask.shape:
            h = first[hname].numpy()[mask]
            out['hist/' + hname] = np.ascontiguousarray(h[sample_index(h.shape[0], HIST_ROWS)])
    if mode == 'train':
        for n, g in S.grads.items():
            g = (g if g is not None else torch.zeros_like(S.vars[n])).detach().numpy()
            # compared at 1e-6 of the largest gradient: float32 storage suffices
            out['grad/' + n] = _sample(g.astype(np.float32), GRAD_SAMPLE)
        if keep_adam:
            for n, v in S.vars_after.items():
                out['adam_delta/' + n] = _sample((v.numpy().astype(np.float64) - S.vars[n].detach().numpy().astype(np.float64)).astype(np.float32), GRAD_SAMPLE)
    else:
        out['predicted_item_ids'] = model.predicted_item_ids.numpy()
        out['predicted_item_probs'] = model.predicted_item_probs.detach().numpy()
        out['recall_at_n'] = np.asarray(model.recall_at_n.detach().numpy())
        out['mrr_at_n'] = np.asarray(model.mrr.detach().numpy())
    if S.dropout_masks:
        # keep-masks in the order the reference applied them: input / positive / negative feature rows (nar_model.py:338,
        # :351, :367), DropoutWrapper outputs per (time step, layer) (:1330-1333), FC1 (:417)
        T, nl = feats['item_clicked'].shape[1], pb.hp.rnn_num_layers
        assert len(S.dropout_masks) == 3 + T * nl + 1
        for j, nm in enumerate(('in', 'pos', 'neg')):
            out['mask/' + nm] = np.packbits(S.dropout_masks[j].numpy())
            out['mask_shape/' + nm] = np.array(S.dropout_masks[j].shape)
        rn = torch.stack(S.dropout_masks[3:3 + T * nl]).reshape(T, nl, *S.dropout_masks[3].shape)
        out['mask/rnn'] = np.packbits(rn.numpy())
        out['mask_shape/rnn'] = np.array(rn.shape)
        out['mask/fc1'] = np.packbits(S.dropout_masks[-1].numpy())
        out['mask_shape/fc1'] = np.array(S.dropout_masks[-1].shape)
    out['meta'] = np.array([mode, 'float64' if float64 else 'float32', str(warm), repr(hp_over or {})])
    return {name + '/' + k: v for k, v in out.items()}


# intermediates the reference itself exposes through tf.summary.histogram (plot_histograms=True) that the golden file keeps.
# ("positive_user_items_features" is not among them: the reference passes the INPUT features to that histogram,
# nar_model.py:350.)
KEEP_HIST = ['user_context_features', 'input_items_features', 'input_user_items_features', 'positive_items_features',
             'input_contextual_item_embedding', 'positive_contextual_item_embedding', 'rnn/outputs', 'rnn_outputs_fc2',
             'predicted_contextual_item_embedding']


def main():
    cases = {}
    cases.update(run_case('train64', keep_adam=True, keep_hist=True))
    cases.update(run_case('train32', float64=False))
    cases.update(run_case('cold64', warm=0))                                   # empty buffer: tf.cond takes the batch statistics
    cases.update(run_case('nov64', hp_over=dict(novelty_reg_factor=0.3)))
    cases.update(run_case('layers2_64', hp_over=dict(rnn_num_layers=2)))
    # internal feature switches (nar_trainer_gcom.py:218-230): recency + ACR embeddings only
    cases.update(run_case('featoff64', hp_over=dict(enabled_internal_features=['recency', 'article_content_embeddings'])))
    cases.update(run_case('gru64', hp_over=dict(rnn_num_layers=2), gru=True))
    cases.update(run_case('drop64', hp_over=dict(dropout_keep_prob=0.8, rnn_num_layers=2)))
    cases.update(run_case('eval64', mode='eval', steps_skip=1))
    path = os.path.join(HERE, 'model_golden.npz')
    np.savez_compressed(path, **cases)
    print('wrote %d arrays, %.1f KB' % (len(cases), os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
