"""Generate tests/golden/model_fn_golden.json: the REFERENCE's nar_module_model_fn (nar_trainer_gcom.py:234-332, imported
unmodified on the TF-API stand-in) is called with the ``params`` dict THIS repo builds (NARHParams.to_params, what
chameleon_recsys_b200.estimator.build_estimator hands to its own model_fn) - TRAIN and EVAL - and with the reference's
ClickedItemsState.  It must accept the dict (every key it reads exists under the reference's name), pick the train / eval
sampling sizes, force keep_prob to 1 in EVAL, build the hook, and produce the same loss as the direct constructor call of
tests/golden/make_model_golden.py on the same batch / variables / sampler seed.  Run once in the build container."""
import importlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import tf1_shim as shim  # noqa: E402
import pandas  # noqa: E402,F401
import google  # noqa: E402

sys.modules.setdefault('pytz', types.ModuleType('pytz'))
_ua = types.ModuleType('ua_parser')
_ua.user_agent_parser = types.ModuleType('ua_parser.user_agent_parser')
sys.modules.setdefault('ua_parser', _ua)
sys.modules.setdefault('ua_parser.user_agent_parser', _ua.user_agent_parser)
_gc = types.ModuleType('google.cloud')                    # gcs_utils.py imports google.cloud.storage (uploads; unused here)
_gc.storage = types.ModuleType('google.cloud.storage')
sys.modules['google.cloud'] = _gc
sys.modules['google.cloud.storage'] = _gc.storage
google.cloud = _gc
pkg = types.ModuleType('refnar')
pkg.__path__ = ['/root/reference/nar_module/nar']
sys.modules['refnar'] = pkg
trainer = importlib.import_module('refnar.nar_trainer_gcom')
ref_state = importlib.import_module('refnar.clicked_items_state')

import torch  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from oracle.golden_sampling import preset_variables  # noqa: E402

torch.set_num_threads(1)
golden = np.load(os.path.join(HERE, 'model_golden.npz'))
out = {}
for mode, case, skip in (('train', 'train64', 0), ('eval', 'eval64', 1)):
    pb = make_problem('tiny', profile='B')
    warm_state(pb, 5)
    it = pb.input_fn()
    for _ in range(skip):
        it.get_next()
    feats, labels = it.get_next()
    assert np.array_equal(feats['item_clicked'], golden[case + '/feat/item_clicked'])
    hp = pb.hp
    params = hp.to_params(pb.session_features_config, pb.articles_features_config, pb.articles_metadata,
                          pb.content_article_embeddings_matrix)
    # the reference state object, brought to the same state as the harness's
    st = ref_state.ClickedItemsState(hp.recent_clicks_buffer_hours, hp.recent_clicks_buffer_max_size,
                                     hp.recent_clicks_for_normalization, pb.plan.num_items)
    st.pop_recent_clicks_buffer = np.array(pb.clicked_items_state.pop_recent_clicks_buffer)
    st.articles_recent_pop_norm = np.array(pb.clicked_items_state.get_articles_recent_pop_norm())
    trainer.clicked_items_state = st
    trainer.FLAGS.disable_eval_benchmarks = True
    trainer.FLAGS.enabled_internal_features = [trainer.ALL_FEATURES]
    preset = preset_variables(golden, 'train64')
    shim.configure(float64=True, seed=3, preset=preset, feeds={
        'articles_metadata': [pb.articles_metadata[k] for k in pb.articles_metadata],
        'content_article_embeddings_matrix': pb.content_article_embeddings_matrix,
        'articles_recent_pop_norm': st.get_articles_recent_pop_norm().astype(np.float32),
        'pop_recent_items_buffer': st.get_recent_clicks_buffer()})
    spec = trainer.nar_module_model_fn({k: shim._t(np.asarray(v)) for k, v in feats.items()},
                                       {k: shim._t(np.asarray(v)) for k, v in labels.items()}, mode, params)
    loss = float(spec.loss.detach())
    ref_loss = float(golden[case + '/total_loss'])
    assert abs(loss - ref_loss) < 1e-12 * abs(ref_loss), (mode, loss, ref_loss)
    hooks = spec.training_chief_hooks if mode == 'train' else spec.evaluation_hooks
    assert len(hooks) == 1 and type(hooks[0]).__name__ == 'ItemsStateUpdaterHook' and hooks[0].clicked_items_state is st
    out[mode] = {'loss': loss, 'golden_case': case, 'params_keys_passed': sorted(k for k in params if k != 'clicked_items_state'),
                 'eval_metric_ops': sorted(spec.eval_metric_ops) if spec.eval_metric_ops else None,
                 'negatives_shape': list(hooks[0].model.batch_negative_items.shape)}
# the trainer's feature / internal-feature configuration builders (nar_trainer_gcom.py:99-231) under a few flag settings
cfgs = []
for clicks, arts, internal in (([trainer.ALL_FEATURES], [trainer.ALL_FEATURES], [trainer.ALL_FEATURES]),
                               (['time', 'location'], ['category'], ['recency', 'article_content_embeddings']),
                               (['device'], [], ['novelty', 'item_clicked_embeddings', 'bogus'])):
    trainer.FLAGS.enabled_clicks_input_features_groups = clicks
    trainer.FLAGS.enabled_articles_input_features_groups = arts
    trainer.FLAGS.enabled_internal_features = internal
    cfgs.append({'flags': [clicks, arts, internal], 'session': trainer.get_session_features_config(),
                 'articles': trainer.get_articles_features_config(), 'internal': trainer.get_internal_enabled_features_config()})
out['feature_configs'] = cfgs
with open(os.path.join(HERE, 'model_fn_golden.json'), 'w') as f:
    json.dump(out, f, indent=1)
print(json.dumps({m: {k: v for k, v in o.items() if k != 'params_keys_passed'} for m, o in out.items() if m != 'feature_configs'}))
