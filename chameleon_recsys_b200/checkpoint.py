"""Checkpoint files for the NAR training state (SURVEY.md section 8f #4).

The reference relies on ``tf.estimator.Estimator``'s ``model_dir``: every ``train()`` call restores the latest
checkpoint and writes a new one at its end (nar_trainer_gcom.py:343-349, :450-459, :511-517), so that a run can be
split across ``train`` / ``evaluate`` calls.  TF's bundle format is not reproduced; one ``.npz`` per checkpoint holds

* ``params/<tf variable name>``, ``adam_m/<...>``, ``adam_v/<...>`` - LOGICAL tensors (TF names, TF shapes, no
  layout padding / column permutation), so a checkpoint does not depend on the internal HBM layout,
* ``global_step``,
* ``state/*`` - the host-side ``ClickedItemsState`` (recent-clicks buffer, popularity counters) when given; the
  reference keeps that object alive in the trainer process instead (nar_trainer_gcom.py:486-489),
* ``baselines/*`` - the baseline recommenders' pair table (``baselines.BaselineTables.export``: occupied entries
  sorted by key, value arrays alongside) when the state holds one, and the session kNN rings under
  ``baselines/sknn_<suffix>_*`` (ids, lens, items, live in insertion order).  Checkpoints without them load as before
  (a kNN ring without saved arrays starts empty).
"""
from __future__ import annotations

import glob
import os
import re
from typing import Optional

import numpy as np

STATE_FIELDS = ('articles_pop', 'articles_recent_pop', 'articles_recent_pop_norm', 'pop_recent_clicks_buffer')


# TensorFlow names the variables of a tf.layers.Dense object after the variable scope of its FIRST call, not the scope it
# is constructed in (found by running the reference's nar_model.py: tests/golden/make_model_golden.py).  plan.ParamLayout
# uses the constructing scope; tensors exported from a real TF checkpoint under their TF names load through this table.
TF_SCOPE_ALIASES = (
    ('main/user_personalized_contextual_article_embedding/input/CAR_representation/', 'main/CAR/CAR_representation/'),
    ('main/recommendations_ranking/cos_sim_positive/matching_dense_layer_', 'main/recommendations_ranking/matching_dense_layer_'),
)


def layout_name(tf_name: str) -> str:
    """TF variable name (optionally with the ':0' tensor suffix) -> the name plan.ParamLayout uses."""
    name = tf_name[:-2] if tf_name.endswith(':0') else tf_name
    for tf_prefix, ours in TF_SCOPE_ALIASES:
        if name.startswith(tf_prefix):
            return ours + name[len(tf_prefix):]
    return name


def checkpoint_path(model_dir: str, global_step: int) -> str:
    return os.path.join(model_dir, 'model.ckpt-%d.npz' % int(global_step))


def latest_checkpoint(model_dir: Optional[str]) -> Optional[str]:
    """tf.train.latest_checkpoint: the file with the highest global step, or None."""
    if not model_dir or not os.path.isdir(model_dir):
        return None
    best, best_step = None, -1
    for p in glob.glob(os.path.join(model_dir, 'model.ckpt-*.npz')):
        m = re.search(r'model\.ckpt-(\d+)\.npz$', p)
        if m and int(m.group(1)) > best_step:
            best, best_step = p, int(m.group(1))
    return best


def save(path: str, engine, clicked_items_state=None) -> str:
    sd = engine.state_dict()
    arrays = {'global_step': np.asarray(sd['global_step'], dtype=np.int64)}
    for group in ('params', 'adam_m', 'adam_v'):
        for name, v in sd[group].items():
            arrays['%s/%s' % (group, name)] = np.asarray(v, dtype=np.float32)
    if clicked_items_state is not None:
        for f in STATE_FIELDS:
            arrays['state/' + f] = np.asarray(getattr(clicked_items_state, f))
        arrays['state/current_step'] = np.asarray(clicked_items_state.current_step, dtype=np.int64)
        tables = getattr(clicked_items_state, 'baselines', None)
        if tables is not None:
            for k, v in tables.state_arrays().items():
                arrays['baselines/' + k] = v
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    tmp = '%s.tmp%d.npz' % (path, os.getpid())      # unique per process: writers never share a temp file
    np.savez(tmp, **arrays)
    os.replace(tmp, path)                     # atomic: a reader never sees a half-written checkpoint
    return path


def load(path: str) -> dict:
    with np.load(path, allow_pickle=False) as z:
        out = {'params': {}, 'adam_m': {}, 'adam_v': {}, 'state': {}, 'baselines': {}, 'global_step': int(z['global_step'])}
        for k in z.files:
            if '/' in k:
                group, name = k.split('/', 1)
                out[group][layout_name(name) if group in ('params', 'adam_m', 'adam_v') else name] = z[k]
    return out


def restore(path: str, engine, clicked_items_state=None) -> int:
    """Load weights + TF-Adam slots + step into ``engine`` (and the host state, if both sides have it)."""
    ck = load(path)
    engine.load_state_dict({'params': ck['params'], 'adam_m': ck['adam_m'], 'adam_v': ck['adam_v'],
                            'global_step': ck['global_step']})
    if clicked_items_state is not None and ck['state']:
        for f in STATE_FIELDS:
            setattr(clicked_items_state, f, np.array(ck['state'][f]))
        clicked_items_state.current_step = int(ck['state']['current_step'])
    if clicked_items_state is not None and getattr(clicked_items_state, 'baselines', None) is not None and ck['baselines']:
        clicked_items_state.baselines.load(ck['baselines'])
    return ck['global_step']


def restore_baselines(path: str, tables) -> bool:
    """Load the baseline tables of checkpoint ``path`` into ``tables``; False (tables untouched) when it has none."""
    ck = load(path)
    if not ck['baselines']:
        return False
    tables.load(ck['baselines'])
    return True
