"""Estimator-shaped boundary of the NAR hot path (the reference's drop-in surface).

* ``nar_module_model_fn(features, labels, mode, params)`` - nar_trainer_gcom.py:234-332: picks the
  train / eval negative-sampling hparams by mode (:237-242), forces keep_prob 1 in eval (:245),
  builds ``NARModuleModel`` (:252-275) and returns an ``EstimatorSpec`` with ``loss``, ``train_op``
  and the ``ItemsStateUpdaterHook`` as training chief hook (:305-322).
* ``build_estimator`` / ``Estimator.train`` - nar_trainer_gcom.py:335-386, :511-517: the minimal
  MonitoredTrainingSession loop: hook.before_run -> train_op -> hook.after_run per batch.

Differences that are inherent to not being a TF graph: ``features``/``labels`` are numpy dicts
(one padded batch, same keys / dtypes / padding as datasets.py), ``train_op`` is a callable, and
the model object is cached across ``train()`` calls instead of being rebuilt from a checkpoint.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import numpy as np

from . import checkpoint as ckpt
from .clicked_items_state import ClickedItemsState
from .datasets import OutOfRangeError
from .hparams import ModeKeys, get_internal_enabled_features_config
from .nar_model import ItemsStateUpdaterHook, NARModuleModel

# Global vars updated by the Estimator hook (nar_trainer_gcom.py:410-415)
clicked_items_state: Optional[ClickedItemsState] = None
eval_sessions_metrics_log: list = []
sessions_negative_items_log: Optional[list] = None                # a list: log every eval session's negatives
sessions_chameleon_recommendations_log: Optional[list] = None     # a list: log every eval session's ranked candidates


@dataclass
class EstimatorSpec:
    mode: str
    loss: Optional[float] = None
    train_op: Optional[Callable] = None
    training_chief_hooks: List = field(default_factory=list)
    eval_metric_ops: Optional[dict] = None
    evaluation_hooks: List = field(default_factory=list)
    model: Optional[NARModuleModel] = None
    predictions: Optional[Callable] = None          # PREDICT: predictions(features, feed, top_n, candidates, ...) -> dict


def nar_module_model_fn(features, labels, mode, params) -> EstimatorSpec:
    if mode == ModeKeys.TRAIN:
        negative_samples = params['train_total_negative_samples']
        negative_sample_from_buffer = params['train_negative_samples_from_buffer']
    elif mode in (ModeKeys.EVAL, ModeKeys.PREDICT):
        negative_samples = params['eval_total_negative_samples']
        negative_sample_from_buffer = params['eval_negative_samples_from_buffer']
    else:
        raise ValueError('mode %r' % (mode,))
    dropout_keep_prob = params['dropout_keep_prob'] if mode == ModeKeys.TRAIN else 1.0
    internal_features_config = params.get('internal_features_config') or get_internal_enabled_features_config()
    eval_metrics_top_n = params['eval_metrics_top_n']

    model = NARModuleModel(mode, features, labels,
                           session_features_config=params['session_features_config'],
                           articles_features_config=params['articles_features_config'],
                           batch_size=params['batch_size'],
                           lr=params['lr'],
                           keep_prob=dropout_keep_prob,
                           negative_samples=negative_samples,
                           negative_sample_from_buffer=negative_sample_from_buffer,
                           reg_weight_decay=params['reg_weight_decay'],
                           softmax_temperature=params['softmax_temperature'],
                           articles_metadata=params['articles_metadata'],
                           content_article_embeddings_matrix=params['content_article_embeddings_matrix'],
                           recent_clicks_buffer_hours=params['recent_clicks_buffer_hours'],
                           recent_clicks_buffer_max_size=params['recent_clicks_buffer_max_size'],
                           recent_clicks_for_normalization=params['recent_clicks_for_normalization'],
                           CAR_embedding_size=params['CAR_embedding_size'],
                           rnn_units=params['rnn_units'],
                           rnn_num_layers=params.get('rnn_num_layers', 1),
                           metrics_top_n=eval_metrics_top_n,
                           plot_histograms=params['save_histograms'],
                           novelty_reg_factor=params['novelty_reg_factor'],
                           diversity_reg_factor=params['diversity_reg_factor'],
                           internal_features_config=internal_features_config,
                           eval_cold_start=params['eval_cold_start'],
                           elapsed_days_smooth_log_base=params.get('elapsed_days_smooth_log_base', 1.3),
                           popularity_smooth_log_base=params.get('popularity_smooth_log_base', 2.0),
                           max_cardinality_for_ohe=params.get('max_cardinality_for_ohe', 10),
                           rnn_cell=params.get('rnn_cell', 'ugrnn'), ranking=params.get('ranking', 'mlp'),
                           rnn_residual_connections=bool(params.get('rnn_residual_connections', False)),
                           sampler_seed=params.get('sampler_seed', 42), init_seed=params.get('init_seed', 42),
                           process_group=params.get('process_group'), device=params.get('device'))

    state = params.get('clicked_items_state') or clicked_items_state
    if state is None:
        raise RuntimeError('clicked_items_state is not set (nar_trainer_gcom.py:486-489 creates it before the Estimator)')
    hooks = [ItemsStateUpdaterHook(mode, model, eval_metrics_top_n=eval_metrics_top_n, clicked_items_state=state,
                                   eval_sessions_metrics_log=eval_sessions_metrics_log,
                                   sessions_negative_items_log=_first_set(
                                       params.get('sessions_negative_items_log'), sessions_negative_items_log),
                                   sessions_chameleon_recommendations_log=_first_set(
                                       params.get('sessions_chameleon_recommendations_log'),
                                       sessions_chameleon_recommendations_log),
                                   content_article_embeddings_matrix=params['content_article_embeddings_matrix'],
                                   articles_metadata=params['articles_metadata'],
                                   eval_negative_sample_relevance=params.get('eval_negative_sample_relevance'),
                                   eval_benchmark_classifiers=params.get('eval_benchmarks') or (),
                                   eval_extended_metrics=bool(params.get('eval_extended_metrics', False)),
                                   eval_metrics_by_session_position=bool(
                                       params.get('eval_metrics_by_session_position', False)),
                                   eval_unsampled_metrics=bool(params.get('eval_unsampled_metrics', False)),
                                   eval_unsampled_benchmarks=bool(params.get('eval_unsampled_benchmarks', False)))]
    if mode == ModeKeys.TRAIN:
        def train_op(feats, labs, feed, sync=True):
            return model.train(feats, labs, feed['pop_recent_items_buffer'], feed['articles_recent_pop_norm'], sync=sync)
        return EstimatorSpec(mode, loss=None, train_op=train_op, training_chief_hooks=hooks, model=model)
    if mode == ModeKeys.PREDICT:
        # one call per batch: the state arrays are read, never updated (no hook runs in PREDICT).  ``recommender``: a
        # baseline's suffix recommends with the tables on the ClickedItemsState instead of the model
        def predict(feats, feed, top_n=None, candidates=None, positions='last', exclude_session_clicks=True,
                    recommender=None):
            if recommender is not None:
                return model.recommend(feats, feed['pop_recent_items_buffer'], None, top_n=top_n, candidates=candidates,
                                       positions=positions, exclude_session_clicks=exclude_session_clicks,
                                       recommender=recommender, baselines=hooks[0].baselines,
                                       articles_pop=feed.get('articles_pop'))
            return model.recommend(feats, feed['pop_recent_items_buffer'], feed['articles_recent_pop_norm'], top_n=top_n,
                                   candidates=candidates, positions=positions, exclude_session_clicks=exclude_session_clicks)
        return EstimatorSpec(mode, loss=None, predictions=predict, model=model)

    # ModeKeys.EVAL (nar_trainer_gcom.py:323-332): loss + eval_metric_ops {hitrate_at_n, mrr_at_n}; each "update op" is
    # one call of model.evaluate, the values are read from the device accumulator at the end
    def eval_update(feats, labs, feed, metrics, step_id=None, before_sync=None):
        return model.evaluate(feats, labs, feed['pop_recent_items_buffer'], feed['articles_recent_pop_norm'],
                              metrics=metrics, step_id=step_id, before_sync=before_sync)
    return EstimatorSpec(mode, loss=None, eval_metric_ops={'hitrate_at_n': eval_update, 'mrr_at_n': eval_update},
                         evaluation_hooks=hooks, model=model)


def _first_set(a, b):
    return a if a is not None else b              # (an empty list is a log that is switched on)


class Estimator:
    """tf.estimator.Estimator stand-in: ``train(input_fn, steps=None)`` runs the hook/train_op loop."""

    def __init__(self, model_fn, params, model_dir=None, config=None):
        self.model_fn = model_fn
        self.params = params
        self.model_dir = model_dir
        self._spec: Optional[EstimatorSpec] = None
        self._eval_spec: Optional[EstimatorSpec] = None
        self.last_loss = None
        self.interactions = 0
        self.h2d_bytes_per_step = 0

    def _ensure_spec(self, features, labels) -> EstimatorSpec:
        if self._spec is None:
            self._spec = self.model_fn(features, labels, ModeKeys.TRAIN, self.params)
            latest = ckpt.latest_checkpoint(self.model_dir)          # Estimator semantics: warm-start from model_dir
            if latest is not None:
                ckpt.restore(latest, self._spec.model.engine, self._state())
        return self._spec

    def _state(self) -> Optional[ClickedItemsState]:
        return self.params.get('clicked_items_state') or clicked_items_state

    def save_checkpoint(self, path: Optional[str] = None) -> str:
        """Write weights + TF-Adam slots + global_step + ClickedItemsState (checkpoint.py); default name
        ``<model_dir>/model.ckpt-<global_step>.npz``."""
        eng = self._spec.model.engine
        if path is None:
            if not self.model_dir:
                raise ValueError('no model_dir and no path')
            path = ckpt.checkpoint_path(self.model_dir, eng.global_step)
        return ckpt.save(path, eng, self._state())

    def restore_checkpoint(self, path: str) -> int:
        return ckpt.restore(path, self._spec.model.engine, self._state())

    def train(self, input_fn, steps: Optional[int] = None, hooks=None):
        """hook.before_run -> train_op -> hook.after_run per batch (MonitoredTrainingSession), software-pipelined:
        while the GPU runs step n, the host folds batch n into ClickedItemsState (it depends on the batch's ids only,
        nar_model.py:1635-1650), fetches batch n+1 (tf.data prefetch(1), datasets.py:142) and stages it - H2D copy,
        negative sampling, row lists, normalisation statistics - on a side stream; the loss of step n is read only after
        step n+1 has been queued (two pinned loss slots, one event per step), so the GPU never waits for the host."""
        batches = _batches(input_fn(), steps)
        n = 0
        nxt = next(batches, None)
        if nxt is None:
            return self
        spec = self._ensure_spec(*nxt)
        eng = spec.model.engine
        for h in spec.training_chief_hooks:
            h.begin()
        # Device-resident ClickedItemsState (default; NAR_DEVICE_STATE=0 keeps the hook's host update + per-step upload):
        # the recent-clicks buffer / popularity live in HBM for the duration of train() and are advanced by one kernel per
        # step on the side stream (what hook.after_run does on the host, nar_model.py:1635-1650); the host object is
        # brought up to date when train() returns.
        use_ds = os.environ.get('NAR_DEVICE_STATE', '1') == '1' and self._state() is not None
        prev_st = None

        def stage_next(batch, slot, after=None):
            if use_ds:                                              # the device state absorbs prev_st first
                return eng.stage_ahead(batch[0], batch[1], None, None, slot, after=after, prev=prev_st)
            feed = {}
            for h in spec.training_chief_hooks:
                feed.update(h.before_run(None))
            return eng.stage_ahead(batch[0], batch[1], feed['pop_recent_items_buffer'], feed['articles_recent_pop_norm'],
                                   slot, after=after)

        if use_ds:
            eng.attach_device_state(self._state())
        st_next = stage_next(nxt, 'pipe0')
        pending = None                                              # (features, labels, out) of the step whose loss is unread
        # baseline recommenders (nar_model.py:1641-1646): every batch is folded into their tables (and the session kNN
        # rings, with the batch's session ids) on the side stream, behind the batch's copy; the main stream's work is
        # unchanged
        tables = getattr(self._state(), 'baselines', None)
        if tables is not None and not tables.trains:
            tables = None

        def fold(st):
            if tables is not None and st['has_clicks']:
                tables.update(st['t']['all_items'], lens=st['fold_lens'], stream=eng.side_stream(), after=st.get('copied'),
                              session_ids=st['fold_sids'])

        def finish(p):
            f_, l_, o_ = p
            o_ = eng.result(o_)                                     # waits for that step only (event), reads its loss
            spec.model._publish(f_, l_, o_)
            self.last_loss = o_.get('total_loss')
            self.interactions += int(o_['stage']['L_global'])

        while nxt is not None:
            features, labels = nxt
            if tables is not None:
                st_next['fold_lens'] = _session_clicks(features, labels)
                st_next['fold_sids'] = features.get('session_id')
            out = eng.submit(st_next)                               # step n queued on the main stream
            if not use_ds:
                fold(st_next)
            prev_st = st_next
            self.h2d_bytes_per_step = st_next['h2d_bytes']           # bytes of the one pinned H2D copy of this step
            if not use_ds:
                run_values = {'clicked_items': features['item_clicked'], 'clicked_timestamps': features['event_timestamp'],
                              'last_item_label': labels['label_last_item']}
                for h in spec.training_chief_hooks:
                    h.after_run(None, run_values)                    # host state now describes "before step n+1"
            n += 1
            nxt = next(batches, None)
            if nxt is not None:
                # slot (n & 1) was last read by step n-1 (= pending): its event gates the side-stream copy
                after = pending[2]['done'] if pending is not None else None
                st_next = stage_next(nxt, 'pipe%d' % (n & 1), after)
                if use_ds:
                    fold(prev_st)                                    # after the device state absorbed it
            elif use_ds:
                eng.advance_device_state(prev_st)                    # the last batch of this train() call
                fold(prev_st)
            if pending is not None:
                finish(pending)                                      # loss of step n-1: the GPU already runs step n
            pending = (features, labels, out)
        if pending is not None:
            finish(pending)
        if use_ds:
            eng.detach_device_state()                                # host ClickedItemsState = the device state (sync)
        for h in spec.training_chief_hooks:
            h.end()
        if self.model_dir:
            # CheckpointSaverHook at the end of train().  Data parallel: weights, Adam slots and the host state are
            # identical on every rank, so rank 0 alone writes and the others wait for the file to be complete.
            if eng.world > 1:
                import torch
                if eng.rank == 0:
                    self.save_checkpoint()
                torch.distributed.barrier(group=eng.pg)
            else:
                self.save_checkpoint()
        return self

    def _use_trained_weights(self, spec: EstimatorSpec, what: str):
        """Point the EVAL / PREDICT graph ``spec`` at the trained weights: the training graph's own (shared, no copy) when
        this Estimator has trained, else the latest checkpoint in model_dir - what tf.estimator.Estimator restores
        (nar_trainer_gcom.py:523).  Without either it raises: never serve randomly initialised weights."""
        if self._spec is not None:
            spec.model.engine.share_params(self._spec.model.engine)        # "restore the latest checkpoint"
            return
        latest = ckpt.latest_checkpoint(self.model_dir)
        if latest is None:
            raise ValueError('Estimator.%s: no trained model - call train() first or point model_dir at a '
                             'directory holding a checkpoint (model_dir=%r)' % (what, self.model_dir))
        restored = getattr(self, '_restored', {})
        if restored.get(id(spec)) != latest:
            ckpt.restore(latest, spec.model.engine, None)                   # weights + step; the state is not touched
            state = self._state()
            if state is not None and getattr(state, 'baselines', None) is not None:
                ckpt.restore_baselines(latest, state.baselines)             # what the baselines learnt with those weights
            restored[id(spec)] = latest
            self._restored = restored

    def predict(self, input_fn, steps: Optional[int] = None, top_n: Optional[int] = None, candidates=None,
                exclude_session_clicks: bool = True, positions: str = 'last', recommender: Optional[str] = None):
        """tf.estimator.Estimator.predict: a generator over the batches of ``input_fn`` that yields one dict per session -
        ``session_id``, ``predicted_item_ids`` / ``predicted_item_scores`` / ``predicted_item_probs`` [top_n] (arrays
        [n_positions, top_n] with ``positions='all'``).  The recommendation is for the article after the session's last
        valid position (``label_last_item`` on an input_fn batch).  ``top_n`` defaults to eval_metrics_top_n;
        ``candidates``: None = the distinct ids of the current recent-clicks buffer, 'catalog' = every article, or an array
        of ids.  Weights as ``evaluate`` gets them; ClickedItemsState, weights, Adam slots and global_step are only read.
        Data parallel (``params['process_group']``): every rank runs the same ``input_fn`` and arguments, scores its share
        of each batch's sessions (NarEngine.recommend) and yields the same dicts as one process.
        ``recommender``: the suffix of one baseline of ``params['eval_benchmarks']`` recommends instead of the model
        (DESIGN.md section 16), with what it learnt in this Estimator's training or, without one, in the latest
        checkpoint: the first top_n ids of the valid set it admits, in its own order; ``predicted_item_scores`` are float64
        and its own scores, id 0 and NaN pad past the admissible ids, and there is no ``predicted_item_probs``.  One
        process only (NotImplementedError data parallel)."""
        import torch
        if positions not in ('last', 'all'):
            raise ValueError("positions must be 'last' or 'all', not %r" % (positions,))
        if recommender is not None:
            from .baselines import SUFFIXES, parse_classifiers
            from .sknn import KNN_SUFFIXES
            if recommender not in SUFFIXES + KNN_SUFFIXES:
                raise ValueError('unknown baseline recommender %r (expected one of %s)'
                                 % (recommender, ', '.join(SUFFIXES + KNN_SUFFIXES)))
            enabled = list(parse_classifiers(self.params.get('eval_benchmarks') or ()))
            if recommender not in enabled:
                raise ValueError('baseline %r is not one of eval_benchmarks (%s)'
                                 % (recommender, ', '.join(enabled) if enabled else 'none'))
            pg = self.params.get('process_group')
            if pg is not None and torch.distributed.get_world_size(pg) > 1:
                raise NotImplementedError('baseline recommenders run on one process; data-parallel prediction with a '
                                          'baseline is not implemented')
        for n, (features, labels) in enumerate(_batches(input_fn(), steps)):
            if getattr(self, '_predict_spec', None) is None:
                self._predict_spec = self.model_fn(features, labels, ModeKeys.PREDICT, self.params)
            spec = self._predict_spec
            if n == 0:
                self._use_trained_weights(spec, 'predict')
            state = self._state()
            feed = {'pop_recent_items_buffer': state.get_recent_clicks_buffer(),
                    'articles_recent_pop_norm': state.get_articles_recent_pop_norm()}
            if recommender is not None:
                feed['articles_pop'] = state.get_articles_pop()
                out = spec.predictions(features, feed, top_n=top_n, candidates=candidates, positions=positions,
                                       exclude_session_clicks=exclude_session_clicks, recommender=recommender)
            else:
                out = spec.predictions(features, feed, top_n=top_n, candidates=candidates, positions=positions,
                                       exclude_session_clicks=exclude_session_clicks)
            sids = features.get('session_id')
            Bg = np.asarray(features['item_clicked']).shape[0]
            qs = out['query_session']
            for b in range(Bg):
                rows = np.flatnonzero(qs == b)
                sel = rows[0] if (positions == 'last' and rows.size) else rows
                row = {'session_id': None if sids is None else np.asarray(sids)[b],
                       'predicted_item_ids': out['predicted_item_ids'][sel],
                       'predicted_item_scores': out['predicted_item_scores'][sel]}
                if recommender is None:
                    row['predicted_item_probs'] = out['predicted_item_probs'][sel]
                yield row
        torch.cuda.synchronize()

    def evaluate(self, input_fn, steps: Optional[int] = None, hooks=None, name=None) -> dict:
        """tf.estimator.Estimator.evaluate: runs the EVAL graph over ``input_fn`` with the current weights and returns
        ``{'loss', 'hitrate_at_n', 'mrr_at_n', 'global_step'}`` (streaming means over all valid labels, nar_model.py:
        835-885; ``loss`` = mean of the per-batch total_loss like Estimator does).  The hook snapshots ClickedItemsState at
        ``begin`` and restores it at ``end`` (nar_model.py:1415, :1693), and keeps updating it batch by batch in between.
        With ``eval_extended_metrics`` also ``ndcg_at_n``, ``item_coverage_at_n``, ``esi-r_at_n``, ``esi-rr_at_n``,
        ``content_eild-r_at_n`` and ``content_eild-rr_at_n``, and each as ``<key>_<suffix>`` for every baseline.  With
        ``eval_metrics_by_session_position`` also ``hitrate_at_n_by_pos_PP``, ``clicks_at_pos_PP`` and
        ``avg_norm_pop_by_pos_PP`` of the model and ``hitrate_at_n_by_pos_<suffix>_PP`` of every baseline, for each
        session position PP ('%02d', from 01) that had a query (none without input).  With ``eval_unsampled_metrics``
        also ``unsampled_hitrate_at_n``, ``unsampled_mrr_at_n``, ``unsampled_ndcg_at_n`` and
        ``unsampled_candidates_per_query``: each label ranked against every article the negative sampler could have drawn
        for it (DESIGN.md section 13; NaN without input).  With ``eval_unsampled_benchmarks`` also
        ``unsampled_hitrate_at_n_<suffix>``, ``unsampled_mrr_at_n_<suffix>`` and ``unsampled_ndcg_at_n_<suffix>`` of every
        baseline and ``unsampled_candidates_per_query``, against the same competitors (DESIGN.md section 14)."""
        import torch
        batches = _batches(input_fn(), steps)
        nxt = next(batches, None)
        if nxt is None:
            empty = {'loss': float('nan'), 'hitrate_at_n': float('nan'), 'mrr_at_n': float('nan'),
                     'global_step': 0 if self._spec is None else self._spec.model.global_step()}
            if self.params.get('eval_extended_metrics'):
                from .baselines import parse_classifiers
                from .eval_metrics import metric_names
                for s in [''] + list(parse_classifiers(self.params.get('eval_benchmarks') or ())):
                    empty.update({k: float('nan') for k in metric_names(s)})
            if self.params.get('eval_unsampled_metrics'):
                from .eval_metrics import UNSAMPLED_KEYS
                empty.update({k: float('nan') for k in UNSAMPLED_KEYS})
            if self.params.get('eval_unsampled_benchmarks'):
                from .baselines import parse_classifiers
                from .eval_metrics import unsampled_bench_keys
                if not self.params.get('eval_benchmarks'):
                    raise ValueError('eval_unsampled_benchmarks ranks the baselines of eval_benchmarks, and none is set')
                for s in parse_classifiers(self.params.get('eval_benchmarks') or ()):
                    empty.update({k: float('nan') for k in unsampled_bench_keys(s)})
                empty['unsampled_candidates_per_query'] = float('nan')
            return empty
        if self._eval_spec is None:
            self._eval_spec = self.model_fn(nxt[0], nxt[1], ModeKeys.EVAL, self.params)
        spec = self._eval_spec
        self._use_trained_weights(spec, 'evaluate')
        for h in spec.evaluation_hooks:
            h.begin()
        metrics = torch.zeros(3, device=spec.model.engine.dev, dtype=torch.float64)
        update = spec.eval_metric_ops['hitrate_at_n']
        n, loss_sum = 0, 0.0
        # per-session logs: the previous batch's pinned copy becomes list entries while the GPU runs this batch
        logs = [h.session_logs for h in spec.evaluation_hooks if getattr(h, 'session_logs', None) is not None]
        overlap = {'before_sync': lambda: [sl.drain() for sl in logs]} if logs else {}
        while nxt is not None:
            features, labels = nxt
            feed = {}
            for h in spec.evaluation_hooks:
                feed.update(h.before_run(None))
            out = update(features, labels, feed, metrics, step_id=n + 1, **overlap)
            run_values = {'clicked_items': features['item_clicked'], 'clicked_timestamps': features['event_timestamp'],
                          'last_item_label': labels['label_last_item'], 'stage': out['stage'],
                          'eval_batch_negative_items': out['negatives'], 'session_ids': features.get('session_id'),
                          'predicted_item_ids': out.get('predicted_item_ids'),
                          'predicted_item_probs': out.get('predicted_item_probs')}
            for h in spec.evaluation_hooks:
                h.after_run(None, run_values)
            loss_sum += out['total_loss']
            n += 1
            nxt = next(batches, None)
        bench = {}
        for h in spec.evaluation_hooks:
            bench.update(h.benchmark_results())
            bench.update(h.extended_results())
            bench.update(h.by_position_results())
            bench.update(h.unsampled_results())
            bench.update(h.unsampled_benchmark_results())
            h.end()
        eng = spec.model.engine
        if eng.world > 1:                                           # data parallel: every rank ranked its own sessions
            torch.distributed.all_reduce(metrics, group=eng.pg)
        m = metrics.cpu().numpy()
        cnt = max(float(m[2]), 1.0)
        return {'loss': loss_sum / max(n, 1), 'hitrate_at_n': float(m[0]) / cnt, 'mrr_at_n': float(m[1]) / cnt,
                'global_step': spec.model.global_step(), **bench}

    @property
    def model(self) -> Optional[NARModuleModel]:
        return None if self._spec is None else self._spec.model


def _batches(it, steps: Optional[int]):
    """(features, labels) from the input_fn iterator ``it`` until it runs out or ``steps`` batches were taken (None: all)."""
    n = 0
    while steps is None or n < steps:
        try:
            batch = it.get_next() if hasattr(it, 'get_next') else next(it)
        except (OutOfRangeError, StopIteration):
            return
        yield batch
        n += 1


def _session_clicks(features, labels) -> np.ndarray:
    """Nonzero clicks of every session of concat(item_clicked, label_last_item) (the baselines' growth bound)."""
    ic = np.asarray(features['item_clicked'])
    return np.count_nonzero(ic, axis=1) + (np.asarray(labels['label_last_item']).reshape(-1) != 0)


def build_estimator(model_dir, content_article_embeddings_matrix, articles_metadata, articles_features_config,
                    session_features_config, hparams, state: ClickedItemsState, **extra) -> Estimator:
    """nar_trainer_gcom.py:335-386 with the flags carried by ``hparams`` (NARHParams)."""
    params = hparams.to_params(session_features_config, articles_features_config, articles_metadata,
                               content_article_embeddings_matrix)
    params['clicked_items_state'] = state
    params.update(extra)
    return Estimator(model_fn=nar_module_model_fn, params=params, model_dir=model_dir)
