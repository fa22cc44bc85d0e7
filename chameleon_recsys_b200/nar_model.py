"""``NARModuleModel`` and ``ItemsStateUpdaterHook`` - the reference's model-side API
(nar_module/nar/nar_model.py:100-129 ctor, :1370-1470 / :1504-1511 / :1635-1650 hook) on top of
the H100 engine.

TF builds a symbolic graph per ``model_fn`` call and the hook feeds placeholders per step; here
the object is built once (weights + ACR table resident in HBM) and ``run(features, labels)``
plays the role of one ``session.run(train_op)``.  Attribute names the hook fetches in the
reference (``item_clicked``, ``event_timestamp``, ``next_item_label``, ``label_last_item``,
``session_id``, ``user_id``, ``batch_negative_items``, ``total_loss``, ``train``) are kept.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from .clicked_items_state import ClickedItemsState, batch_clicks_for_state_update
from .hparams import ModeKeys
from .plan import FeaturePlan, ParamLayout


class NARModuleModel:

    def __init__(self, mode, inputs, labels,
                 session_features_config,
                 articles_features_config,
                 batch_size,
                 lr, keep_prob, negative_samples, negative_sample_from_buffer,
                 content_article_embeddings_matrix,
                 rnn_num_layers=1,
                 softmax_temperature=1.0,
                 reg_weight_decay=0.0,
                 recent_clicks_buffer_hours=1.0,
                 recent_clicks_buffer_max_size=1000,
                 recent_clicks_for_normalization=1000,
                 articles_metadata=None,
                 plot_histograms=False,
                 metrics_top_n=5,
                 elapsed_days_smooth_log_base=1.3,
                 popularity_smooth_log_base=2.0,
                 CAR_embedding_size=256,
                 rnn_units=256,
                 max_cardinality_for_ohe=10,
                 novelty_reg_factor=0.0,
                 diversity_reg_factor=0.0,
                 internal_features_config={'recency': True,
                                           'novelty': True,
                                           'article_content_embeddings': True,
                                           'item_clicked_embeddings': True},
                 eval_cold_start=False,
                 # --- extensions (not in the reference signature) ---
                 rnn_cell='ugrnn', ranking='mlp', sampler_seed=42, init_seed=42, device=None,
                 process_group=None, fwd_precision=4, bwd_precision=1, rnn_residual_connections=False):
        from .engine import NarEngine          # imports torch + the CUDA library; fails loudly without them
        self.mode = mode
        self.lr = lr
        self.keep_prob = keep_prob
        self.is_training = (mode == ModeKeys.TRAIN)
        self.negative_samples = negative_samples
        self.negative_sample_from_buffer = negative_sample_from_buffer
        self.rnn_num_layers = rnn_num_layers
        self.metrics_top_n = metrics_top_n
        self.reg_weight_decay = reg_weight_decay
        self.batch_size = batch_size
        self.session_features_config = session_features_config
        self.articles_features_config = articles_features_config
        self.internal_features_config = internal_features_config
        self.items_vocab_size = articles_features_config['article_id']['cardinality']
        self.content_article_embeddings_matrix = content_article_embeddings_matrix
        self.articles_metadata = articles_metadata
        self.plan = FeaturePlan(session_features_config, articles_features_config, internal_features_config,
                                max_cardinality_for_ohe, content_article_embeddings_matrix.shape[1],
                                self.items_vocab_size)
        self.layout = ParamLayout(self.plan, CAR_embedding_size, rnn_units, rnn_num_layers, rnn_cell=rnn_cell,
                                  residual=rnn_residual_connections)
        self.engine = NarEngine(self.plan, self.layout, content_article_embeddings_matrix, articles_metadata,
                                negative_samples=negative_samples,
                                negative_sample_from_buffer=negative_sample_from_buffer,
                                softmax_temperature=softmax_temperature, reg_weight_decay=reg_weight_decay, lr=lr,
                                recent_clicks_buffer_max_size=recent_clicks_buffer_max_size,
                                recent_clicks_for_normalization=recent_clicks_for_normalization,
                                elapsed_days_smooth_log_base=elapsed_days_smooth_log_base,
                                popularity_smooth_log_base=popularity_smooth_log_base, ranking=ranking,
                                rnn_cell=rnn_cell, rnn_residual=rnn_residual_connections,
                                sampler_seed=sampler_seed, device=device,
                                process_group=process_group, fwd_precision=fwd_precision,
                                bwd_precision=bwd_precision,
                                keep_prob=keep_prob if mode == ModeKeys.TRAIN else 1.0,
                                novelty_reg_factor=novelty_reg_factor)
        self.engine.set_params(self.layout.init_logical(init_seed))
        # fetch targets of the reference hook (numpy after each run)
        self.item_clicked = None
        self.event_timestamp = None
        self.next_item_label = None
        self.label_last_item = None
        self.session_id = None
        self.user_id = None
        self.batch_negative_items = None
        self.total_loss = None
        self.predicted_item_ids = None
        self.predicted_item_probs = None
        self._features = inputs
        self._labels = labels
        self._last = None

    # ``train`` is the train_op: call it with the hook's feed (state arrays) to run one step
    def train(self, features: Dict[str, np.ndarray], labels: Dict[str, np.ndarray], pop_recent_items_buffer: np.ndarray,
              articles_recent_pop_norm: np.ndarray, sync: bool = True) -> dict:
        out = self.engine.train_step(features, labels, pop_recent_items_buffer, articles_recent_pop_norm, sync=sync)
        self._publish(features, labels, out)
        return out

    def evaluate(self, features: Dict[str, np.ndarray], labels: Dict[str, np.ndarray], pop_recent_items_buffer: np.ndarray,
                 articles_recent_pop_norm: np.ndarray, metrics=None, step_id=None, before_sync=None) -> dict:
        """One EVAL batch (the eval_metric_ops update): loss, ``predicted_item_ids`` / ``predicted_item_probs``
        (nar_model.py:520-524) and the HR@n / MRR@n accumulators (:835-885) for ``metrics_top_n``."""
        out = self.engine.eval_step(features, labels, pop_recent_items_buffer, articles_recent_pop_norm,
                                    top_n=self.metrics_top_n, metrics=metrics, step_id=step_id, before_sync=before_sync)
        self._publish(features, labels, out)
        self.predicted_item_ids = out.get('predicted_item_ids')
        self.predicted_item_probs = out.get('predicted_item_probs')
        return out

    def recommend(self, features: Dict[str, np.ndarray], pop_recent_items_buffer: np.ndarray,
                  articles_recent_pop_norm: np.ndarray, top_n: Optional[int] = None, candidates=None, positions: str = 'last',
                  exclude_session_clicks: bool = True, recommender: Optional[str] = None, baselines=None,
                  articles_pop=None) -> dict:
        """Top-n next-article recommendations for the batch ``features`` (NarEngine.recommend): ``top_n`` defaults to
        ``metrics_top_n``; ``candidates`` None = the recent-clicks buffer's distinct ids, 'catalog' = every article, or an
        array of ids.  Reads the weights and the given state; changes neither.  ``recommender``: the suffix of one
        baseline of ``baselines`` (the BaselineTables of the ClickedItemsState) recommends instead of the model
        (recommend_baseline)."""
        if recommender is not None:
            return self.recommend_baseline(recommender, baselines, features, pop_recent_items_buffer, articles_pop,
                                           top_n=top_n, candidates=candidates, positions=positions,
                                           exclude_session_clicks=exclude_session_clicks)
        return self.engine.recommend(features, pop_recent_items_buffer, articles_recent_pop_norm,
                                     self.metrics_top_n if top_n is None else top_n, candidates=candidates,
                                     positions=positions, exclude_session_clicks=exclude_session_clicks)

    def recommend_baseline(self, recommender: str, baselines, features: Dict[str, np.ndarray],
                           pop_recent_items_buffer: np.ndarray, articles_pop: Optional[np.ndarray], top_n: Optional[int] = None,
                           candidates=None, positions: str = 'last', exclude_session_clicks: bool = True) -> dict:
        """Top-n recommendations of the baseline ``recommender`` (DESIGN.md section 16) for the queries and candidates
        ``recommend`` would use: the first ``top_n`` admissible ids of each query's valid set in the baseline's order
        (BaselineTables.recommend), with the popularity baseline counting ``pop_recent_items_buffer`` and item_knn
        normalising with ``articles_pop``.  Every argument is checked before any launch.  Reads the tables; changes
        nothing.  -> numpy dict: query_session [Q], query_position [Q], predicted_item_ids [Q, top_n] int64,
        predicted_item_scores [Q, top_n] float64 (the baseline's own scores; id 0 and NaN past the admissible ids),
        candidates [N] (ascending)."""
        import torch
        from .baselines import SUFFIXES, BaselineTables
        from .dp import session_lengths
        from .sknn import KNN_SUFFIXES, MAX_T as MAX_KNN_T
        if recommender not in SUFFIXES + KNN_SUFFIXES:
            raise ValueError('unknown baseline recommender %r (expected one of %s)'
                             % (recommender, ', '.join(SUFFIXES + KNN_SUFFIXES)))
        if baselines is None or recommender not in baselines.enabled:
            raise ValueError('baseline %r is not one of eval_benchmarks (%s)'
                             % (recommender, ', '.join(baselines.enabled) if baselines is not None else 'none'))
        if self.engine.world > 1:
            raise NotImplementedError('baseline recommenders run on one process; data-parallel prediction with a baseline '
                                      'is not implemented')
        if positions not in ('last', 'all'):
            raise ValueError("positions must be 'last' or 'all', not %r" % (positions,))
        if pop_recent_items_buffer is None:
            raise ValueError('recommend needs the host recent-clicks buffer')
        if recommender == 'item_knn' and articles_pop is None:
            raise ValueError("the 'item_knn' baseline needs the articles' popularity")
        cand = np.sort(self.engine.resolve_candidates(candidates, pop_recent_items_buffer))
        N = int(cand.size)
        top_n = self.metrics_top_n if top_n is None else top_n
        if isinstance(top_n, (bool, np.bool_)) or not isinstance(top_n, (int, np.integer)):
            raise ValueError('top_n must be an integer')
        top_n = int(top_n)
        if not 1 <= top_n <= min(N, BaselineTables.MAX_TOP_N):
            raise ValueError('top_n=%d outside [1, min(N=%d, %d)]' % (top_n, N, BaselineTables.MAX_TOP_N))
        item_clicked = np.asarray(features['item_clicked'], dtype=np.int64)
        Bg, T = item_clicked.shape
        limit = MAX_KNN_T if recommender in KNN_SUFFIXES else BaselineTables.MAX_T
        if T > limit:
            raise ValueError('baseline %r recommends for sessions of at most %d positions, not %d' % (recommender, limit, T))
        lens_g = session_lengths(features['session_size'], T)
        if positions == 'last':
            q_sess = np.flatnonzero(lens_g > 0).astype(np.int64)
            q_t = (lens_g[lens_g > 0] - 1).astype(np.int64)
        else:
            q_sess = np.repeat(np.arange(Bg, dtype=np.int64), lens_g)
            q_t = np.arange(q_sess.size, dtype=np.int64) - np.repeat(np.cumsum(lens_g) - lens_g, lens_g)
        out = {'query_session': q_sess, 'query_position': q_t, 'candidates': cand,
               'predicted_item_ids': np.zeros((q_sess.size, top_n), np.int64),
               'predicted_item_scores': np.full((q_sess.size, top_n), np.nan)}
        if q_sess.size == 0:
            return out
        d = baselines.dev
        ids, scores = baselines.recommend(recommender, torch.from_numpy(item_clicked).to(d),
                                          torch.from_numpy((q_sess * T + q_t).astype(np.int32)).to(d),
                                          torch.from_numpy(cand).to(d), pop_recent_items_buffer, articles_pop, top_n,
                                          exclude_session_clicks=exclude_session_clicks)
        baselines.check_errors()
        out['predicted_item_ids'] = ids.cpu().numpy()
        out['predicted_item_scores'] = scores.cpu().numpy()
        return out

    def _publish(self, features, labels, out):
        self.item_clicked = features['item_clicked']
        self.event_timestamp = features['event_timestamp'][..., None]
        self.next_item_label = labels['label_next_item']
        self.label_last_item = labels['label_last_item']
        self.session_id = features.get('session_id')
        self.user_id = features.get('user_id')
        self.batch_negative_items = out['negatives']        # device tensor [B,T,K] int64
        self.total_loss = out.get('total_loss')
        self._last = out

    def global_step(self) -> int:
        return self.engine.global_step


class ItemsStateUpdaterHook:
    """Train-mode parts of the reference SessionRunHook (nar_model.py:1370-1470, :1635-1650):
    ``before_run`` hands the per-step host state to the graph (the 46 MB ACR matrix is NOT re-fed:
    it lives in HBM), ``after_run`` folds the batch's clicks back into ``ClickedItemsState``."""

    def __init__(self, mode, model: NARModuleModel, eval_metrics_top_n, clicked_items_state: ClickedItemsState,
                 eval_sessions_metrics_log=None, sessions_negative_items_log=None,
                 sessions_chameleon_recommendations_log=None, content_article_embeddings_matrix=None,
                 articles_metadata=None, eval_negative_sample_relevance=None, eval_benchmark_classifiers=(),
                 eval_metrics_by_session_position=False, eval_cold_start=False, eval_extended_metrics=False,
                 eval_unsampled_metrics=False, eval_unsampled_benchmarks=False):
        self.mode = mode
        self.model = model
        self.eval_metrics_top_n = eval_metrics_top_n
        self.clicked_items_state = clicked_items_state
        self.eval_sessions_metrics_log = eval_sessions_metrics_log
        # the per-session logs (nar_model.py:1529-1581): each is on iff its list was given; a session_logs.SessionLogs
        # object packs them on the GPU and appends to the lists
        self.sessions_negative_items_log = sessions_negative_items_log
        self.sessions_chameleon_recommendations_log = sessions_chameleon_recommendations_log
        self.session_logs_on = mode == ModeKeys.EVAL and (sessions_negative_items_log is not None or
                                                          sessions_chameleon_recommendations_log is not None)
        self.session_logs = None
        if self.session_logs_on and model.engine.world > 1:
            raise NotImplementedError('the per-session evaluation logs run on one process; data-parallel evaluation of '
                                      'them is not implemented')
        # NDCG, coverage, novelty and diversity of the model and every baseline (create_eval_metrics, nar_model.py:
        # 1696-1721): an eval_metrics.EvalMetrics accumulator, row 0 the model, rows 1.. the baselines' rows
        self.eval_negative_sample_relevance = eval_negative_sample_relevance
        self.extended_metrics = eval_extended_metrics and mode == ModeKeys.EVAL
        self.extended = None
        if self.extended_metrics:
            from .eval_metrics import check_params
            if model.engine.world > 1:
                raise NotImplementedError('the extended evaluation metrics run on one process; data-parallel evaluation '
                                          'of them is not implemented')
            check_params(eval_metrics_top_n, eval_negative_sample_relevance)
        # hit rate by session position of the model and every baseline (nar_model.py:1718-1719): an
        # eval_metrics.ByPosition accumulator with the same rows
        self.by_position_on = eval_metrics_by_session_position and mode == ModeKeys.EVAL
        self.by_position = None
        if self.by_position_on:
            from .eval_metrics import check_by_position_params
            if model.engine.world > 1:
                raise NotImplementedError('the hit rate by session position runs on one process; data-parallel '
                                          'evaluation of it is not implemented')
            check_by_position_params(eval_metrics_top_n)
        # hit rate, MRR and NDCG of each label against every article the negative sampler could have drawn for it
        # (NarEngine.rank_labels): an int64 rank histogram [top_n + 2] on the device, read once at the end
        self.unsampled_on = eval_unsampled_metrics and mode == ModeKeys.EVAL
        self.unsampled_hist = None
        if self.unsampled_on and model.engine.world > 1:
            raise NotImplementedError('the unsampled evaluation metrics run on one process; data-parallel evaluation of '
                                      'them is not implemented')
        # the same for every baseline (BaselineTables.rank_unsampled): an int64 histogram [n_rows, top_n + 2]
        self.unsampled_bench_on = eval_unsampled_benchmarks and mode == ModeKeys.EVAL
        self.unsampled_bench_hist = None
        if self.unsampled_bench_on:
            if model.engine.world > 1:
                raise NotImplementedError('the unsampled evaluation of the baselines runs on one process; data-parallel '
                                          'evaluation of it is not implemented')
            if not eval_benchmark_classifiers:
                raise ValueError('eval_unsampled_benchmarks ranks the baselines of eval_benchmarks, and none is set')
        # baseline recommenders (nar_model.py:1399-1407): [{'recommender': <suffix>, 'params': {...}}]; their state is the
        # BaselineTables object on the ClickedItemsState, shared by the TRAIN and EVAL hooks
        self.bench_metrics = None
        self.baselines = None
        if eval_benchmark_classifiers:
            from .baselines import BaselineTables, parse_classifiers
            wanted = parse_classifiers(eval_benchmark_classifiers)
            eng = model.engine
            if eng.world > 1:
                raise NotImplementedError('baseline recommenders run on one process; data-parallel evaluation of the '
                                          'baselines is not implemented')
            tables = clicked_items_state.baselines
            if tables is None:
                tables = BaselineTables(eval_benchmark_classifiers, clicked_items_state.num_items, acr=eng.acr,
                                        acr_dim=model.plan.acr_dim, device=eng.dev.index)
                clicked_items_state.baselines = tables
            elif tables.params != wanted:
                raise ValueError('ClickedItemsState already holds baselines %r, not %r' % (tables.params, wanted))
            self.baselines = tables

    def begin(self):
        if self.mode == ModeKeys.EVAL:
            self.clicked_items_state.save_state_checkpoint()        # nar_model.py:1415
            if self.unsampled_on:
                import torch
                self.unsampled_hist = torch.zeros(self.eval_metrics_top_n + 2, dtype=torch.int64,
                                                  device=self.model.engine.dev)
            if self.baselines is not None:
                import torch
                self.bench_metrics = torch.zeros(self.baselines.n_rows, 3, dtype=torch.float64, device=self.model.engine.dev)
                if self.unsampled_bench_on:
                    self.unsampled_bench_hist = torch.zeros(self.baselines.n_rows, self.eval_metrics_top_n + 2,
                                                            dtype=torch.int64, device=self.model.engine.dev)
            if self.extended_metrics:
                if self.extended is None:
                    from .eval_metrics import EvalMetrics
                    eng, tables = self.model.engine, self.baselines
                    self.extended = EvalMetrics(1 + (tables.n_rows if tables is not None else 0),
                                                self.clicked_items_state.num_items, eng.acr, self.model.plan.acr_dim,
                                                self.eval_metrics_top_n, self.eval_negative_sample_relevance,
                                                acr_norm=None if tables is None else tables.acr_norm)
                self.extended.begin(self.clicked_items_state.get_recent_clicks_buffer())
            if self.by_position_on:
                if self.by_position is None:
                    from .eval_metrics import ByPosition
                    self.by_position = ByPosition(1 + (self.baselines.n_rows if self.baselines is not None else 0),
                                                  self.clicked_items_state.num_items, self.eval_metrics_top_n,
                                                  self.model.engine.dev)
                self.by_position.begin()
            if self.session_logs_on:
                if self.session_logs is None:
                    from .session_logs import SessionLogs
                    self.session_logs = SessionLogs(self.clicked_items_state.num_items, self.model.engine.dev,
                                                    self.sessions_negative_items_log,
                                                    self.sessions_chameleon_recommendations_log)
                self.session_logs.begin()

    def before_run(self, run_context=None) -> dict:
        """-> feed dict (nar_model.py:1458-1467)."""
        return {'articles_recent_pop_norm': self.clicked_items_state.get_articles_recent_pop_norm(),
                'pop_recent_items_buffer': self.clicked_items_state.get_recent_clicks_buffer()}

    def after_run(self, run_context, run_values: dict):
        """run_values: {'clicked_items','clicked_timestamps','last_item_label'} (nar_model.py:1505-1508).  In EVAL with
        baselines enabled also 'stage' (the staged batch of the step), 'eval_batch_negative_items' ([B,T,K] device) and
        'session_ids' ([B], needed by the session kNN baselines): the baselines rank the batch against the state BEFORE
        it, then learn from it (nar_model.py:1609-1632).  With the extended metrics on also 'predicted_item_ids' (the
        model's ranked candidates [L, 1+K] on the device, None without queries): the model's and the baselines' top-n
        lists are measured with the popularity the batch was fed with, before the state learns from the batch
        (:1591-1603).  The hit rate by session position takes the same lists.  With a per-session log on also
        'predicted_item_probs' [L, 1+K] and 'session_ids'.  With the unsampled metrics on, every label of the staged
        batch is ranked against the sampler's whole pool: the batch's clicks and labels and the recent-clicks buffer the
        step was fed with, before the state learns from the batch.  With the baselines' unsampled metrics on, each
        baseline ranks the same labels against the same pool right after its sampled scoring."""
        ext, bp = self.extended, self.by_position           # set in EVAL only
        pool = None
        if self.unsampled_hist is not None or self.unsampled_bench_hist is not None:
            pool = self.model.engine.unsampled_pool(run_values['clicked_items'], run_values['last_item_label'],
                                                    self.clicked_items_state.get_recent_clicks_buffer())
        if self.unsampled_hist is not None:
            self.model.engine.rank_labels(run_values['stage'], pool, self.eval_metrics_top_n, hist=self.unsampled_hist)
        if self.session_logs is not None:
            st = run_values['stage']
            t, pred = st['t'], run_values.get('predicted_item_ids')
            self.session_logs.add(run_values.get('session_ids'), t['label_next'], t['pos_idx'], t['sess_off'], st['L'],
                                  negatives=run_values['eval_batch_negative_items'], pred_ids=pred,
                                  pred_probs=run_values.get('predicted_item_probs'),
                                  cand=None if pred is None else self.model.engine.buffer(st, 'row_item').view(-1)[st['L']:],
                                  cand_stride=1 if pred is None else pred.shape[1], pop=t['pop_norm'])
        if ext is not None or bp is not None:
            st = run_values['stage']
            pred = run_values.get('predicted_item_ids')
            if pred is not None:
                # each query's label is column 0 of the candidate ids the ranking read
                cand = self.model.engine.buffer(st, 'row_item').view(-1)[st['L']:]
                if ext is not None:
                    ext.add_lists(pred, cand, st['t']['pop_norm'], label_stride=pred.shape[1])
                if bp is not None:
                    bp.add(pred, cand, st['T'], pos_idx=st['t']['pos_idx'], sess_off=st['t']['sess_off'],
                           pop=st['t']['pop_norm'], label_stride=pred.shape[1])
        if self.baselines is not None and self.mode == ModeKeys.EVAL:
            t = run_values['stage']['t']
            out_ids = None
            if ext is not None or bp is not None:
                import torch
                out_ids = torch.empty(self.baselines.n_rows, t['label_next'].numel(), self.eval_metrics_top_n,
                                      dtype=torch.int64, device=self.model.engine.dev)
            self.baselines.score(t['item_clicked'], t['label_next'], run_values['eval_batch_negative_items'],
                                 self.clicked_items_state.get_recent_clicks_buffer(),
                                 self.clicked_items_state.get_articles_pop(), self.eval_metrics_top_n, self.bench_metrics,
                                 out_ids=out_ids)
            if self.unsampled_bench_hist is not None:
                self.baselines.rank_unsampled(t['item_clicked'], t['label_next'], t['all_items'], pool,
                                              self.clicked_items_state.get_articles_pop(), self.eval_metrics_top_n,
                                              self.unsampled_bench_hist)
            if out_ids is not None:
                mask = sum(1 << self.baselines.row(s) for s in self.baselines.enabled)
                if ext is not None:
                    ext.add_lists(out_ids, t['label_next'].view(-1), t['pop_norm'], row0=1, row_mask=mask)
                if bp is not None:
                    bp.add(out_ids, t['label_next'].view(-1), run_values['stage']['T'], row0=1, row_mask=mask)
            if run_values['stage']['has_clicks']:
                self.baselines.update(t['all_items'], lens=np.count_nonzero(np.concatenate(
                    [run_values['clicked_items'], np.asarray(run_values['last_item_label']).reshape(-1, 1)], axis=1), axis=1),
                    session_ids=run_values.get('session_ids'))
        if ext is not None:
            t = run_values['stage']['t']
            ext.add_clicks(t['item_clicked'], t['label_next'])
        self.clicked_items_state.update_from_batch(run_values['clicked_items'], run_values['clicked_timestamps'],
                                                   run_values['last_item_label'])

    def benchmark_results(self) -> dict:
        """{'hitrate_at_n_<suffix>', 'mrr_at_n_<suffix>'} of this evaluation's baselines ({} without baselines)."""
        if self.baselines is None or self.bench_metrics is None:
            return {}
        return self.baselines.results(self.bench_metrics)

    def extended_results(self) -> dict:
        """The extended metrics of this evaluation ({} with them off): the model's keys without a suffix, each baseline's
        as ``<key>_<suffix>``."""
        if self.extended is None:
            return {}
        from .eval_metrics import KEYS, COVERAGE_KEY
        rows = self.extended.results()
        named = [('', rows[0])] + ([(s, rows[1 + self.baselines.row(s)]) for s in self.baselines.enabled]
                                   if self.baselines is not None else [])
        return {k + ('_' + s if s else ''): r[k] for s, r in named for k in KEYS + (COVERAGE_KEY,)}

    def by_position_results(self) -> dict:
        """The hit rate by session position of this evaluation ({} with it off): the model's keys without a suffix, each
        baseline's with its suffix (eval_metrics.ByPosition.results)."""
        if self.by_position is None:
            return {}
        names = [(0, '')] + ([(1 + self.baselines.row(s), s) for s in self.baselines.enabled]
                             if self.baselines is not None else [])
        return self.by_position.results(names)

    def unsampled_results(self) -> dict:
        """The unsampled metrics of this evaluation (eval_metrics.unsampled_results; {} with them off)."""
        if self.unsampled_hist is None:
            return {}
        from .eval_metrics import unsampled_results
        return unsampled_results(self.unsampled_hist.cpu().numpy(), self.eval_metrics_top_n)

    def unsampled_benchmark_results(self) -> dict:
        """The baselines' unsampled metrics of this evaluation (BaselineTables.unsampled_results; {} with them off)."""
        if self.unsampled_bench_hist is None:
            return {}
        return self.baselines.unsampled_results(self.unsampled_bench_hist)

    def end(self, session=None):
        if self.mode == ModeKeys.EVAL:
            if self.session_logs is not None:
                self.session_logs.end()
            self.clicked_items_state.restore_state_checkpoint()     # nar_model.py:1693
