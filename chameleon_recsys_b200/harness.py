"""Assemble one runnable NAR problem (configs + synthetic catalog + session stream + host state).

Plays the role of the bootstrap part of the reference trainer's ``main``
(nar_trainer_gcom.py:462-489): load ACR resources -> feature configs -> ClickedItemsState.
Used by tests, bench.py and __graft_entry__.smoke().
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import numpy as np

from .clicked_items_state import ClickedItemsState
from .datasets import prepare_dataset_iterator
from .hparams import (NARHParams, Workload, get_articles_features_config,
                      get_internal_enabled_features_config, get_session_features_config, workload)
from .plan import FeaturePlan, ParamLayout
from .synthetic import SessionStream, make_catalog


@dataclass
class Problem:
    wl: Workload
    hp: NARHParams
    session_features_config: dict
    articles_features_config: dict
    internal_features_config: Dict[str, bool]
    content_article_embeddings_matrix: np.ndarray
    articles_metadata: Dict[str, np.ndarray]
    plan: FeaturePlan
    layout: ParamLayout
    clicked_items_state: ClickedItemsState
    stream: SessionStream

    def params(self) -> dict:
        return self.hp.to_params(self.session_features_config, self.articles_features_config,
                                 self.articles_metadata, self.content_article_embeddings_matrix)

    def input_fn(self, batch_size=None):
        return prepare_dataset_iterator(self.stream, self.session_features_config,
                                        batch_size=batch_size or self.hp.batch_size,
                                        truncate_session_length=self.hp.truncate_session_length)


def make_problem(name_or_wl, profile=None, session_len=None, seed: int = 42, state_cls=None, **hp_overrides) -> Problem:
    wl = name_or_wl if isinstance(name_or_wl, Workload) else workload(name_or_wl, profile, session_len)
    if hp_overrides:
        wl.hp = wl.hp.copy(**hp_overrides)
    hp = wl.hp
    V, E = wl.num_items, wl.acr_dim
    acfg = get_articles_features_config(V, hp.enabled_articles_input_features_groups)
    scfg = get_session_features_config(V, hp.enabled_clicks_input_features_groups)
    icfg = get_internal_enabled_features_config(hp.enabled_internal_features)
    acr, meta = make_catalog(V, E, acfg, hp.content_embedding_scale_factor, seed=seed)
    plan = FeaturePlan(scfg, acfg, icfg, hp.max_cardinality_for_ohe, E, V)
    layout = ParamLayout(plan, hp.CAR_embedding_size, hp.rnn_units, hp.rnn_num_layers, rnn_cell=hp.rnn_cell,
                         residual=hp.rnn_residual_connections)
    state = (state_cls or ClickedItemsState)(hp.recent_clicks_buffer_hours, hp.recent_clicks_buffer_max_size,
                              hp.recent_clicks_for_normalization, V)
    stream = SessionStream(V, scfg, hp.truncate_session_length, wl.session_len, seed=seed,
                           sessions_per_tick=hp.batch_size)
    return Problem(wl, hp, scfg, acfg, icfg, acr, meta, plan, layout, state, stream)


def warm_state(problem: Problem, n_batches: int):
    """Feed ``n_batches`` through the host state only (buffer / popularity warm-up, SURVEY 8d)."""
    it = problem.input_fn()
    for _ in range(n_batches):
        feats, labels = it.get_next()
        problem.clicked_items_state.update_from_batch(feats['item_clicked'], feats['event_timestamp'],
                                                      labels['label_last_item'])
