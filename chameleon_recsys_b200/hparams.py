"""Hyper-parameters and feature configs of the NAR training hot path.

Names and defaults mirror the reference's flags and ``NARModuleModel`` ctor so a
reference user finds the same knobs:

* flags:        nar_module/nar/nar_trainer_gcom.py:37-67
* params dict:  nar_module/nar/nar_trainer_gcom.py:355-384
* ctor kwargs:  nar_module/nar/nar_model.py:102-129
* feature cfgs: nar_module/nar/nar_trainer_gcom.py:99-128 (articles), :150-218 (sessions)
"""
from __future__ import annotations

import copy
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

# nar_model.py:22-23
ARTICLE_REQ_FEATURES = ['article_id', 'created_at_ts']
SESSION_REQ_SEQ_FEATURES = ['item_clicked', 'event_timestamp']

VALID_INTERNAL_FEATURES = ['recency', 'novelty', 'article_content_embeddings', 'item_clicked_embeddings']
ALL_FEATURES = 'ALL'


class ModeKeys:
    """Stand-in for tf.estimator.ModeKeys (same string values)."""
    TRAIN = 'train'
    EVAL = 'eval'
    PREDICT = 'infer'


def get_embedding_size(unique_val_count: int, const_mult: int = 8) -> int:
    """nar_model.py:25-26."""
    return int(math.floor(const_mult * unique_val_count ** 0.25))


def get_articles_features_config(num_items: int,
                                 enabled_articles_input_features_groups=(ALL_FEATURES,),
                                 category_cardinality: int = 461) -> dict:
    """nar_trainer_gcom.py:99-128.  The gcom trainer forgets the article_id
    cardinality (nar_model.py:183 reads it); the Adressa trainer sets it
    (nar_trainer_adressa.py:130-132) - we always set it."""
    cfg = {
        'article_id': {'type': 'categorical', 'dtype': 'int', 'cardinality': int(num_items)},
        'created_at_ts': {'type': 'numerical', 'dtype': 'int'},
        'category_id': {'type': 'categorical', 'dtype': 'int', 'cardinality': int(category_cardinality)},
    }
    feature_groups = {'category': ['category_id']}
    groups = list(enabled_articles_input_features_groups)
    if groups != [ALL_FEATURES]:
        for g, feats in feature_groups.items():
            if g not in groups:
                for f in feats:
                    del cfg[f]
    return cfg


def get_session_features_config(num_items: int,
                                enabled_clicks_input_features_groups=(ALL_FEATURES,)) -> dict:
    """nar_trainer_gcom.py:150-218 (G1 cardinalities)."""
    cfg = {
        'single_features': {
            'user_id': {'type': 'categorical', 'dtype': 'int', 'cardinality': 341193},
            'session_id': {'type': 'categorical', 'dtype': 'int'},
            'session_start': {'type': 'categorical', 'dtype': 'int'},
            'session_size': {'type': 'categorical', 'dtype': 'int'},
        },
        'sequence_features': {
            'event_timestamp': {'type': 'numerical', 'dtype': 'int'},
            'item_clicked': {'type': 'categorical', 'dtype': 'int', 'cardinality': int(num_items)},
            'environment': {'type': 'categorical', 'dtype': 'int', 'cardinality': 5},
            'deviceGroup': {'type': 'categorical', 'dtype': 'int', 'cardinality': 6},
            'os': {'type': 'categorical', 'dtype': 'int', 'cardinality': 23},
            'country': {'type': 'categorical', 'dtype': 'int', 'cardinality': 12},
            'region': {'type': 'categorical', 'dtype': 'int', 'cardinality': 29},
            'local_hour_sin': {'type': 'numerical', 'dtype': 'float'},
            'local_hour_cos': {'type': 'numerical', 'dtype': 'float'},
            'local_weekday': {'type': 'numerical', 'dtype': 'float'},
            'referrer_type': {'type': 'categorical', 'dtype': 'int', 'cardinality': 8},
        },
    }
    feature_groups = {
        'time': ['local_hour_sin', 'local_hour_cos', 'local_weekday'],
        'device': ['environment', 'deviceGroup', 'os'],
        'location': ['country', 'region'],
        'referrer': ['referrer_type'],
    }
    groups = list(enabled_clicks_input_features_groups)
    if groups != [ALL_FEATURES]:
        for g, feats in feature_groups.items():
            if g not in groups:
                for f in feats:
                    del cfg['sequence_features'][f]
    return cfg


def get_internal_enabled_features_config(enabled_internal_features=(ALL_FEATURES,)) -> Dict[str, bool]:
    """nar_trainer_gcom.py:220-231."""
    feats = list(enabled_internal_features)
    if feats == [ALL_FEATURES]:
        enabled = set(VALID_INTERNAL_FEATURES)
    else:
        enabled = set(feats).intersection(VALID_INTERNAL_FEATURES)
    return {f: (f in enabled) for f in VALID_INTERNAL_FEATURES}


@dataclass
class NARHParams:
    """One object carrying every hparam the hot path reads (reference flag names)."""
    # nar_trainer_gcom.py:37-60
    batch_size: int = 64
    truncate_session_length: int = 20
    learning_rate: float = 1e-3
    dropout_keep_prob: float = 1.0
    reg_l2: float = 0.0002
    softmax_temperature: float = 1.0
    recent_clicks_buffer_hours: float = 1.0
    recent_clicks_buffer_max_size: int = 500
    recent_clicks_for_normalization: int = 500
    eval_metrics_top_n: int = 3
    CAR_embedding_size: int = 512
    rnn_units: int = 1024
    rnn_num_layers: int = 1
    train_total_negative_samples: int = 5
    train_negative_samples_from_buffer: int = 10
    eval_total_negative_samples: int = 20
    eval_negative_samples_from_buffer: int = 50
    novelty_reg_factor: float = 0.0
    diversity_reg_factor: float = 0.0      # dead in the reference (nar_model.py:685-702)
    content_embedding_scale_factor: float = 1.0
    enabled_clicks_input_features_groups: List[str] = field(default_factory=lambda: [ALL_FEATURES])
    enabled_articles_input_features_groups: List[str] = field(default_factory=lambda: [ALL_FEATURES])
    enabled_internal_features: List[str] = field(default_factory=lambda: [ALL_FEATURES])
    # nar_model.py:117-121
    elapsed_days_smooth_log_base: float = 1.3
    popularity_smooth_log_base: float = 2.0
    max_cardinality_for_ohe: int = 10
    # --- extensions (documented in DESIGN.md) ---
    rnn_cell: str = 'ugrnn'          # 'ugrnn' = reference code (nar_model.py:1317)
    # build_rnn's residual_connections (nar_model.py:1319-1323; the reference calls it with the default False): layer 0
    # projects its input to rnn_units and adds it to the cell's output, layers > 0 add their input (DESIGN.md section 15)
    rnn_residual_connections: bool = False
    ranking: str = 'mlp'             # 'mlp' = reference code (nar_model.py:447-500); 'cosine' = north_star wording
    sampler_seed: int = 42           # RANDOM_SEED, nar_trainer_gcom.py:33
    init_seed: int = 42
    # baseline recommenders evaluated next to the model (nar_trainer_gcom.py:280-300): suffixes or
    # {'recommender': <suffix>, 'params': {...}} of 'pop_recent', 'coocurrent', 'item_knn', 'cb', 'sr', and the session
    # kNN baselines 'v-sknn' / 'sknn' (baselines.py, sknn.py; they need the batches' 'session_id' feature)
    eval_benchmarks: tuple = ()
    # NDCG, item coverage, ESI-R / ESI-RR and EILD-R / EILD-RR of the model and every baseline in Estimator.evaluate
    # (the reference hook's create_eval_metrics; eval_metrics.py)
    eval_extended_metrics: bool = False
    # the hit rate at the 1st, 2nd, ... click of a session for the model and every baseline, and the model's query count
    # and mean label popularity per position, in Estimator.evaluate (the reference trainer's flag of the same name,
    # nar_trainer_gcom.py:56; eval_metrics.ByPosition)
    eval_metrics_by_session_position: bool = False
    # hit rate, MRR and NDCG of each label ranked against every article the negative sampler could have drawn for it, in
    # Estimator.evaluate (DESIGN.md section 13; NarEngine.rank_labels)
    eval_unsampled_metrics: bool = False
    # the same unsampled hit rate, MRR and NDCG for every baseline of eval_benchmarks, ranked against the same competitors
    # (DESIGN.md section 14; BaselineTables.rank_unsampled)
    eval_unsampled_benchmarks: bool = False

    def to_params(self, session_features_config, articles_features_config, articles_metadata,
                  content_article_embeddings_matrix) -> dict:
        """The ``params`` dict handed to ``nar_module_model_fn`` (nar_trainer_gcom.py:355-384)."""
        params = {
            'batch_size': self.batch_size,
            'lr': self.learning_rate,
            'dropout_keep_prob': self.dropout_keep_prob,
            'reg_weight_decay': self.reg_l2,
            'recent_clicks_buffer_hours': self.recent_clicks_buffer_hours,
            'recent_clicks_buffer_max_size': self.recent_clicks_buffer_max_size,
            'recent_clicks_for_normalization': self.recent_clicks_for_normalization,
            'eval_metrics_top_n': self.eval_metrics_top_n,
            'CAR_embedding_size': self.CAR_embedding_size,
            'rnn_units': self.rnn_units,
            'rnn_num_layers': self.rnn_num_layers,
            'train_total_negative_samples': self.train_total_negative_samples,
            'train_negative_samples_from_buffer': self.train_negative_samples_from_buffer,
            'eval_total_negative_samples': self.eval_total_negative_samples,
            'eval_negative_samples_from_buffer': self.eval_negative_samples_from_buffer,
            'softmax_temperature': self.softmax_temperature,
            'save_histograms': False,
            'eval_metrics_by_session_position': self.eval_metrics_by_session_position,
            'novelty_reg_factor': self.novelty_reg_factor,
            'diversity_reg_factor': self.diversity_reg_factor,
            'eval_negative_sample_relevance': 0.1,
            'eval_cold_start': False,
            'session_features_config': session_features_config,
            'articles_features_config': articles_features_config,
            'articles_metadata': articles_metadata,
            'content_article_embeddings_matrix': content_article_embeddings_matrix,
            # extensions
            'internal_features_config': get_internal_enabled_features_config(self.enabled_internal_features),
            'elapsed_days_smooth_log_base': self.elapsed_days_smooth_log_base,
            'popularity_smooth_log_base': self.popularity_smooth_log_base,
            'max_cardinality_for_ohe': self.max_cardinality_for_ohe,
            'sampler_seed': self.sampler_seed,
            'init_seed': self.init_seed,
            'rnn_cell': self.rnn_cell,
            'ranking': self.ranking,
        }
        if self.eval_benchmarks:                 # the key exists only when baselines are requested
            params['eval_benchmarks'] = list(self.eval_benchmarks)
        if self.eval_extended_metrics:           # likewise only when requested
            params['eval_extended_metrics'] = True
        if self.eval_unsampled_metrics:
            params['eval_unsampled_metrics'] = True
        if self.eval_unsampled_benchmarks:
            params['eval_unsampled_benchmarks'] = True
        if self.rnn_residual_connections:
            params['rnn_residual_connections'] = True
        return params

    def copy(self, **kw) -> 'NARHParams':
        h = copy.deepcopy(self)
        for k, v in kw.items():
            if not hasattr(h, k):
                raise AttributeError(k)
            setattr(h, k, v)
        return h


# ---------------------------------------------------------------------------
# The BASELINE.json workloads (SURVEY.md section 8: (V,E,H,B,S,K); C=64 tiny else 1024)
# ---------------------------------------------------------------------------
@dataclass
class Workload:
    name: str
    num_items: int
    acr_dim: int
    hp: NARHParams
    profile: str = 'B'           # 'A' = no context/metadata features; 'B' = G1 script features
    session_len: str = 'g1'      # 'g1' = min(2+Geom(.53), S) ; 'dense' = all S


def _script_hparams(**kw) -> NARHParams:
    """run_nar_train_gcom_local.sh:17-39 / README.md:283-299 values."""
    base = dict(learning_rate=1e-4, dropout_keep_prob=1.0, reg_l2=1e-5, softmax_temperature=0.1,
                recent_clicks_buffer_hours=1.0, recent_clicks_buffer_max_size=20000,
                recent_clicks_for_normalization=2000, CAR_embedding_size=1024, rnn_units=255,
                rnn_num_layers=1, train_negative_samples_from_buffer=3000,
                eval_negative_samples_from_buffer=3000, novelty_reg_factor=0.0)
    base.update(kw)
    return NARHParams(**base)


def workload(name: str, profile: Optional[str] = None, session_len: Optional[str] = None) -> Workload:
    if name == 'tiny':
        hp = _script_hparams(batch_size=64, truncate_session_length=5, CAR_embedding_size=64, rnn_units=64,
                             train_total_negative_samples=10, eval_total_negative_samples=10,
                             recent_clicks_buffer_max_size=2000, recent_clicks_for_normalization=500,
                             train_negative_samples_from_buffer=300, eval_negative_samples_from_buffer=300)
        w = Workload('tiny', 1000, 64, hp)
    elif name == 'g1':
        hp = _script_hparams(batch_size=256, truncate_session_length=20,
                             train_total_negative_samples=50, eval_total_negative_samples=50)
        w = Workload('g1', 46034, 250, hp)
    elif name == 'adressa':
        hp = _script_hparams(batch_size=1024, truncate_session_length=30,
                             train_total_negative_samples=100, eval_total_negative_samples=100,
                             train_negative_samples_from_buffer=5000, eval_negative_samples_from_buffer=5000)
        w = Workload('adressa', 13000, 250, hp)
    elif name == 'g1x8':
        hp = _script_hparams(batch_size=4096, truncate_session_length=20,
                             train_total_negative_samples=50, eval_total_negative_samples=50)
        w = Workload('g1x8', 46034, 250, hp)
    elif name == 'stress':
        hp = _script_hparams(batch_size=8192, truncate_session_length=20, rnn_units=512,
                             train_total_negative_samples=500, eval_total_negative_samples=500)
        w = Workload('stress', 1000000, 512, hp)
    else:
        raise ValueError('unknown workload %r' % name)
    if profile is not None:
        w.profile = profile
    if session_len is not None:
        w.session_len = session_len
    if w.profile == 'A':
        w.hp.enabled_clicks_input_features_groups = ['NONE']
        w.hp.enabled_articles_input_features_groups = ['NONE']
        w.hp.enabled_internal_features = ['article_content_embeddings', 'item_clicked_embeddings']
    return w
