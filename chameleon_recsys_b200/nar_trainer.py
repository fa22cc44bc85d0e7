"""The temporal train / evaluate loop of the reference trainer (nar_trainer_gcom.py:495-582) and the writers of its
three result files (nar_trainer_gcom.py:390-407, nar_utils.py:31-40), as plain functions: no flags, no GCS, no ML Engine
(DESIGN.md section 7).

The hour files are cut into chunks of ``training_hours_for_each_eval``; the model trains on a chunk and is evaluated on the
first hour of the next one; every ``save_results_each_n_evals`` chunks ``eval_stats_benchmarks.csv`` is rewritten and the
per-session logs are appended to their JSON-lines files.
"""
from __future__ import annotations

import csv
import json
import os
from typing import Iterator, List, Sequence

from .datasets import prepare_dataset_iterator


def chunks(l: Sequence, n: int) -> Iterator[Sequence]:
    """Successive ``n``-sized chunks of ``l`` (utils.py:53-56)."""
    for i in range(0, len(l), n):
        yield l[i:i + n]


def append_lines_to_text_file(filename: str, lines):
    with open(filename, 'a') as f:
        f.writelines([line + '\n' for line in lines])


def save_sessions_negative_items(model_output_dir, sessions_negative_items_list,
                                 output_file='eval_sessions_negative_samples.json'):
    """Append one JSON object per session: the negative samples each of its clicks was evaluated against, so that
    recommenders outside the framework can be measured on the same candidates."""
    append_lines_to_text_file(os.path.join(model_output_dir, output_file),
                              (json.dumps({'session_id': x['session_id'], 'negative_items': x['negative_items']})
                               for x in sessions_negative_items_list))


def save_sessions_chameleon_recommendations_log(model_output_dir, sessions_chameleon_recommendations_log_list, eval_hour_id,
                                                output_file='eval_chameleon_recommendations_log.json'):
    """Append one JSON object per session: per click the label, the ranked candidates, their probabilities and their
    normalised recent popularity - the input of re-ranking experiments."""
    append_lines_to_text_file(os.path.join(model_output_dir, output_file),
                              (json.dumps({'eval_hour_id': eval_hour_id,
                                           'session_id': x['session_id'],
                                           'next_click_labels': x['next_click_labels'],
                                           'predicted_item_ids': x['predicted_item_ids'],
                                           'predicted_item_probs': x['predicted_item_probs'],
                                           'predicted_item_norm_pop': x['predicted_item_norm_pop']})
                               for x in sessions_chameleon_recommendations_log_list))


def save_eval_benchmark_metrics_csv(eval_sessions_metrics_log, output_dir, training_hours_for_each_eval,
                                    output_csv='eval_stats_benchmarks.csv'):
    """One row per evaluation, the file rewritten in full: ``index``, every metric key in first-seen order (an empty cell
    where an evaluation lacks it), then the ``hour`` and ``day`` the evaluation stands for."""
    keys: List[str] = []
    for row in eval_sessions_metrics_log:
        keys.extend(k for k in row if k not in keys)
    with open(os.path.join(output_dir, output_csv), 'w', newline='') as f:
        w = csv.writer(f, lineterminator='\n')
        w.writerow(['index'] + keys + ['hour', 'day'])
        for i, row in enumerate(eval_sessions_metrics_log):
            hours = (i + 1) * training_hours_for_each_eval
            w.writerow([i] + [row.get(k, '') for k in keys] + [hours % 24, int(hours / 24)])


def run_train_eval_loop(estimator, train_files, session_features_config, hparams, *, train_files_from, train_files_up_to,
                        training_hours_for_each_eval, save_results_each_n_evals, model_output_dir,
                        save_eval_sessions_negative_samples=False, save_eval_sessions_recommendations=False) -> list:
    """``train_files``: the sorted hour files; ``[train_files_from, train_files_up_to]`` (inclusive) are used.  Returns
    the metrics log: ``estimator.evaluate``'s result of every evaluation, in order.  The per-session logs are switched on
    through ``estimator.params`` (lists the evaluation hook appends to) and emptied in place after each flush."""
    if train_files_from > train_files_up_to:
        raise Exception('Final training file cannot be lower than Starting training file')
    train_files = list(train_files)[train_files_from:train_files_up_to + 1]
    batch_size, truncate = hparams.batch_size, hparams.truncate_session_length

    def input_fn(files):
        return lambda: prepare_dataset_iterator(files, session_features_config, batch_size=batch_size,
                                                truncate_session_length=truncate)

    negatives_log = recommendations_log = None
    for on, key in ((save_eval_sessions_negative_samples, 'sessions_negative_items_log'),
                    (save_eval_sessions_recommendations, 'sessions_chameleon_recommendations_log')):
        if on and estimator.params.get(key) is None:
            estimator.params[key] = []
            if getattr(estimator, '_eval_spec', None) is not None:
                estimator._eval_spec = None                   # its hook was built without the list
    if save_eval_sessions_negative_samples:
        negatives_log = estimator.params['sessions_negative_items_log']
    if save_eval_sessions_recommendations:
        recommendations_log = estimator.params['sessions_chameleon_recommendations_log']

    eval_sessions_metrics_log: list = []
    eval_hour_id = 0

    def flush(last: bool):
        nonlocal eval_hour_id
        save_eval_benchmark_metrics_csv(eval_sessions_metrics_log, model_output_dir,
                                        training_hours_for_each_eval=training_hours_for_each_eval)
        if negatives_log is not None:
            save_sessions_negative_items(model_output_dir, negatives_log)
            del negatives_log[:]
        if recommendations_log is not None:
            save_sessions_chameleon_recommendations_log(model_output_dir, recommendations_log, eval_hour_id)
            del recommendations_log[:]
            if not last:
                eval_hour_id += 1

    training_files_chunks = list(chunks(train_files, training_hours_for_each_eval))
    for chunk_id in range(len(training_files_chunks) - 1):
        estimator.train(input_fn=input_fn(list(training_files_chunks[chunk_id])))
        # the first hour of the next chunk is the evaluation set
        eval_sessions_metrics_log.append(estimator.evaluate(input_fn=input_fn(training_files_chunks[chunk_id + 1][0])))
        if chunk_id % save_results_each_n_evals == 0:
            flush(last=False)
    flush(last=True)
    return eval_sessions_metrics_log
