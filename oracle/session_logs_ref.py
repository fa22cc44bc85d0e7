"""Numpy spec of the per-session evaluation logs the reference hook fills in ``after_run`` (nar_model.py:1529-1581):

* ``sessions_negative_items_log``: per session ``{'session_id': str, 'negative_items': [[K ids] per query]}``;
* ``sessions_chameleon_recommendations_log``: per session ``{'session_id': str, 'next_click_labels': [label per query],
  'predicted_item_ids': [[1 + K ids]], 'predicted_item_probs': [[1 + K floats]], 'predicted_item_norm_pop': [[1 + K]]}``.

A query is a cell (b, t) with ``next_item_labels[b, t] != 0``, visited session by session, t ascending; every session of
the batch gets an entry, also one without a query (empty lists).  Probabilities are ``ndarray.round(decimals=7)`` of the
float32 array (numpy computes rint(x * 1e7) / 1e7 in the array's dtype); the popularity is ``pop_norm[ids]`` rounded the
same way in ``pop_norm``'s dtype - float64 in the reference's host state, float32 when it is the array the model was fed.
Values are the Python objects ``ndarray.tolist()`` gives (a float32 widens exactly to the float it prints as).
"""
from __future__ import annotations

import numpy as np


def negative_items_log(session_ids, next_item_labels, eval_negative_items) -> list:
    labels, neg = np.asarray(next_item_labels), np.asarray(eval_negative_items)
    return [{'session_id': str(sid), 'negative_items': neg[b][labels[b] != 0].tolist()}
            for b, sid in enumerate(np.asarray(session_ids))]


def recommendations_log(session_ids, next_item_labels, predicted_item_ids, predicted_item_probs, pop_norm) -> list:
    labels, ids = np.asarray(next_item_labels), np.asarray(predicted_item_ids)
    probs = np.asarray(predicted_item_probs).round(decimals=7)
    pops = np.asarray(pop_norm)[ids].round(decimals=7)
    out = []
    for b, sid in enumerate(np.asarray(session_ids)):
        q = labels[b] != 0
        out.append({'session_id': str(sid),
                    'next_click_labels': labels[b][q].tolist(),
                    'predicted_item_ids': ids[b][q].tolist(),
                    'predicted_item_probs': probs[b][q].tolist(),
                    'predicted_item_norm_pop': pops[b][q].tolist()})
    return out


def scatter_compact(rows, pos_idx, B: int, T: int) -> np.ndarray:
    """Compact per-row values [L, ...] at flat positions ``pos_idx`` [L] (b * T + t) -> the padded [B, T, ...] array."""
    rows = np.asarray(rows)
    out = np.zeros((B * T,) + rows.shape[1:], dtype=rows.dtype)
    out[np.asarray(pos_idx, dtype=np.int64)[:rows.shape[0]]] = rows
    return out.reshape((B, T) + rows.shape[1:])


def session_logs_ref(session_ids, next_item_labels, eval_negative_items=None, predicted_item_ids=None,
                     predicted_item_probs=None, pop_norm=None, pos_idx=None):
    """-> (negatives log or None, recommendations log or None) of one batch.  ``predicted_item_ids`` / ``_probs`` are
    [B, T, 1 + K], or with ``pos_idx`` the compact [L, 1 + K] rows of the valid positions."""
    labels = np.asarray(next_item_labels)
    neg_log = rec_log = None
    if eval_negative_items is not None:
        neg_log = negative_items_log(session_ids, labels, eval_negative_items)
    if predicted_item_ids is not None:
        if pos_idx is not None:
            B, T = labels.shape
            predicted_item_ids = scatter_compact(predicted_item_ids, pos_idx, B, T)
            predicted_item_probs = scatter_compact(predicted_item_probs, pos_idx, B, T)
        rec_log = recommendations_log(session_ids, labels, predicted_item_ids, predicted_item_probs, pop_norm)
    return neg_log, rec_log
