"""nar_trainer.run_train_eval_loop and save_eval_benchmark_metrics_csv against the reference trainer's main loop
(nar_trainer_gcom.py:495-582, nar_utils.py:31-40): chunking, train / evaluate order, flush cadence, eval_hour_id, the CSV."""
import csv
import json
import types

import pytest

from chameleon_recsys_b200 import nar_trainer


class StubEstimator:
    """Records the calls; every evaluate appends one entry per fake session to the logs the loop switched on."""

    def __init__(self):
        self.params = {}
        self.calls = []
        self.n_eval = 0

    def train(self, input_fn):
        self.calls.append(('train', _files_of(input_fn)))

    def evaluate(self, input_fn):
        self.calls.append(('eval', _files_of(input_fn)))
        neg, rec = self.params.get('sessions_negative_items_log'), self.params.get('sessions_chameleon_recommendations_log')
        for s in range(2):
            sid = str(100 * self.n_eval + s)
            if neg is not None:
                neg.append({'session_id': sid, 'negative_items': [[1, 2]]})
            if rec is not None:
                rec.append({'session_id': sid, 'next_click_labels': [3], 'predicted_item_ids': [[3, 1, 2]],
                            'predicted_item_probs': [[0.5, 0.25, 0.25]], 'predicted_item_norm_pop': [[0.1, 0.2, 0.3]]})
        self.n_eval += 1
        out = {'loss': 1.0 / self.n_eval, 'hitrate_at_n': 0.5, 'sessions_count': 2}
        if self.n_eval == 2:
            out['late_metric'] = 7
        return out


def _files_of(input_fn):
    """The files an input_fn of the loop was made for (its closure holds them)."""
    cells = [c.cell_contents for c in input_fn.__closure__]
    files = [c for c in cells if isinstance(c, (str, list))]
    assert len(files) == 1
    return files[0]


HP = types.SimpleNamespace(batch_size=4, truncate_session_length=5)
FILES = ['h%02d' % i for i in range(7)]


def _run(tmp_path, est=None, **kw):
    est = est or StubEstimator()
    args = dict(train_files_from=0, train_files_up_to=6, training_hours_for_each_eval=2, save_results_each_n_evals=1,
                model_output_dir=str(tmp_path))
    args.update(kw)
    log = nar_trainer.run_train_eval_loop(est, FILES, {}, HP, **args)
    return est, log


def test_chunks():
    assert [list(c) for c in nar_trainer.chunks(FILES, 3)] == [FILES[0:3], FILES[3:6], FILES[6:]]
    assert list(nar_trainer.chunks([], 2)) == []


@pytest.mark.parametrize('hours,want', [
    (2, [('train', ['h00', 'h01']), ('eval', 'h02'), ('train', ['h02', 'h03']), ('eval', 'h04'),
         ('train', ['h04', 'h05']), ('eval', 'h06')]),
    (3, [('train', ['h00', 'h01', 'h02']), ('eval', 'h03'), ('train', ['h03', 'h04', 'h05']), ('eval', 'h06')]),
])
def test_train_chunk_then_evaluate_first_file_of_next(tmp_path, hours, want):
    est, log = _run(tmp_path, training_hours_for_each_eval=hours)
    assert est.calls == want                       # the last chunk is only ever evaluated on, never trained on
    assert len(log) == sum(1 for c in want if c[0] == 'eval') and log[0]['loss'] == 1.0


def test_from_up_to_slicing_and_error(tmp_path):
    est, _ = _run(tmp_path, train_files_from=1, train_files_up_to=4)
    assert est.calls == [('train', ['h01', 'h02']), ('eval', 'h03')]
    est, log = _run(tmp_path, train_files_from=2, train_files_up_to=2)
    assert est.calls == [] and log == []
    with pytest.raises(Exception, match='Final training file'):
        _run(tmp_path, train_files_from=3, train_files_up_to=2)


@pytest.mark.parametrize('each_n,want_ids', [(1, [0, 0, 1, 1, 2, 2]), (2, [0, 0, 1, 1, 1, 1])])
def test_eval_hour_id_and_appending(tmp_path, each_n, want_ids):
    """3 evaluations of 2 sessions.  Flushing every chunk: ids 0, 1, 2.  Every 2nd chunk (chunk 0 and chunk 2 flush; the
    id moves on after each flush of the recommendations log): chunk 0 -> 0, chunks 1 + 2 -> 1; the final flush is empty."""
    est, _ = _run(tmp_path, save_results_each_n_evals=each_n, save_eval_sessions_negative_samples=True,
                  save_eval_sessions_recommendations=True)
    rec = [json.loads(l) for l in (tmp_path / 'eval_chameleon_recommendations_log.json').read_text().splitlines()]
    neg = [json.loads(l) for l in (tmp_path / 'eval_sessions_negative_samples.json').read_text().splitlines()]
    assert [r['eval_hour_id'] for r in rec] == want_ids
    assert [r['session_id'] for r in rec] == [n['session_id'] for n in neg] == ['0', '1', '100', '101', '200', '201']
    assert list(rec[0]) == ['eval_hour_id', 'session_id', 'next_click_labels', 'predicted_item_ids', 'predicted_item_probs',
                            'predicted_item_norm_pop']
    assert list(neg[0]) == ['session_id', 'negative_items']
    assert est.params['sessions_negative_items_log'] == [] and est.params['sessions_chameleon_recommendations_log'] == []
    # a second run appends to the same files
    _run(tmp_path, save_eval_sessions_negative_samples=True, save_eval_sessions_recommendations=True)
    assert (tmp_path / 'eval_sessions_negative_samples.json').read_text().count('\n') == 12
    assert (tmp_path / 'eval_chameleon_recommendations_log.json').read_text().count('\n') == 12


def test_eval_hour_id_stays_without_the_recommendations_log(tmp_path):
    est, _ = _run(tmp_path, save_eval_sessions_negative_samples=True)
    assert not (tmp_path / 'eval_chameleon_recommendations_log.json').exists()
    assert 'sessions_chameleon_recommendations_log' not in est.params
    assert (tmp_path / 'eval_sessions_negative_samples.json').read_text().count('\n') == 6


def test_logs_off_writes_the_csv_only(tmp_path):
    est, _ = _run(tmp_path)
    assert sorted(p.name for p in tmp_path.iterdir()) == ['eval_stats_benchmarks.csv']
    assert est.params == {}


def test_an_existing_eval_graph_is_rebuilt_with_the_list(tmp_path):
    est = StubEstimator()
    est._eval_spec = object()
    _run(tmp_path, est=est, save_eval_sessions_negative_samples=True)
    assert est._eval_spec is None
    given = []
    est = StubEstimator()
    est.params['sessions_negative_items_log'] = given
    est._eval_spec = spec = object()
    _run(tmp_path, est=est, save_eval_sessions_negative_samples=True)
    assert est._eval_spec is spec and est.params['sessions_negative_items_log'] is given


def test_metrics_csv(tmp_path):
    log = [{'loss': 0.5, 'hitrate_at_n': 0.25}, {'loss': 0.4, 'hitrate_at_n': 0.3, 'mrr_at_n_pop': 0.1},
           {'hitrate_at_n': 0.35, 'loss': 0.3}, {'loss': 0.2}, {'loss': 0.1}]
    nar_trainer.save_eval_benchmark_metrics_csv(log, str(tmp_path), training_hours_for_each_eval=5)
    rows = list(csv.reader(open(tmp_path / 'eval_stats_benchmarks.csv')))
    assert rows[0] == ['index', 'loss', 'hitrate_at_n', 'mrr_at_n_pop', 'hour', 'day']     # union, first-seen order
    assert [r[0] for r in rows[1:]] == ['0', '1', '2', '3', '4']
    assert [r[-2] for r in rows[1:]] == ['5', '10', '15', '20', '1']                      # (i + 1) * 5 % 24
    assert [r[-1] for r in rows[1:]] == ['0', '0', '0', '0', '1']                         # int((i + 1) * 5 / 24)
    assert rows[1][1:4] == ['0.5', '0.25', ''] and rows[2][3] == '0.1' and rows[4][2] == ''
    # rewritten in full, not appended to
    nar_trainer.save_eval_benchmark_metrics_csv(log[:2], str(tmp_path), training_hours_for_each_eval=5)
    assert len(list(csv.reader(open(tmp_path / 'eval_stats_benchmarks.csv')))) == 3


def test_loop_rewrites_the_csv_each_flush(tmp_path):
    _, log = _run(tmp_path)
    rows = list(csv.reader(open(tmp_path / 'eval_stats_benchmarks.csv')))
    assert rows[0] == ['index', 'loss', 'hitrate_at_n', 'sessions_count', 'late_metric', 'hour', 'day']
    assert len(rows) == 1 + len(log) == 4 and [r[-2] for r in rows[1:]] == ['2', '4', '6']
    assert [r[4] for r in rows[1:]] == ['', '7', '']
