"""Generate tests/golden/lstm_golden.npz: outputs of the REFERENCE model code (nar_model.py's NARModuleModel, imported
unmodified) on the eager TF-1.x stand-in (tf1_shim.py), with an LSTMCell stand-in handed out where build_rnn asks for
tf.contrib.rnn.UGRNNCell - the effect of un-commenting nar_model.py:1316
(`cell = tf.nn.rnn_cell.LSTMCell(rnn_units, state_is_tuple=True)`), as make_model_golden.py's gru64 case does for :1315.

Same per-case contents as model_golden.npz (make_model_golden.run_case).  Cases: lstm64 (float64 TRAIN, one layer, with
the first Adam step), lstm_drop64 (two layers, dropout_keep_prob 0.8, the reference run's keep-masks recorded) and
lstm_eval64 (EVAL: ranking and recall@n / MRR@n).  What this pins is the cell's place and wiring in the reference graph;
the cell's arithmetic is the stand-in's reading of TF 1.12 rnn_cell_impl.py, not TensorFlow's.

Run once in the build container (python tests/golden/make_lstm_golden.py); the .npz is committed."""
import os

import numpy as np
import torch

import make_model_golden as mg        # imports the reference's nar_model.py on the stand-in

shim = mg.shim


class LSTMCell:
    """tf.nn.rnn_cell.LSTMCell(num_units, state_is_tuple=True) (TF 1.12 rnn_cell_impl.py; no peepholes, cell clip or
    projection, forget_bias 1.0, tanh): z = [x, h] @ kernel + bias, columns i | j | f | o;
    c' = sigmoid(f + 1) * c + sigmoid(i) * tanh(j); h' = sigmoid(o) * tanh(c'); output h'.
    The (c, h) tuple travels as one [B, 2H] tensor [c | h], so the stand-in's dynamic_rnn and MultiRNNCell (which zero-
    initialise and carry a state of width state_size) take it unchanged."""

    def __init__(self, num_units, **k):
        self.num_units = int(num_units)
        self.scope_name = 'lstm_cell'
        self.kernel = None

    @property
    def state_size(self):
        return 2 * self.num_units

    def __call__(self, inputs, state):
        n = self.num_units
        if self.kernel is None:
            with shim.variable_scope(self.scope_name):
                self.kernel = shim.get_variable('kernel', [inputs.shape[-1] + n, 4 * n])
                self.bias = shim.get_variable('bias', [4 * n], initializer=shim.tf.zeros_initializer())
        c, h = state[:, :n], state[:, n:]
        z = torch.cat([inputs, h], 1) @ self.kernel + self.bias
        i, j, f, o = z[:, :n], z[:, n:2 * n], z[:, 2 * n:3 * n], z[:, 3 * n:]
        c_new = torch.sigmoid(f + 1.0) * c + torch.sigmoid(i) * torch.tanh(j)
        h_new = torch.sigmoid(o) * torch.tanh(c_new)
        return h_new, torch.cat([c_new, h_new], 1)


def run_lstm_case(name, **kw):
    # run_case(gru=True) installs shim.GRUCell as tf.contrib.rnn.UGRNNCell; bound to the LSTM stand-in for this call
    gru = shim.GRUCell
    shim.GRUCell = LSTMCell
    try:
        return mg.run_case(name, gru=True, **kw)
    finally:
        shim.GRUCell = gru


def main():
    cases = {}
    cases.update(run_lstm_case('lstm64', keep_adam=True))
    cases.update(run_lstm_case('lstm_drop64', hp_over=dict(dropout_keep_prob=0.8, rnn_num_layers=2)))
    cases.update(run_lstm_case('lstm_eval64', mode='eval', steps_skip=1))
    path = os.path.join(mg.HERE, 'lstm_golden.npz')
    np.savez_compressed(path, **cases)
    print('wrote %d arrays, %.1f KB' % (len(cases), os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
