"""Generate tests/golden/residual_golden.npz: outputs of the REFERENCE model code (nar_model.py's NARModuleModel, imported
unmodified) on the eager TF-1.x stand-in (tf1_shim.py) with build_rnn called with residual_connections=True - the
effect of passing residual_connections=True at the call site nar_model.py:408, which leaves it at its default False.
The branch that switch selects (:1319-1323) wraps every cell in tf.contrib.rnn.ResidualWrapper and layer 0 also in
tf.contrib.rnn.InputProjectionWrapper(cell, rnn_units).  The stand-in has neither wrapper; this file adds both to it, as
we read them in TF 1.12:

* ResidualWrapper (rnn_cell_impl.py) overrides __call__, so it opens no variable scope: output cell(x) + x, state the
  cell's own.
* InputProjectionWrapper (contrib/rnn/python/ops/core_rnn_cell.py) defines call, so it runs in the scope
  input_projection_wrapper.  There, _Linear(x, num_proj, bias=True) creates kernel [in, num_proj] with the scope's
  initializer (xavier, from `main`) and bias [num_proj] with zeros; no activation.  The wrapped cell runs in the same
  scope: .../multi_rnn_cell/cell_0/input_projection_wrapper/{kernel, bias, <cell>_cell/...}.

Same per-case contents as model_golden.npz (make_model_golden.run_case); the GRU case uses its GRUCell substitution and
the LSTM case make_lstm_golden.py's.  Every case runs CAR_embedding_size 64 with rnn_units 48: a transposed or mis-sized
projection fails, and the product pads 48 to 64 columns.  Cases: res64 (float64 TRAIN, one UGRNN layer, with the first
Adam step), res_drop64 (three UGRNN layers, dropout_keep_prob 0.8, the reference run's keep-masks recorded), res_gru64
(GRU, two layers), res_lstm64 (LSTM, two layers) and res_eval64 (EVAL, two UGRNN layers: ranking and recall@n / MRR@n).
tests/test_residual_oracle.py checks oracle/residual_ref.py against it.

Run once in the build container (python tests/golden/make_residual_golden.py); the .npz is committed."""
import os

import numpy as np

import make_lstm_golden as lg        # imports make_model_golden, which imports the reference's nar_model.py on the stand-in
import make_model_golden as mg

shim = mg.shim


class ResidualWrapper:
    """tf.contrib.rnn.ResidualWrapper(cell): __call__ -> (cell(x) + x, the cell's new state); no scope of its own."""

    def __init__(self, cell, residual_fn=None):
        self.cell = cell

    @property
    def state_size(self):
        return self.cell.state_size

    def __call__(self, inputs, state):
        out, new = self.cell(inputs, state)
        return out + inputs, new


class InputProjectionWrapper:
    """tf.contrib.rnn.InputProjectionWrapper(cell, num_proj): in the scope input_projection_wrapper, x -> x @ kernel + bias
    (_Linear with bias; kernel: the scope's initializer, bias: zeros), then the cell in the same scope."""

    def __init__(self, cell, num_proj, activation=None, input_size=None):
        assert activation is None
        self.cell, self.num_proj = cell, int(num_proj)
        self.kernel = None

    @property
    def state_size(self):
        return self.cell.state_size

    def __call__(self, inputs, state):
        with shim.variable_scope('input_projection_wrapper'):
            if self.kernel is None:
                self.kernel = shim.get_variable('kernel', [inputs.shape[-1], self.num_proj])
                self.bias = shim.get_variable('bias', [self.num_proj], initializer=shim.tf.zeros_initializer())
            return self.cell(inputs @ self.kernel + self.bias, state)


shim.tf.contrib.rnn.ResidualWrapper = ResidualWrapper
shim.tf.contrib.rnn.InputProjectionWrapper = InputProjectionWrapper

_build_rnn = mg.ref.NARModuleModel.build_rnn


def _build_rnn_residual(self, the_input, lengths, rnn_units=256, residual_connections=False):
    return _build_rnn(self, the_input, lengths, rnn_units=rnn_units, residual_connections=True)


mg.ref.NARModuleModel.build_rnn = _build_rnn_residual

HP = dict(rnn_units=48, rnn_residual_connections=True)


def main():
    cases = {}
    cases.update(mg.run_case('res64', keep_adam=True, hp_over=dict(HP)))
    cases.update(mg.run_case('res_drop64', hp_over=dict(HP, dropout_keep_prob=0.8, rnn_num_layers=3)))
    cases.update(mg.run_case('res_gru64', hp_over=dict(HP, rnn_num_layers=2), gru=True))
    cases.update(lg.run_lstm_case('res_lstm64', hp_over=dict(HP, rnn_num_layers=2)))
    cases.update(mg.run_case('res_eval64', mode='eval', steps_skip=1, hp_over=dict(HP, rnn_num_layers=2)))
    path = os.path.join(mg.HERE, 'residual_golden.npz')
    np.savez_compressed(path, **cases)
    print('wrote %d arrays, %.1f KB' % (len(cases), os.path.getsize(path) / 1024))


if __name__ == '__main__':
    main()
