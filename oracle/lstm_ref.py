"""TEST INFRASTRUCTURE - the oracle with the session RNN built from tf.nn.rnn_cell.LSTMCell (rnn_cell='lstm').

nar_model.py:1308-1342 builds the session RNN; :1316 keeps `#cell = tf.nn.rnn_cell.LSTMCell(rnn_units, state_is_tuple=True)`
one comment away from the UGRNNCell it runs (:1317).  LstmOracle is NarOracle (oracle/nar_oracle.py) with that cell in
rnn(); everything else - features, CAR, FC1 / FC2, scorer, loss, Adam, the dropout sites - is NarOracle's.

Pinning, as for the GRU branch: tests/golden/lstm_golden.npz comes from the reference's nar_model.py, unmodified, run on
the eager TF-1.x stand-in with an LSTMCell handed out where the code asks for UGRNNCell (tests/golden/make_lstm_golden.py).
That pins where the cell sits in the graph and how it is wired (variable names and shapes, DropoutWrapper on the output
only, the state carried past a session's length, layer k > 0 fed by layer k-1's dropped output).  The cell's arithmetic
is our reading of TF 1.12 rnn_cell_impl.py LSTMCell.call, restated here and in the stand-in; TensorFlow itself is unpinned.

LSTMCell(H, state_is_tuple=True): no peepholes, no cell clip, no projection, forget_bias = 1.0, activation tanh:
    z  = [x, h] @ kernel + bias             kernel [in+H, 4H], bias [4H] (zeros initialiser), columns i | j | f | o
    c' = sigmoid(f + forget_bias) * c + sigmoid(i) * tanh(j)
    h' = sigmoid(o) * tanh(c')              output h', state (c', h'), both zero at t = 0
"""
from __future__ import annotations

import torch

from .nar_oracle import NarOracle

FORGET_BIAS = 1.0       # LSTMCell default; a constant inside the cell, not part of the stored bias


def lstm_cell(x, c, h, kernel, bias):
    """One tf.nn.rnn_cell.LSTMCell step (rnn_cell_impl.py LSTMCell.call) -> (c', h')."""
    H = h.shape[-1]
    z = torch.cat([x, h], dim=1) @ kernel + bias
    i, j, f, o = z[:, :H], z[:, H:2 * H], z[:, 2 * H:3 * H], z[:, 3 * H:]
    c_new = torch.sigmoid(f + FORGET_BIAS) * c + torch.sigmoid(i) * torch.tanh(j)
    h_new = torch.sigmoid(o) * torch.tanh(c_new)
    return c_new, h_new


class LstmOracle(NarOracle):
    def __init__(self, *args, **kw):
        kw['rnn_cell'] = 'lstm'
        super().__init__(*args, **kw)

    def rnn(self, x, lengths, pos_key=None):
        """nar_model.py:1308-1342 with LSTMCell: MultiRNNCell of DropoutWrapper(LSTMCell, output_keep_prob) inside
        dynamic_rnn(sequence_length).  The dropped OUTPUT h feeds the next layer / FC1; the carried state (c, h) is not
        dropped; past a session's length the output is zero and the state is carried unchanged."""
        B, T, _ = x.shape
        H = self.H
        cs = [torch.zeros(B, H, dtype=self.dtype) for _ in range(self.layers)]
        hs = [torch.zeros(B, H, dtype=self.dtype) for _ in range(self.layers)]
        outs = []
        for t in range(T):
            inp = x[:, t]
            new = []
            for i in range(self.layers):
                base = 'main/RNN/rnn/multi_rnn_cell/cell_{}/lstm_cell/'.format(i)
                c, h = lstm_cell(inp, cs[i], hs[i], self._p(base + 'kernel'), self._p(base + 'bias'))
                new.append((c, h))
                inp = h if pos_key is None else self._dropout(h, 8 + i, pos_key[:, t], t=t)
            alive = (t < lengths).to(self.dtype).unsqueeze(-1)
            outs.append(inp * alive)
            cs = [alive * c + (1.0 - alive) * c0 for (c, _), c0 in zip(new, cs)]
            hs = [alive * h + (1.0 - alive) * h0 for (_, h), h0 in zip(new, hs)]
        return torch.stack(outs, dim=1)
