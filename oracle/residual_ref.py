"""TEST INFRASTRUCTURE - the oracle with the reference's residual session stack (rnn_residual_connections=True).

nar_model.py:1308-1361 build_rnn takes `residual_connections` (default False; the call site :408 leaves it there).  Its
branch at :1319-1323 wraps every cell in tf.contrib.rnn.ResidualWrapper and layer 0 also in InputProjectionWrapper(.., H):

    layer 0:   DropoutWrapper(InputProjectionWrapper(ResidualWrapper(cell), H))   x -> P = x Wp + bp -> cell(P) + P
    layer i>0: DropoutWrapper(ResidualWrapper(cell))                               cell(x) + x

ResidualOracle is NarOracle (oracle/nar_oracle.py) with that stack in rnn(), for each of the three cells (UGRNN, GRU and,
with oracle/lstm_ref.lstm_cell, LSTM).  Everything else - features, CAR, FC1 / FC2, scorer, loss, Adam, the dropout
sites - is NarOracle's.  The state a cell carries to the next time step is its own h (and c), not the residual sum; the
DropoutWrapper drops the residual sum, which is what the next layer and FC1 see.

Pinning: tests/golden/residual_golden.npz comes from the reference's nar_model.py, unmodified, run on the eager TF-1.x
stand-in with build_rnn called with residual_connections=True (tests/golden/make_residual_golden.py).  The two wrappers'
behaviour is our reading of TF 1.12 rnn_cell_impl.py (ResidualWrapper) and contrib/rnn/.../core_rnn_cell.py
(InputProjectionWrapper: a _Linear with bias, no activation, in the scope input_projection_wrapper); TensorFlow itself
is unpinned.
"""
from __future__ import annotations

import torch

from .lstm_ref import lstm_cell
from .nar_oracle import NarOracle

RNN = 'main/RNN/rnn/multi_rnn_cell/'
PROJ = RNN + 'cell_0/input_projection_wrapper/'


def cell_scope(i: int, rnn_cell: str) -> str:
    """TF scope of layer i's cell in the residual stack: layer 0's cell sits inside the projection wrapper's scope."""
    return RNN + 'cell_{}/'.format(i) + ('input_projection_wrapper/' if i == 0 else '') + rnn_cell + '_cell/'


class ResidualOracle(NarOracle):
    def rnn(self, x, lengths, pos_key=None):
        """nar_model.py:1308-1342 with residual_connections=True inside dynamic_rnn(sequence_length): past a session's
        length the output is zero and the state is carried unchanged."""
        B, T, _ = x.shape
        H = self.H
        P = x @ self._p(PROJ + 'kernel') + self._p(PROJ + 'bias')            # InputProjectionWrapper, no activation
        hs = [torch.zeros(B, H, dtype=self.dtype) for _ in range(self.layers)]
        cs = [torch.zeros(B, H, dtype=self.dtype) for _ in range(self.layers)]
        outs = []
        for t in range(T):
            inp = P[:, t]
            new = []
            for i in range(self.layers):
                base = cell_scope(i, self.rnn_cell)
                c = cs[i]
                if self.rnn_cell == 'lstm':
                    c, h = lstm_cell(inp, cs[i], hs[i], self._p(base + 'kernel'), self._p(base + 'bias'))
                elif self.rnn_cell == 'gru':
                    gi = torch.cat([inp, hs[i]], dim=1) @ self._p(base + 'gates/kernel') + self._p(base + 'gates/bias')
                    r, u = torch.sigmoid(gi[:, :H]), torch.sigmoid(gi[:, H:])
                    cand = torch.tanh(torch.cat([inp, r * hs[i]], dim=1) @ self._p(base + 'candidate/kernel') +
                                      self._p(base + 'candidate/bias'))
                    h = u * hs[i] + (1.0 - u) * cand
                else:
                    m = torch.cat([inp, hs[i]], dim=1) @ self._p(base + 'kernel') + self._p(base + 'bias')
                    g = torch.sigmoid(m[:, :H] + 1.0)                         # forget_bias = 1.0
                    h = g * hs[i] + (1.0 - g) * torch.tanh(m[:, H:])
                new.append((c, h))
                out = h + inp                                                  # ResidualWrapper
                inp = out if pos_key is None else self._dropout(out, 8 + i, pos_key[:, t], t=t)
            alive = (t < lengths).to(self.dtype).unsqueeze(-1)
            outs.append(inp * alive)
            cs = [alive * c + (1.0 - alive) * c0 for (c, _), c0 in zip(new, cs)]
            hs = [alive * h + (1.0 - alive) * h0 for (_, h), h0 in zip(new, hs)]
        return torch.stack(outs, dim=1)
