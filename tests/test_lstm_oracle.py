"""rnn_cell='lstm' on the CPU: the oracle's LSTM branch (oracle/lstm_ref.py) against outputs of the REFERENCE's own model
code, a hand-sized cell step, finite differences through two layers, and the parameter layout's TF-name round trip (for
the GRU as well).

tests/golden/lstm_golden.npz ran nar_model.py unmodified on the TF-1.x stand-in with an LSTMCell stand-in in place of
UGRNNCell (= un-commenting nar_model.py:1316; generator tests/golden/make_lstm_golden.py).  That pins the cell's place
and wiring in the graph; the cell arithmetic is the TF 1.12 rnn_cell_impl.py reading both sides restate."""
import math
import os

import numpy as np
import pytest
import torch

from chameleon_recsys_b200.harness import make_problem
from oracle.golden_sampling import preset_variables, sample_index
from oracle.lstm_ref import LstmOracle, lstm_cell
from tools.gpu_step_check import make_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'lstm_golden.npz')


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def _layout_name(n: str) -> str:
    n = n.replace('main/user_personalized_contextual_article_embedding/input/CAR_representation', 'main/CAR/CAR_representation')
    return n.replace('main/recommendations_ranking/cos_sim_positive/', 'main/recommendations_ranking/')


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _load(d, case, hp_over):
    P = case + '/'
    pb = make_problem('tiny', profile='B', rnn_cell='lstm', **hp_over)
    orc = make_oracle(pb, torch.float64)
    assert isinstance(orc, LstmOracle)
    tf_vars = preset_variables(d, case)
    assert set(_layout_name(n) for n in tf_vars) == set(pb.layout.init_logical(1).keys())   # same variables, same shapes
    for n, v in tf_vars.items():
        assert pb.layout.init_logical(1)[_layout_name(n)].shape == v.shape, n
    orc.set_params({_layout_name(n): v for n, v in tf_vars.items()})
    f = {k[len(P) + 5:]: d[k] for k in d.files if k.startswith(P + 'feat/')}
    lab = {k[len(P) + 6:]: d[k] for k in d.files if k.startswith(P + 'label/')}
    return pb, orc, f, lab, d[P + 'negatives'], d[P + 'buffer'], d[P + 'pop_norm'], tf_vars


def _masks(d, P):
    def unpack(n):
        shp = tuple(int(v) for v in d[P + 'mask_shape/' + n])
        return np.unpackbits(d[P + 'mask/' + n])[:int(np.prod(shp))].reshape(shp).astype(bool)
    rnn = unpack('rnn')                                      # [T, layers, B, H]
    over = {1: unpack('in'), 2: unpack('pos'), 3: unpack('neg'), 4: unpack('fc1')}
    for t in range(rnn.shape[0]):
        for i in range(rnn.shape[1]):
            over[(8 + i, t)] = rnn[t, i]
    return over


# (the float64 graphs agree to ~1e-10 in the loss and ~4e-9 in the logits: the reference run keeps float32 inputs - the
# millisecond timestamps, the sampled logits stored - where the oracle is float64 throughout)
@pytest.mark.parametrize('case,hp_over', [('lstm64', {}), ('lstm_drop64', {'dropout_keep_prob': 0.8, 'rnn_num_layers': 2})])
def test_train_graph_matches_reference_code(golden, case, hp_over):
    d = golden
    P = case + '/'
    pb, orc, f, lab, neg, buf, pop, tf_vars = _load(d, case, hp_over)
    assert sum('lstm_cell/kernel' in n for n in tf_vars) == pb.hp.rnn_num_layers
    kw = {}
    if (P + 'mask/rnn') in d.files:
        orc.mask_override = _masks(d, P)                    # the keep-masks the reference run drew
        kw = dict(train_step=1)
    o = orc.forward(f, lab, neg, buf, pop, **kw)
    mask = o['mask'].numpy().astype(bool)
    assert mask.sum() > 100
    assert abs(float(o['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) < 1e-9
    lg = o['logits'].detach().numpy()[mask].reshape(-1)
    ref = d[P + 'logits_sample']
    assert _rel(lg[sample_index(lg.size, ref.size)], ref) < 1e-8
    grads = orc.compute_gradients(o)
    gmax = max(float(np.abs(d[k]).max()) for k in d.files if k.startswith(P + 'grad/'))
    for n_tf in tf_vars:
        g_ref = d[P + 'grad/' + n_tf]
        g = grads[_layout_name(n_tf)].detach().numpy().reshape(-1)
        assert float(np.abs(g[sample_index(g.size, g_ref.size)] - g_ref).max()) < 1e-6 * gmax, n_tf
    if kw:
        # without the reference's masks the result differs: the comparison above is not vacuous
        orc.mask_override = None
        o2 = orc.forward(f, lab, neg, buf, pop, train_step=1)
        assert abs(float(o2['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) > 1e-4
    if (P + 'adam_delta/main/CAR/PreCAR_representation/bias') in d.files:
        before = orc.get_params()
        orc.apply_gradients(grads)
        after = orc.get_params()
        for n_tf in tf_vars:
            n = _layout_name(n_tf)
            ref = d[P + 'adam_delta/' + n_tf].astype(np.float64)
            delta = (after[n].astype(np.float64) - before[n].astype(np.float64)).reshape(-1)
            delta = delta[sample_index(delta.size, ref.size)]
            sel = np.abs(d[P + 'grad/' + n_tf].astype(np.float64)) > 1e-9 * gmax
            if sel.any():
                assert float(np.abs(delta - ref)[sel].max()) < 2e-3 * pb.hp.learning_rate, n_tf


def test_eval_graph_matches_reference_code(golden):
    d = golden
    P = 'lstm_eval64/'
    pb, orc, f, lab, neg, buf, pop, _ = _load(d, 'lstm_eval64', {})
    o = orc.forward(f, lab, neg, buf, pop)
    mask = o['mask'].numpy().astype(bool)
    assert abs(float(o['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) < 1e-9
    assert _rel(o['logits'].detach().numpy()[mask], d[P + 'logits_scaled'][mask]) < 1e-8
    ids, probs, hits, rr, cnt = orc.rank_and_metrics(o, lab, neg, pb.hp.eval_metrics_top_n)
    assert np.array_equal(np.asarray(ids)[mask], d[P + 'predicted_item_ids'][mask])
    assert _rel(np.asarray(probs)[mask], d[P + 'predicted_item_probs'][mask]) < 1e-8
    assert cnt == mask.sum()
    assert abs(hits / cnt - float(d[P + 'recall_at_n'])) < 1e-12
    assert abs(rr / cnt - float(d[P + 'mrr_at_n'])) < 1e-12


def test_cell_step_closed_form():
    """One LSTMCell step at H = 2, in = 1, worked by hand: forget_bias 1 enters the f gate only."""
    sig = lambda v: 1.0 / (1.0 + math.exp(-v))      # noqa: E731
    x = torch.tensor([[0.5]], dtype=torch.float64)
    c = torch.tensor([[0.2, -0.4]], dtype=torch.float64)
    h = torch.tensor([[0.1, 0.3]], dtype=torch.float64)
    kernel = torch.zeros(3, 8, dtype=torch.float64)
    kernel[0] = torch.tensor([1.0, -1.0, 2.0, 0.0, 0.5, 0.0, -2.0, 1.0])        # x row
    kernel[1, 0] = 1.0                                                         # h[0] -> i[0]
    kernel[2, 7] = -1.0                                                        # h[1] -> o[1]
    bias = torch.tensor([0.0, 0.1, 0.0, 0.0, 0.0, 0.0, 0.3, 0.0], dtype=torch.float64)
    c1, h1 = lstm_cell(x, c, h, kernel, bias)
    # pre-activations: i = (0.6, -0.4), j = (1.0, 0.0), f = (0.25, 0.0), o = (-0.7, 0.2)
    want_c = [sig(0.25 + 1) * 0.2 + sig(0.6) * math.tanh(1.0), sig(0.0 + 1) * -0.4 + sig(-0.4) * math.tanh(0.0)]
    want_h = [sig(-0.7) * math.tanh(want_c[0]), sig(0.2) * math.tanh(want_c[1])]
    assert np.allclose(c1.numpy()[0], want_c, rtol=0, atol=1e-15)
    assert np.allclose(h1.numpy()[0], want_h, rtol=0, atol=1e-15)


def test_finite_difference_gradients_two_layers():
    """fp64 central differences of a weighted sum of the two-layer output w.r.t. both layers' kernels and biases and the
    input, with sessions of length 0, 1, T and in between (the state is carried past a session's end)."""
    pb = make_problem('tiny', profile='A', rnn_cell='lstm', rnn_units=3, rnn_num_layers=2)
    orc = make_oracle(pb, torch.float64)
    rs = np.random.RandomState(0)
    n_in, H, B, T = 4, 3, 4, 5
    shapes = {'main/RNN/rnn/multi_rnn_cell/cell_0/lstm_cell/kernel': (n_in + H, 4 * H),
              'main/RNN/rnn/multi_rnn_cell/cell_0/lstm_cell/bias': (4 * H,),
              'main/RNN/rnn/multi_rnn_cell/cell_1/lstm_cell/kernel': (2 * H, 4 * H),
              'main/RNN/rnn/multi_rnn_cell/cell_1/lstm_cell/bias': (4 * H,)}
    names = list(shapes)
    x0 = torch.tensor(rs.randn(B, T, n_in))
    lengths = torch.tensor([0, 1, T, 3])
    w = torch.tensor(rs.randn(B, T, H))

    def f(x, *ps):
        orc.params = dict(zip(names, ps))
        return (orc.rnn(x, lengths) * w).sum()

    ps = [torch.tensor(rs.randn(*shapes[n]) * 0.6, requires_grad=True) for n in names]
    x = x0.clone().requires_grad_(True)
    assert torch.autograd.gradcheck(f, (x, *ps), eps=1e-6, atol=1e-8, rtol=1e-6)
    out = orc.rnn(x0, lengths).detach()
    assert not out[0].any() and not out[1, 1:].any() and not out[3, 3:].any()      # zero output past the length


def test_param_layout_round_trip_h255():
    """ParamLayout(rnn_cell='lstm' and 'gru') at H = 255 (Hp = 256), two layers: logical -> internal -> logical is exact,
    every TF column block lands in its Hp-wide block (LSTM i | j | f | o; GRU r | u from gates/*, c from candidate/*), the
    input rows and biases of a layer in one Wx / b, the recurrent rows in Wh (GRU: Wh and Whc), and the padding rows /
    columns stay zero."""
    # per cell and TF kernel: kernel, bias, column blocks, bias initialiser value, recurrent block, first block in Wx / b
    cells = {'lstm': [('lstm_cell/kernel', 'lstm_cell/bias', 4, 0.0, 'Wh', 0)],
             'gru': [('gru_cell/gates/kernel', 'gru_cell/gates/bias', 2, 1.0, 'Wh', 0),
                     ('gru_cell/candidate/kernel', 'gru_cell/candidate/bias', 1, 0.0, 'Whc', 2)]}
    for cell, kernels in cells.items():
        pb = make_problem('tiny', profile='B', rnn_cell=cell, rnn_units=255, rnn_num_layers=2)
        lay = pb.layout
        H, Hp, C = 255, 256, lay.C
        assert lay.Hp == Hp
        G = sum(n for _, _, n, _, _, _ in kernels)
        rs = np.random.RandomState(3)
        lg = {k: rs.randn(*v.shape).astype(np.float32) for k, v in lay.init_logical(1).items()}
        back = lay.to_logical(lay.to_internal(lg))
        assert sorted(back) == sorted(lg)
        for k in lg:
            assert np.array_equal(back[k], lg[k]), (cell, k)
        flat = lay.to_internal(lg)
        for i, n_in, n_in_p in ((0, C, C), (1, H, Hp)):
            base = 'main/RNN/rnn/multi_rnn_cell/cell_{}/'.format(i)
            want = {'Wx': np.zeros((n_in_p, G * Hp), np.float32), 'b': np.zeros((1, G * Hp), np.float32)}
            for kname, bname, n, _, wh, g0 in kernels:
                k, b = lg[base + kname], lg[base + bname]
                assert k.shape == (n_in + H, n * H) and b.shape == (n * H,)
                want[wh] = np.zeros((Hp, n * Hp), np.float32)
                for g in range(n):
                    col = (g0 + g) * Hp
                    want['Wx'][:n_in, col:col + H] = k[:n_in, g * H:(g + 1) * H]
                    want['b'][0, col:col + H] = b[g * H:(g + 1) * H]
                    want[wh][:H, g * Hp:g * Hp + H] = k[n_in:, g * H:(g + 1) * H]
            for key, m in want.items():
                t = lay.by_key['rnn%d/%s' % (i, key)]
                assert (t.rows, t.ld) == m.shape and not t.reg, (cell, i, key)       # not L2-regularised
                assert np.array_equal(flat[t.offset:t.offset + t.size].reshape(m.shape), m), (cell, i, key)
        # bias initialisers: LSTM zeros (forget_bias 1.0 is a constant of the cell); GRU gates ones, candidate zeros
        init = lay.init_logical(42)
        for _, bname, n, value, _, _ in kernels:
            assert np.array_equal(init['main/RNN/rnn/multi_rnn_cell/cell_0/' + bname], np.full(n * H, value, np.float32))
