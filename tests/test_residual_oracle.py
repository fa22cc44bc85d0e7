"""rnn_residual_connections=True on the CPU: the oracle's residual session stack (oracle/residual_ref.py) against outputs
of the REFERENCE's own model code, finite differences through the projection and the skip paths, the parameter layout,
and the params dict with the switch off.

tests/golden/residual_golden.npz ran nar_model.py unmodified on the TF-1.x stand-in with build_rnn called with
residual_connections=True (generator tests/golden/make_residual_golden.py, which adds ResidualWrapper and
InputProjectionWrapper to the stand-in).  That pins the wrappers' place and wiring in the graph and the variable names;
the wrappers' arithmetic is the TF 1.12 reading both sides restate."""
import os

import numpy as np
import pytest
import torch

from chameleon_recsys_b200.harness import make_problem
from chameleon_recsys_b200.hparams import NARHParams
from oracle.golden_sampling import preset_variables, sample_index
from oracle.residual_ref import ResidualOracle
from tools.gpu_step_check import make_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'residual_golden.npz')
RNN = 'main/RNN/rnn/multi_rnn_cell/'
PROJ = RNN + 'cell_0/input_projection_wrapper/'

CASES = {'res64': dict(), 'res_drop64': dict(dropout_keep_prob=0.8, rnn_num_layers=3),
         'res_gru64': dict(rnn_cell='gru', rnn_num_layers=2), 'res_lstm64': dict(rnn_cell='lstm', rnn_num_layers=2),
         'res_eval64': dict(rnn_num_layers=2)}


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


def _load(d, case):
    P = case + '/'
    pb = make_problem('tiny', profile='B', rnn_units=48, rnn_residual_connections=True, **CASES[case])
    orc = make_oracle(pb, torch.float64)
    assert isinstance(orc, ResidualOracle)
    tf_vars = preset_variables(d, case)
    init = pb.layout.init_logical(1)
    assert set(_layout_name(n) for n in tf_vars) == set(init)          # same variables, same shapes
    for n, v in tf_vars.items():
        assert init[_layout_name(n)].shape == v.shape, n
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


# the bars of tests/test_lstm_oracle.py: the float64 graphs agree to ~1e-10 in the loss and ~4e-9 in the logits (the
# reference run keeps some float32 inputs)
@pytest.mark.parametrize('case', ['res64', 'res_drop64', 'res_gru64', 'res_lstm64'])
def test_train_graph_matches_reference_code(golden, case):
    d = golden
    P = case + '/'
    pb, orc, f, lab, neg, buf, pop, tf_vars = _load(d, case)
    assert sum(n.endswith('_cell/kernel') or n.endswith('gates/kernel') for n in tf_vars) == pb.hp.rnn_num_layers
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
    assert np.abs(d[P + 'grad/' + PROJ + 'kernel']).max() > 1e-3 * gmax      # the projection is on the gradient path
    if kw:
        orc.mask_override = None                            # without the reference's masks the result differs
        o2 = orc.forward(f, lab, neg, buf, pop, train_step=1)
        assert abs(float(o2['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) > 1e-4
    if (P + 'adam_delta/' + PROJ + 'kernel') in d.files:
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


def test_train_graph_differs_without_residual(golden):
    """The plain stack on the same inputs (the layer-0 cell fed E instead of the projection, no skip paths) does not
    reproduce the golden loss: the comparison above tests the residual wiring."""
    d = golden
    P = 'res64/'
    pb, orc, f, lab, neg, buf, pop, tf_vars = _load(d, 'res64')
    o = orc.forward(f, lab, neg, buf, pop)
    plain = make_oracle(pb, torch.float64, residual=False)
    params = {k: v.detach().numpy() for k, v in orc.params.items()}
    k0 = params[PROJ + 'ugrnn_cell/kernel']
    W = params[PROJ + 'kernel']                                      # fold the projection into a [C + H, 2H] kernel
    params[RNN + 'cell_0/ugrnn_cell/kernel'] = np.concatenate([W @ k0[:48], k0[48:]])
    params[RNN + 'cell_0/ugrnn_cell/bias'] = params[PROJ + 'ugrnn_cell/bias'] + params[PROJ + 'bias'] @ k0[:48]
    plain.set_params(params)
    o2 = plain.forward(f, lab, neg, buf, pop)
    ref = float(d[P + 'total_loss'])
    assert abs(float(o['total_loss'].detach()) - ref) / abs(ref) < 1e-9
    assert abs(float(o2['total_loss'].detach()) - ref) / abs(ref) > 1e-4


def test_eval_graph_matches_reference_code(golden):
    d = golden
    P = 'res_eval64/'
    pb, orc, f, lab, neg, buf, pop, _ = _load(d, 'res_eval64')
    o = orc.forward(f, lab, neg, buf, pop)
    mask = o['mask'].numpy().astype(bool)
    assert abs(float(o['total_loss'].detach()) - float(d[P + 'total_loss'])) / abs(float(d[P + 'total_loss'])) < 1e-9
    assert _rel(o['logits'].detach().numpy()[mask], d[P + 'logits_scaled'][mask]) < 1e-8
    ids, probs, hits, rr, cnt = orc.rank_and_metrics(o, lab, neg, pb.hp.eval_metrics_top_n)
    assert np.array_equal(np.asarray(ids)[mask], d[P + 'predicted_item_ids'][mask])
    # the probabilities are a softmax of the logits at temperature 0.1: ten times their error (measured 1.2e-8)
    assert _rel(np.asarray(probs)[mask], d[P + 'predicted_item_probs'][mask]) < 1e-7
    assert cnt == mask.sum()
    assert abs(hits / cnt - float(d[P + 'recall_at_n'])) < 1e-12
    assert abs(rr / cnt - float(d[P + 'mrr_at_n'])) < 1e-12


@pytest.mark.parametrize('cell', ['ugrnn', 'gru', 'lstm'])
def test_finite_difference_gradients(cell):
    """fp64 central differences of a weighted sum of a two-layer residual stack's output w.r.t. Wp, bp, both layers'
    cell variables and the input, with sessions of length 0, 1, T and in between (the state is carried past a session's
    end), and with the cells' kernels zeroed so that only the skip paths carry the gradient."""
    pb = make_problem('tiny', profile='A', rnn_cell=cell, rnn_units=3, rnn_num_layers=2, rnn_residual_connections=True)
    orc = make_oracle(pb, torch.float64)
    rs = np.random.RandomState(0)
    n_in, H, B, T = 4, 3, 4, 5
    G = {'ugrnn': 2, 'gru': 2, 'lstm': 4}[cell]
    shapes = {PROJ + 'kernel': (n_in, H), PROJ + 'bias': (H,)}
    for i in range(2):
        base = RNN + 'cell_%d/' % i + ('input_projection_wrapper/' if i == 0 else '') + cell + '_cell/'
        if cell == 'gru':
            shapes.update({base + 'gates/kernel': (2 * H, 2 * H), base + 'gates/bias': (2 * H,),
                           base + 'candidate/kernel': (2 * H, H), base + 'candidate/bias': (H,)})
        else:
            shapes.update({base + 'kernel': (2 * H, G * H), base + 'bias': (G * H,)})
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
    # cells whose kernels are zero: UGRNN / GRU / LSTM outputs are then functions of the biases only, and the gradient
    # w.r.t. the input reaches it through the projection and the two skip paths alone: d out / d x = Wp (per live step)
    zs = [torch.zeros_like(p) if (n.endswith('kernel') and n != PROJ + 'kernel') else p.detach() for n, p in zip(names, ps)]
    xg = x0.clone().requires_grad_(True)
    gx, = torch.autograd.grad(f(xg, *zs), xg)
    want = (w @ zs[0].t()) * (torch.arange(T)[None, :] < lengths[:, None]).unsqueeze(-1).to(w.dtype)
    assert torch.allclose(gx, want, rtol=0, atol=1e-12)


def test_param_layout():
    """ParamLayout(residual=True) at H = 255 (Hp = 256), C 64, two layers: rnn0/Wp [C, Hp] and rnn0/bp [Hp] under the
    projection's TF names, unregularised, padded columns zero; layer 0's Wx has Hp input rows and its TF kernel [2H, G*H]
    lives under the projection wrapper's scope; layer 1 keeps its names; logical -> internal -> logical is exact."""
    for cell, G in (('ugrnn', 2), ('gru', 3), ('lstm', 4)):
        pb = make_problem('tiny', profile='B', rnn_cell=cell, rnn_units=255, rnn_num_layers=2, rnn_residual_connections=True)
        lay = pb.layout
        C, H, Hp = lay.C, 255, 256
        assert lay.residual and lay.Hp == Hp
        wp, bp = lay.by_key['rnn0/Wp'], lay.by_key['rnn0/bp']
        assert (wp.tf_name, wp.logical_shape, wp.rows, wp.ld, wp.reg) == (PROJ + 'kernel', (C, H), C, Hp, False)
        assert (bp.tf_name, bp.logical_shape, bp.rows, bp.ld, bp.reg) == (PROJ + 'bias', (H,), 1, Hp, False)
        assert wp.offset >= lay.reg_end and bp.offset >= lay.reg_end
        wx0, wx1 = lay.by_key['rnn0/Wx'], lay.by_key['rnn1/Wx']
        assert (wx0.rows, wx0.ld) == (Hp, G * Hp) and (wx1.rows, wx1.ld) == (Hp, G * Hp)
        assert all(not t.reg for t in lay.tensors if '/RNN/' in t.tf_name)
        names = lay.logical_names()
        k0 = [n for n in names if n.startswith(PROJ) and n.endswith('kernel') and n != PROJ + 'kernel']
        assert k0 and all(n.startswith(PROJ + cell + '_cell/') for n in k0)
        assert not any(n.startswith(RNN + 'cell_0/' + cell) for n in names)
        assert any(n.startswith(RNN + 'cell_1/' + cell + '_cell/') for n in names)
        init = lay.init_logical(5)
        assert init[PROJ + 'kernel'].shape == (C, H) and np.array_equal(init[PROJ + 'bias'], np.zeros(H, np.float32))
        for n in k0:
            assert init[n].shape[0] == 2 * H, n
        rs = np.random.RandomState(3)
        lg = {k: rs.randn(*v.shape).astype(np.float32) for k, v in init.items()}
        flat = lay.to_internal(lg)
        back = lay.to_logical(flat)
        assert sorted(back) == sorted(lg) and all(np.array_equal(back[k], lg[k]) for k in lg)
        Wp = flat[wp.offset:wp.offset + wp.size].reshape(C, Hp)
        assert np.array_equal(Wp[:, :H], lg[PROJ + 'kernel']) and not Wp[:, H:].any()
        assert not flat[bp.offset + H:bp.offset + Hp].any()
        Wx0 = flat[wx0.offset:wx0.offset + wx0.size].reshape(Hp, G * Hp)
        assert not Wx0[H:].any()
    # the plain layout is unchanged by the switch's existence
    a = make_problem('tiny', profile='B', rnn_num_layers=2).layout
    assert not a.residual and 'rnn0/Wp' not in a.by_key and a.by_key['rnn0/Wx'].rows == a.C


def test_params_dict_unchanged_when_off():
    """to_params writes 'rnn_residual_connections' only when it is True, like the other extensions."""
    pb = make_problem('tiny', profile='B')
    args = (pb.session_features_config, pb.articles_features_config, pb.articles_metadata, pb.content_article_embeddings_matrix)
    off = NARHParams().to_params(*args)
    assert 'rnn_residual_connections' not in off
    assert NARHParams(rnn_residual_connections=False).to_params(*args).keys() == off.keys()
    on = NARHParams(rnn_residual_connections=True).to_params(*args)
    assert on.pop('rnn_residual_connections') is True and on.keys() == off.keys()
