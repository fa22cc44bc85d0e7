"""How csrc/engine.cu's run_step wires the residual session stack (rnn_residual_connections=True, DESIGN.md section 15)
against the fp64 oracle (oracle/residual_ref.py) at 3xTF32, and nar_residual_add bit for bit (pytest -m gpu).

The residual stack adds its own wiring to the training step: the projection P = E Wp + bp, nar_residual_add after every
layer, the layer-input dgrad accumulated onto the gradient of the layer's output (for layer 0 that is dP), the Wp dgrad
with the tanh epilogue, dWp / dbp on the auxiliary stream, the dropout masks re-applied to a gradient that also carries
the skip path, and a bf16x3 plane for Wp.  tests/test_residual_gpu.py checks the stack at the loose bars of
tests/test_gpu_parity.py (3e-2 per gradient); here every case meets the bars of tests/test_step_wiring_gpu.py unchanged,
with its machinery (measure, check): negatives bit-exact; xe, L2 and novelty losses, logits, per-tensor gradients and
touched embedding rows against fp64; exact zeros; a zero gradient and a zero value at every padding entry of the flat
buffer, Wp[:, H:Hp] and bp[H:Hp] included; per-element TF-Adam with the regularised tensors taken from the oracle (so Wp
and bp inside the L2 range fail); no non-finite value.  rnn_units is 48 (Hp 64) unless a case says otherwise, so the
projection and every layer carry padded columns; at 64 Wp is square with no padding, at 300 it pads to Hp 512, and at
CAR_embedding_size 100 the projection GEMM has K = 100.

Worst values measured over every case here on an H100 80GB HBM3 at its 700 W power limit, against the step-wiring bars
(the worst case in brackets).  Every one is within the bar, so none is loosened:
    LOSS_TOL          1.5e-5   8.5e-6 (ugrnn-cold-b2)
    LOGIT_TOL         1.5e-4   3.7e-5 (lstm-g1; tiny cases <= 1.5e-5)
    GRAD_TOL          1e-4     5.0e-5 (lstm-g1; tiny cases <= 2.3e-5, lstm-H300)
    ROW_TOL           1.5e-4   4.9e-5 (lstm-g1)
    ADAM_TOL          1e-6     2.8e-7 (lstm-g1)
    SUM_ZERO_ABS      2e-6     1.7e-6 (lstm-cold-b2, matching_dense_layer_4/bias)
    GRAD_TOL_DEFAULT  3e-2     7.7e-3 (ugrnn-default-precision)

The unsynced 30-step trajectory is held to TRAJ_TOL = 5e-3, not to the plain stack's 1e-3, because the residual stack
carries rounding further along a trajectory than the plain stack does, and the 1e-3 bar is smaller than that effect.
Measured over the same 30 G1 batches (batch 64), as the largest relative loss gap:
- the fp32 oracle against the fp64 oracle, each on its own Adam path, on the CPU.  Both compute the same model and
  differ only in rounding: 1.20e-3 ugrnn, 1.04e-3 gru, 1.36e-3 lstm with the residual stack; 4.1e-4 ugrnn without it;
- the engine against the fp32 oracle, on the H100: 1.00e-3 ugrnn, 1.35e-3 gru, 8.8e-4 lstm at the default precision;
  1.45e-3 ugrnn, 1.48e-3 gru with 3xTF32 forward and backward, so a more precise engine is not closer.  Without the
  residual stack the gap was 5.6e-4 ugrnn and 5.3e-4 gru in the same run.
The gap therefore comes from rounding, amplified by the trajectory, and not from the engine's arithmetic.  TRAJ_TOL is
3.4x the worst engine value.  Whether the weights reach the forward GEMMs after every update does not rest on this bar:
test_planes_follow_adam_updates checks the bf16x3 planes bit for bit.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from test_step_wiring_gpu import (CELLS, EXEMPT, GRAD_TOL, LOGIT_TOL, LOSS_TOL, SOFTMAX_SUMS, _engine,  # noqa: E402
                                  _one_label, _padding_mask, _state, check, measure)

pytestmark = pytest.mark.gpu

RES = dict(rnn_residual_connections=True)
TINY = dict(RES, rnn_units=48)
# largest relative loss gap over a 30-step unsynced trajectory (the plain stack's bar is 1e-3): see the module docstring
TRAJ_TOL = 5e-3


def _cases():
    c = {}
    for cell in CELLS:
        for layers in (1, 2, 4):
            for rk in ('mlp', 'cosine'):
                c['%s-%dl-%s' % (cell, layers, rk)] = dict(hp=dict(rnn_num_layers=layers, ranking=rk))
        # dropout: every candidate row materialised (dedup off); the masks of layers 0 .. n-1 are re-applied to a
        # gradient that also carries the skip path
        c[cell + '-drop-2l'] = dict(hp=dict(rnn_num_layers=2, dropout_keep_prob=0.7))
        c[cell + '-drop-4l'] = dict(hp=dict(rnn_num_layers=4, dropout_keep_prob=0.7))
        c[cell + '-nov-mlp'] = dict(hp=dict(novelty_reg_factor=0.5))
        c[cell + '-nov-cosine'] = dict(hp=dict(novelty_reg_factor=0.5, ranking='cosine'))
        c[cell + '-every-row'] = dict(ekw=dict(dedup=False))
        c[cell + '-profileA'] = dict(profile='A')
        # two sessions, empty buffer: zero-padded negatives and the padding slot of the per-unique-id layer 1
        c[cell + '-cold-b2'] = dict(hp=dict(batch_size=2), warm=0)
        c[cell + '-one-label'] = dict(batch_map=_one_label)
        c[cell + '-C100'] = dict(hp=dict(CAR_embedding_size=100))
        # 64: H == C == Hp, a square Wp without padding; 300 pads to Hp 512
        for H in (30, 64, 255, 300):
            c['%s-H%d' % (cell, H)] = dict(hp=dict(rnn_units=H))
        # bf16x3 forward (the Wp plane) and single-pass TF32 backward, at that precision's bar
        c[cell + '-default-precision'] = dict(hp=dict(rnn_num_layers=2), prec=(4, 1))
    # realistic tile and split-K counts: C 1024, H 255 (Hp 256), K 50, 46K items
    for cell in ('ugrnn', 'lstm'):
        c[cell + '-g1'] = dict(name='g1', hp=dict(batch_size=16), warm=30)
    for name, cfg in c.items():
        hp = cfg.setdefault('hp', {})
        hp['rnn_cell'] = name.split('-')[0]
        hp.update(RES if cfg.get('name') == 'g1' else dict(TINY, **hp))
    return c


CASES = _cases()


@pytest.mark.parametrize('case', sorted(CASES))
def test_step_matches_fp64(case):
    check(measure(case, CASES))


# ------------------------------------------------------------------------------------------------ edges
@pytest.mark.parametrize('cell', CELLS)
def test_step_without_labelled_positions(cell):
    """L = 0 after a real step: gradients and loss exactly 0, and submit leaves weights, Adam slots and step alone."""
    pb, eng, _ = _engine(cell, rnn_num_layers=2, **TINY)
    it = pb.input_fn()
    buf, pop = _state(pb)
    eng.train_step(*it.get_next(), buf, pop)
    assert float(eng.grads.abs().max()) > 0 and float(eng.view('rnn0/Wp', eng.grads).abs().max()) > 0
    f, l = it.get_next()
    f = dict(f); f['session_size'] = np.minimum(f['session_size'], 1)
    before = [t.clone() for t in (eng.params, eng.adam_m, eng.adam_v)]
    step = eng.global_step
    st = eng.stage(f, l, buf, pop)
    assert st['L'] == 0
    eng.grads.fill_(float('nan')); eng.loss_dev.fill_(float('nan'))
    out = eng.result(eng.submit(st))
    assert out['xe_loss'] == 0.0 and out['reg_loss'] == 0.0 and out['nov_reg_loss'] == 0.0
    assert not eng.grads.any() and not eng.loss_dev.isnan().any()
    assert all(bool((a == b).all()) for a, b in zip(before, (eng.params, eng.adam_m, eng.adam_v)))
    assert eng.global_step == step


@pytest.mark.parametrize('cell', CELLS)
def test_two_ranks_sum_to_the_whole_batch(cell):
    """Data parallel emulated in one process (world 2, rank 0 and 1 on one device), 2 residual layers: each rank's shard
    gradient, summed, and the losses, summed, against the oracle's whole batch at the tight bars.  Only rank 0 adds the
    L2 term, and it covers the tensors the oracle regularises: Wp and bp lie past the regularised range."""
    import torch
    from oracle import sampler_ref
    from tools import gpu_step_check as g
    pb, _, orc = _engine(cell, rnn_num_layers=2, **TINY)
    hp, lay = pb.hp, pb.layout
    assert min(lay.by_key['rnn0/Wp'].offset, lay.by_key['rnn0/bp'].offset) >= lay.reg_end
    f, l = pb.input_fn().get_next()
    buf, pop = _state(pb)
    logical = lay.init_logical(hp.init_seed)
    gsum, losses, lasts, negs = None, [], [], []
    for r in range(2):
        e = g.make_engine(pb, fwd_precision=3, bwd_precision=3)
        e.set_params(logical)
        e.world, e.rank = 2, r
        st = e.stage(f, l, buf, pop)
        e.grads.fill_(float('nan')); e.loss_dev.fill_(float('nan'))
        o = e.step(st, train=True, keep=True)
        torch.cuda.synchronize()
        gsum = e.grads.double().clone() if gsum is None else gsum + e.grads.double()
        losses.append(e.loss_dev.double().cpu().numpy().copy())
        lasts.append({k: v for k, v in e.last.items()})
        negs.append(o['negatives'].cpu().numpy())
        assert st['L'] > 0
    allc = np.concatenate([f['item_clicked'], l['label_last_item']], axis=1)
    K = hp.train_total_negative_samples
    neg = sampler_ref.sample_negatives(allc, buf, K, hp.train_negative_samples_from_buffer, hp.sampler_seed, 1)
    assert np.array_equal(np.concatenate(negs, 0), neg)
    w = {k: v.detach().clone() for k, v in orc.params.items()}
    o, grads = orc.train_step(f, l, neg, buf, pop, kinks=g.engine_kinks(lasts, f['session_size'], f['item_clicked'].shape[1], K + 1))
    xe, reg = float(o['xe_loss']), float(o['reg_loss'])
    assert reg > 0
    assert abs(losses[0][0] + losses[1][0] - xe) / xe <= LOSS_TOL
    assert abs(losses[0][1] - reg) / reg <= LOSS_TOL and losses[1][1] == 0.0
    got = lay.to_logical(gsum.cpu().numpy())
    assert any('input_projection_wrapper/kernel' in k for k in grads)
    for k, gr in grads.items():
        gr = gr.detach()
        if orc.regularised(k):
            gr = gr - orc.reg * w[k]
        gr = gr.numpy()
        if k not in SOFTMAX_SUMS:
            assert not got[k][gr == 0].any(), k
        if k != EXEMPT and np.abs(gr).max() > 0:
            assert np.abs(got[k] - gr).max() <= GRAD_TOL * np.abs(gr).max(), k
    assert not gsum.cpu().numpy()[_padding_mask(lay)].any()


@pytest.mark.parametrize('cell', CELLS)
def test_eval_step_matches_fp64(cell):
    """eval_step (no dropout, no gradients) at fwd_precision 3, 2 residual layers with dropout and novelty configured:
    logits and losses against the oracle's forward."""
    import torch
    from oracle import sampler_ref
    pb, eng, orc = _engine(cell, rnn_num_layers=2, dropout_keep_prob=0.7, novelty_reg_factor=0.5, **TINY)
    hp = pb.hp
    f, l = pb.input_fn().get_next()
    buf, pop = _state(pb)
    eng.loss_dev.fill_(float('nan'))
    out = eng.eval_step(f, l, buf, pop, top_n=3, step_id=1, keep=True)
    allc = np.concatenate([f['item_clicked'], l['label_last_item']], axis=1)
    neg = sampler_ref.sample_negatives(allc, buf, hp.train_total_negative_samples, hp.train_negative_samples_from_buffer,
                                       hp.sampler_seed, 1)
    assert np.array_equal(out['negatives'].cpu().numpy(), neg)
    with torch.no_grad():
        o = orc.forward(f, l, neg, buf, pop)
    mask = o['mask'].numpy()
    lg, lg_ref = out['logits'].cpu().numpy(), o['logits'].numpy()[mask]
    assert np.abs(lg - lg_ref).max() <= LOGIT_TOL * np.abs(lg_ref).max()
    for key in ('xe_loss', 'reg_loss', 'nov_reg_loss'):
        assert abs(out[key] - float(o[key])) <= LOSS_TOL * abs(float(o[key])), key


@pytest.mark.parametrize('cell', CELLS)
def test_unsynced_trajectory_g1(cell):
    """30 steps at G1 (batch 64, H 255 -> Hp 256), default precision, each side on its own Adam trajectory: the engine's
    updates feed its forward GEMMs through the refreshed bf16x3 planes, Wp's included, and the loss stays within
    TRAJ_TOL relative of the fp32 oracle's."""
    import torch
    from tools import gpu_step_check as g
    res = g.run_trajectory('g1', 'B', 30, 30, hp_over=dict(RES, batch_size=64, rnn_cell=cell), oracle_dtype=torch.float32)
    assert all(s['neg_equal'] for s in res['steps'])
    assert res['max_rel'] < TRAJ_TOL, [(s['step'], s['rel']) for s in res['steps'] if s['rel'] >= TRAJ_TOL]


@pytest.mark.parametrize('cell', CELLS)
def test_planes_follow_adam_updates(cell):
    """Default precision, 2 residual layers: after 3 Adam steps an EVAL step gives, bit for bit, the logits of a fresh
    engine that packs its bf16x3 planes from the trained weights, and not those of the initial weights.  So every
    forward plane, Wp's included, follows the updates (a plane left at the initial weights would fail the first)."""
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools import gpu_step_check as g
    pb = make_problem('tiny', profile='B', rnn_cell=cell, rnn_num_layers=2, **TINY)
    warm_state(pb, 5)
    logical = pb.layout.init_logical(pb.hp.init_seed)
    eng = g.make_engine(pb)
    assert (eng.fwd_prec, eng.bwd_prec) == (4, 1)
    eng.set_params(logical)
    it = pb.input_fn()
    st = pb.clicked_items_state
    for _ in range(3):
        f, l = it.get_next()
        eng.train_step(f, l, *_state(pb))
        st.update_from_batch(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
    f, l = it.get_next()
    fresh, init = g.make_engine(pb), g.make_engine(pb)
    fresh.set_params(eng.get_params())
    init.set_params(logical)
    fresh.global_step = init.global_step = eng.global_step        # the same evaluation negatives
    outs = [e.eval_step(f, l, *_state(pb), top_n=3) for e in (eng, fresh, init)]
    assert all(torch.equal(o['negatives'], outs[0]['negatives']) for o in outs)
    trained, again, first = (o['logits'] for o in outs)
    assert torch.equal(trained, again)
    assert not torch.equal(trained, first)


def test_estimator_runs_hp_1024(tmp_path):
    """rnn_units 1000 (Hp 1024), LSTM, 2 residual layers: train, evaluate and predict through Estimator give finite
    results, and every padding entry (Wp[:, 1000:1024] and bp[1000:1024] among them) stays zero in the weights and the
    Adam slots."""
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B', rnn_cell='lstm', rnn_num_layers=2, batch_size=24, **dict(RES, rnn_units=1000))
    assert pb.layout.Hp == 1024
    warm_state(pb, 5)
    est = build_estimator(str(tmp_path), pb.content_article_embeddings_matrix, pb.articles_metadata,
                          pb.articles_features_config, pb.session_features_config, pb.hp, pb.clicked_items_state, device=0)
    est.train(pb.input_fn, steps=3)
    assert np.isfinite(est.last_loss)
    ev = est.evaluate(pb.input_fn, steps=2)
    assert np.isfinite(ev['loss']) and 0.0 <= ev['hitrate_at_n'] <= 1.0
    batch = pb.input_fn().get_next()
    preds = list(est.predict(lambda: iter([batch]), top_n=5, candidates='catalog'))
    assert preds and all(np.isfinite(p['predicted_item_scores']).all() for p in preds)
    eng = est.model.engine
    assert float(eng.view('rnn0/Wp')[:, :1000].abs().max()) > 0
    pad = _padding_mask(pb.layout)
    for buf in (eng.params, eng.adam_m, eng.adam_v):
        assert not buf.cpu().numpy()[pad].any()


# ------------------------------------------------------------------------------------------------ nar_residual_add
NAR_ERR_INVALID = -1
SENT_BITS = 0x7FA5A5A5          # a NaN no add produces: the sentinel of every entry a call must not write
GUARD_ROWS = 3


def _lib():
    from chameleon_recsys_b200 import _lib as lib_mod, ops
    return lib_mod.load(), ops


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


def _operands(rows, cols, ld, seed):
    """h and res [rows + GUARD_ROWS, ld] (padding columns and guard rows 7.0 and 9.0): normals over 80 orders of
    magnitude, with +-inf, inf - inf, NaN, -0 + 0, -0 + -0, subnormal sums, exact cancellations and overflow to inf."""
    rs = np.random.RandomState(seed)
    n = (rows, cols)
    h = (rs.standard_normal(n) * np.exp(rs.uniform(-40, 40, n))).astype(np.float32)
    r = (rs.standard_normal(n) * np.exp(rs.uniform(-40, 40, n))).astype(np.float32)
    k = rs.randint(0, 16, n)
    sub = lambda: (rs.randint(-(1 << 23) + 1, 1 << 23, n) * np.float32(2.0 ** -149)).astype(np.float32)  # noqa: E731
    for code, hv, rv in ((0, np.inf, None), (1, -np.inf, np.inf), (2, np.nan, None), (3, -0.0, 0.0), (4, -0.0, -0.0),
                         (5, sub(), sub()), (6, None, None), (7, 3e38, 3e38), (8, -np.inf, None), (9, None, np.nan)):
        m = k == code
        if hv is not None:
            h[m] = hv[m] if isinstance(hv, np.ndarray) else hv
        if rv is not None:
            r[m] = rv[m] if isinstance(rv, np.ndarray) else rv
    r[k == 6] = -h[k == 6]
    H = np.full((rows + GUARD_ROWS, ld), 7.0, np.float32)
    R = np.full((rows + GUARD_ROWS, ld), 9.0, np.float32)
    H[:rows, :cols], R[:rows, :cols] = h, r
    return H, R


def _want(H, R, rows, cols):
    with np.errstate(all='ignore'):
        return H[:rows, :cols] + R[:rows, :cols]          # numpy float32: IEEE round-to-nearest, no flush to zero


def _same(got, want):
    """bit for bit, except that a NaN's payload is the hardware's: NaN exactly where the IEEE sum is NaN"""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


def _call(lib, ops, h, res, rows, cols, ld, out):
    p = lambda x: x if isinstance(x, C.c_void_p) or x is None else ops._p(x)  # noqa: E731
    return lib.nar_residual_add(p(h), p(res), rows, cols, ld, p(out), ops._stream())


@pytest.mark.parametrize('pad', [0, 4, 60])
@pytest.mark.parametrize('cols', [4, 48, 64, 1024])
@pytest.mark.parametrize('rows', [1, 3, 257, 4096])
def test_residual_add_bits(rows, cols, pad):
    """out = h + res bit for bit with numpy's float32 add, ld = cols + pad; the columns [cols, ld) and the guard rows past
    `rows` keep the sentinel.  At 4096 x 1024 there are 1M float4 elements and the capped grid (132 * 8 blocks of 256
    threads) has 270K threads: the grid-stride loop wraps."""
    import torch
    lib, ops = _lib()
    ld = cols + pad
    H, R = _operands(rows, cols, ld, rows * 131 + cols * 7 + pad)
    h, r = torch.from_numpy(H).cuda(), torch.from_numpy(R).cuda()
    out = torch.from_numpy(np.full(H.shape, SENT_BITS, np.uint32).view(np.float32)).cuda()
    assert _call(lib, ops, h, r, rows, cols, ld, out) == 0
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    _same(got[:rows, :cols], _want(H, R, rows, cols))
    b = _bits(out)
    assert (b[:rows, cols:] == SENT_BITS).all() and (b[rows:] == SENT_BITS).all()
    assert np.array_equal(h.cpu().numpy().view(np.uint32), H.view(np.uint32))
    assert np.array_equal(r.cpu().numpy().view(np.uint32), R.view(np.uint32))


@pytest.mark.parametrize('alias', ['h', 'res'])
@pytest.mark.parametrize('rows, cols, pad', [(3, 48, 4), (257, 64, 60), (4096, 1024, 4)])
def test_residual_add_in_place(rows, cols, pad, alias):
    """out is h, or out is res (as the header allows): the same bits, the aliased buffer's padding and guard rows
    untouched, the other operand unchanged."""
    import torch
    lib, ops = _lib()
    ld = cols + pad
    H, R = _operands(rows, cols, ld, rows + cols + pad)
    h, r = torch.from_numpy(H).cuda(), torch.from_numpy(R).cuda()
    out, keep, KEEP = (h, r, R) if alias == 'h' else (r, h, H)
    ALIAS = H if alias == 'h' else R
    assert _call(lib, ops, h, r, rows, cols, ld, out) == 0
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    _same(got[:rows, :cols], _want(H, R, rows, cols))
    assert np.array_equal(got[:rows, cols:].view(np.uint32), ALIAS[:rows, cols:].view(np.uint32))
    assert np.array_equal(got[rows:].view(np.uint32), ALIAS[rows:].view(np.uint32))
    assert np.array_equal(keep.cpu().numpy().view(np.uint32), KEEP.view(np.uint32))


def _small():
    import torch
    h = torch.ones(8, 16, device='cuda')
    r = torch.ones(8, 16, device='cuda')
    out = torch.from_numpy(np.full((8, 16), SENT_BITS, np.uint32).view(np.float32)).cuda()
    return h, r, out


@pytest.mark.parametrize('rows, cols', [(0, 8), (-1, 8), (4, 0)])
def test_residual_add_nothing_to_do(rows, cols):
    """rows <= 0 or cols = 0: OK, and nothing written."""
    import torch
    lib, ops = _lib()
    h, r, out = _small()
    assert _call(lib, ops, h, r, rows, cols, 16, out) == 0
    torch.cuda.synchronize()
    assert (_bits(out) == SENT_BITS).all()


@pytest.mark.parametrize('which', ['h_null', 'res_null', 'out_null', 'cols_not_x4', 'ld_not_x4', 'ld_below_cols',
                                   'cols_negative', 'h_misaligned', 'res_misaligned', 'out_misaligned'])
def test_residual_add_rejects(which):
    """Null pointers, cols or ld not a multiple of 4, ld < cols, cols < 0 and a pointer off 16-byte alignment return
    NAR_ERR_INVALID and write nothing.  The misaligned views (one float past an allocation's start) come with rows = 0,
    so the check must come before the nothing-to-do return, and no kernel ever runs on them."""
    import torch
    lib, ops = _lib()
    h, r, out = _small()
    a = dict(h=h, res=r, out=out, rows=4, cols=8, ld=16)
    if which.endswith('_null'):
        a[which[:-5]] = None
    elif which.endswith('_misaligned'):
        k = which[:-11]
        a[k] = C.c_void_p(a[k].data_ptr() + 4)
        a['rows'] = 0
    else:
        a.update({'cols_not_x4': dict(cols=6), 'ld_not_x4': dict(ld=18), 'ld_below_cols': dict(cols=16, ld=12),
                  'cols_negative': dict(cols=-4)}[which])
    assert _call(lib, ops, a['h'], a['res'], a['rows'], a['cols'], a['ld'], a['out']) == NAR_ERR_INVALID
    torch.cuda.synchronize()
    assert (_bits(out) == SENT_BITS).all()


@pytest.mark.parametrize('which', ['src', 'dst'])
def test_dropout_rows_rejects_misaligned(which):
    """nar_dropout_rows reads and writes float4s: a src or dst one float off 16-byte alignment returns NAR_ERR_INVALID,
    checked before the rows = 0 return (so no kernel runs on it), and nothing is written."""
    import torch
    lib, ops = _lib()
    _, src, dst = _small()
    row_pos = torch.zeros(8, dtype=torch.int32, device='cuda')
    p = {'src': ops._p(src), 'dst': ops._p(dst)}
    p[which] = C.c_void_p(p[which].value + 4)
    assert lib.nar_dropout_rows(p['src'], p['dst'], 0, 8, 16, ops._p(row_pos), 0, 0, 0, 9, 0.8, 42, 1,
                                ops._stream()) == NAR_ERR_INVALID
    # the same call on aligned pointers is a valid no-op
    assert lib.nar_dropout_rows(ops._p(src), ops._p(dst), 0, 8, 16, ops._p(row_pos), 0, 0, 0, 9, 0.8, 42, 1,
                                ops._stream()) == 0
    torch.cuda.synchronize()
    assert (_bits(dst) == SENT_BITS).all()
