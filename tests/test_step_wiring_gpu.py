"""How csrc/engine.cu's run_step puts the kernels together, against the fp64 oracle (pytest -m gpu).

The kernels have their own fp64 tests; this file checks the wiring between them: which buffer feeds which GEMM over how
many rows, which dgrad accumulates where, where the dropout masks are applied again in the backward pass, how the
per-unique-id layer 1 splits its gradient, which rank adds the L2 term and which parameter range the optimiser
regularises.  Every case trains one or two `tiny` steps (one G1-shaped case) with 3xTF32 forward and backward GEMMs
(fwd_precision=3, bwd_precision=3), so that the engine comes within a few fp32 roundings of the fp64 oracle and a
missing or misplaced term cannot hide in TF32 noise.  The oracle differentiates leaky_relu at the engine's slope choices
(tools/gpu_step_check.engine_kinks).

Every case starts the engine's gradients, loss accumulators and step workspace from NaN and asserts:
- the sampled negatives are the oracle's, bit for bit;
- xe, L2 and novelty losses within LOSS_TOL relative, logits within LOGIT_TOL of the largest |logit|;
- per logical tensor, max |g - g_ref| <= GRAD_TOL * max |g_ref|; every entry whose fp64 gradient is exactly 0 is exactly 0;
  each touched row of the embedding tables within ROW_TOL of its own max (floor 1e-3 of the tensor max);
- every padding entry of the flat buffer (Hp - H rows / columns, Fp - F columns, the ld padding of the matching layers,
  the gaps between tensors) has a gradient of exactly 0 and stays exactly 0 through Adam;
- Adam, from the engine's own gradient and its state before the step, matches TF-Adam in fp64 (reg_l2 * w added on the
  tensors the oracle regularises, bias correction at the step's count) within fp32 rounding: ADAM_TOL.

`matching_dense_layer_4/bias` is exempt from the relative gradient bar: its gradient (the sum over each position's
softmax gradient) is exactly 0 in exact arithmetic, so any value is rounding noise relative to nothing.  The same sum
makes a column of `matching_dense_layer_3/bias` exactly 0 whenever its leaky_relu slope is the same for all candidates
of every position (frequent with two sessions); fp64 then often rounds to exactly 0 where the engine keeps ~1e-7.  On
those two tensors an exact-zero entry of the oracle may hold up to SUM_ZERO_ABS in the engine instead of exactly 0.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

# Bars (3xTF32 forward and backward against fp64).  Each is within 4x of the worst value measured over every case here on
# an H100 80GB HBM3 at its 700 W power limit (the worst case in brackets):
LOSS_TOL = 1.5e-5          # xe / L2 / novelty loss, relative                  4.6e-6 (gru-cold-b2)
LOGIT_TOL = 1.5e-4         # max |logit error| / max |logit|                    4.4e-5 (ugrnn-g1; tiny cases <= 1.6e-5)
GRAD_TOL = 1e-4            # max |g - g_ref| / max |g_ref| per tensor          4.3e-5 (ugrnn-g1; tiny cases <= 2.7e-5)
ROW_TOL = 1.5e-4           # the same per touched embedding row                5.1e-5 (ugrnn-g1)
ADAM_TOL = 1e-6            # Adam: see measure()                               2.8e-7 (ugrnn-g1)
SUM_ZERO_ABS = 2e-6        # |g| where the exact gradient is a softmax sum     7.2e-7 (lstm-cold-b2)
GRAD_TOL_DEFAULT = 3e-2    # fwd_precision 4 / bwd_precision 1 (bf16x3 forward, single-pass TF32 backward): 7.7e-3

CELLS = ('ugrnn', 'gru', 'lstm')
EXEMPT = 'main/recommendations_ranking/matching_dense_layer_4/bias'
# gradients that are sums of each position's softmax gradient (which sums to 0) wherever the slope of the layer-3
# leaky_relu is the same for all of a position's candidates: exactly 0 in exact arithmetic, and fp64 often lands on 0
SOFTMAX_SUMS = (EXEMPT, 'main/recommendations_ranking/matching_dense_layer_3/bias')


def _one_label(feats, labels):
    """Every session two clicks long: one labelled position each."""
    f = {k: np.array(v, copy=True) for k, v in feats.items()}
    l = {k: np.array(v, copy=True) for k, v in labels.items()}
    f['session_size'] = np.minimum(f['session_size'], 2)
    f['item_clicked'][:, 2:] = 0
    l['label_next_item'][:, 1:] = 0
    l['label_last_item'] = f['item_clicked'][:, 1:2].copy()
    return f, l


def _cases():
    c = {}
    for cell in CELLS:
        for layers in (1, 2, 4):
            for rk in ('mlp', 'cosine'):
                c['%s-%dl-%s' % (cell, layers, rk)] = dict(hp=dict(rnn_num_layers=layers, ranking=rk))
        # dropout: every candidate row materialised (dedup off), masks re-applied in the backward pass
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
        for H in (30, 100, 255, 300):
            c['%s-H%d' % (cell, H)] = dict(hp=dict(rnn_units=H))
    for K in (127, 128):
        # 1 + K = 128 fits one M tile of the fused scorer product, 129 does not (engine.cu fused_product)
        c['ugrnn-K%d' % K] = dict(hp=dict(train_total_negative_samples=K))
        c['ugrnn-K%d-default-precision' % K] = dict(hp=dict(train_total_negative_samples=K), prec=(4, 1))
    # realistic tile and split-K counts: C 1024, H 255, K 50, 46K items
    c['ugrnn-g1'] = dict(name='g1', hp=dict(batch_size=16), warm=30)
    for name in list(c):
        c[name].setdefault('hp', {})['rnn_cell'] = name.split('-')[0]
    return c


CASES = _cases()


def _padding_mask(layout):
    """True at every flat-buffer entry no logical entry maps to."""
    ones = {k: np.ones(v.shape, np.float32) for k, v in layout.init_logical(0).items()}
    return layout.to_internal(ones) == 0


def _adam_ref(layout, regularised, raw, reg, lr):
    """TF-Adam (nar_model.py:708-722) in fp64 from the engine's gradient and its state before the step; reg * w is added
    on the tensors the oracle regularises (not on a range the layout reports)."""
    # the engine's (and TF's) fp32 hyperparameters: 1 - float32(0.999) is 1.3e-5 off 1e-3
    b1, b2, eps, lr = (float(np.float32(x)) for x in (0.9, 0.999, 1e-8, lr))
    p0, m0, v0 = (x.astype(np.float64) for x in raw['before'])
    g = raw['flat_grads'].astype(np.float64)
    r = np.zeros_like(g)
    for t in layout.tensors:
        if regularised(t.tf_name):
            r[t.offset:t.offset + t.size] = reg
    gg = g + r * p0
    m1 = b1 * m0 + (1 - b1) * gg
    v1 = b2 * v0 + (1 - b2) * gg * gg
    t = raw['t']
    lr_t = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    p1 = p0 - lr_t * m1 / (np.sqrt(v1) + eps)
    ag = np.abs(g) + np.abs(r * p0)
    return (p1, m1, v1), (b1 * np.abs(m0) + (1 - b1) * ag, b2 * v0 + (1 - b2) * ag * ag)


def measure(case, cases=CASES):
    """Run one case of `cases` (CASES, or another dict of the same form) -> the worst value of every measured quantity
    over its steps."""
    import torch
    from tools import gpu_step_check as g
    cfg = cases[case]
    fwd, bwd = cfg.get('prec', (3, 3))
    ekw = dict(fwd_precision=fwd, bwd_precision=bwd, **cfg.get('ekw', {}))
    res = g.run_case(cfg.get('name', 'tiny'), cfg.get('profile', 'B'), cfg.get('warm', 5), cfg.get('steps', 2),
                     hp_over=cfg['hp'], oracle_dtype=torch.float64, engine_kw=ekw, raw=True, batch_map=cfg.get('batch_map'))
    lay, hp = res['layout'], res['hp']
    pad = _padding_mask(lay)
    m = {'neg_equal': True, 'L_min': 1 << 30, 'loss_rel': 0.0, 'logit_rel': 0.0, 'grad_rel': 0.0, 'grad_worst': '',
         'row_rel': 0.0, 'zero_violations': 0, 'zero_entries': 0, 'pad_violations': 0, 'pad_entries': int(pad.sum()),
         'nonfinite': 0, 'applied': True, 'adam_m': 0.0, 'adam_v': 0.0, 'adam_w': 0.0, 'exempt_abs': 0.0,
         'sum_zero_abs': 0.0}
    for s in res['steps']:
        raw = s['raw']
        m['neg_equal'] &= s['neg_equal']
        m['L_min'] = min(m['L_min'], s['L'])
        m['applied'] &= raw['applied']
        for got, want in zip(raw['loss'], raw['loss_ref']):
            if want != 0.0 or got != 0.0:
                m['loss_rel'] = max(m['loss_rel'], abs(got - want) / max(abs(want), 1e-30))
        m['logit_rel'] = max(m['logit_rel'], g.rel(raw['logits'], raw['logits_ref']))
        m['nonfinite'] += int((~np.isfinite(raw['flat_grads'])).sum())
        for k, gr in raw['grads_ref'].items():
            ge = raw['grads'][k].astype(np.float64)
            err = np.abs(ge - gr)
            zero = gr == 0
            m['zero_entries'] += int(zero.sum())
            if k in SOFTMAX_SUMS:
                m['sum_zero_abs'] = max(m['sum_zero_abs'], float(np.abs(ge[zero]).max(initial=0.0)))
                zero = np.zeros_like(zero)
            bad = int((ge[zero] != 0).sum())
            if bad:
                m['zero_violations'] += bad
                m.setdefault('zero_detail', {})[k] = [bad, float(np.abs(ge[zero]).max()), float(np.abs(gr).max()),
                                                      np.argwhere((ge != 0) & zero)[:4].tolist()]
            if k == EXEMPT:
                m['exempt_abs'] = max(m['exempt_abs'], float(np.abs(ge).max()))
                continue
            scale = float(np.abs(gr).max())
            e = float(err.max()) / scale if scale > 0 else float(err.max())
            if e > m['grad_rel']:
                m['grad_rel'], m['grad_worst'] = e, k
            if gr.ndim == 2 and (k.endswith('items_embedding') or '_cat_embedding/' in k):
                rowmax = np.abs(gr).max(axis=1)
                touched = rowmax > 0
                if touched.any():
                    rr = err.max(axis=1)[touched] / np.maximum(rowmax[touched], 1e-3 * scale)
                    m['row_rel'] = max(m['row_rel'], float(rr.max()))
        fg = raw['flat_grads']
        m['pad_violations'] += int((fg[pad] != 0).sum())
        for x in raw['after']:
            m['pad_violations'] += int((x[pad] != 0).sum())
        # m and v: error over the magnitude of the terms they sum (fp32 rounding: a few 2^-24); w: error beyond one fp32
        # ulp of w, over lr (the step itself is ~lr)
        (p1, m1, v1), (sm, sv) = _adam_ref(lay, res['regularised'], raw, hp.reg_l2, hp.learning_rate)
        pe, me, ve = (x.astype(np.float64) for x in raw['after'])
        for key, got, want, sc in (('adam_m', me, m1, sm), ('adam_v', ve, v1, sv)):
            m[key] = max(m[key], float((np.abs(got - want) / np.maximum(sc, 1e-35)).max()))
        ulp = np.spacing(np.abs(p1).astype(np.float32)).astype(np.float64)
        m['adam_w'] = max(m['adam_w'], float(np.maximum(np.abs(pe - p1) - ulp, 0).max() / hp.learning_rate))
    m['tight'] = (fwd, bwd) == (3, 3)
    return m


def check(m):
    assert m['neg_equal'], 'negatives must be bit-exact'
    assert m['L_min'] > 0 and m['applied']
    assert m['nonfinite'] == 0, m
    assert m['zero_violations'] == 0, m
    assert m['pad_violations'] == 0, m
    assert m['adam_m'] <= ADAM_TOL and m['adam_v'] <= ADAM_TOL and m['adam_w'] <= ADAM_TOL, m
    if m['tight']:
        assert m['loss_rel'] <= LOSS_TOL, m
        assert m['logit_rel'] <= LOGIT_TOL, m
        assert m['grad_rel'] <= GRAD_TOL, m
        assert m['row_rel'] <= ROW_TOL, m
        assert m['sum_zero_abs'] <= SUM_ZERO_ABS and m['exempt_abs'] <= SUM_ZERO_ABS, m
    else:
        assert m['grad_rel'] <= GRAD_TOL_DEFAULT, m


@pytest.mark.parametrize('case', sorted(CASES))
def test_step_matches_fp64(case):
    check(measure(case))


# ------------------------------------------------------------------------------------------------ edges
def _engine(cell, **hp):
    import torch
    from chameleon_recsys_b200.harness import make_problem, warm_state
    from tools import gpu_step_check as g
    pb = make_problem('tiny', profile='B', rnn_cell=cell, **hp)
    warm_state(pb, 5)
    eng = g.make_engine(pb, fwd_precision=3, bwd_precision=3)
    orc = g.make_oracle(pb, torch.float64)
    logical = pb.layout.init_logical(pb.hp.init_seed)
    eng.set_params(logical); orc.set_params(logical)
    return pb, eng, orc


def _state(pb):
    return pb.clicked_items_state.get_recent_clicks_buffer().copy(), pb.clicked_items_state.get_articles_recent_pop_norm().copy()


@pytest.mark.parametrize('cell', CELLS)
def test_step_without_labelled_positions(cell):
    """L = 0 after a real step: gradients and loss exactly 0, and submit leaves weights, Adam slots and step alone."""
    pb, eng, _ = _engine(cell)
    it = pb.input_fn()
    buf, pop = _state(pb)
    eng.train_step(*it.get_next(), buf, pop)
    assert float(eng.grads.abs().max()) > 0
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
    """Data parallel emulated in one process (world 2, rank 0 and 1 on one device): each rank's shard gradient, summed,
    and the losses, summed, against the oracle's whole batch at the tight bars; only rank 0 adds the L2 term."""
    import torch
    from oracle import sampler_ref
    from tools import gpu_step_check as g
    pb, _, orc = _engine(cell, rnn_num_layers=2)
    hp = pb.hp
    f, l = pb.input_fn().get_next()
    buf, pop = _state(pb)
    logical = pb.layout.init_logical(hp.init_seed)
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
    got = pb.layout.to_logical(gsum.cpu().numpy())
    for k, gr in grads.items():
        gr = gr.detach()
        if orc.regularised(k):
            gr = gr - orc.reg * w[k]
        gr = gr.numpy()
        if k not in SOFTMAX_SUMS:
            assert not got[k][gr == 0].any(), k
        if k != EXEMPT and np.abs(gr).max() > 0:
            assert np.abs(got[k] - gr).max() <= GRAD_TOL * np.abs(gr).max(), k


@pytest.mark.parametrize('cell', CELLS)
def test_eval_step_matches_fp64(cell):
    """eval_step (no dropout, no gradients) at fwd_precision 3: logits and losses against the oracle's forward."""
    import torch
    from oracle import sampler_ref
    pb, eng, orc = _engine(cell, rnn_num_layers=2, dropout_keep_prob=0.7, novelty_reg_factor=0.5)
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


@pytest.mark.parametrize('cell, H', [('ugrnn', 100), ('gru', 300), ('lstm', 300)])
def test_estimator_runs_hidden_sizes_padded_past_a_kernel_size(cell, H, tmp_path):
    """rnn_units 100 (Hp 128) and 300 (Hp 512) train, evaluate and predict through Estimator; the padding stays zero."""
    from chameleon_recsys_b200.estimator import build_estimator
    from chameleon_recsys_b200.harness import make_problem, warm_state
    pb = make_problem('tiny', profile='B', rnn_cell=cell, rnn_units=H, batch_size=24)
    assert pb.layout.Hp == (128 if H == 100 else 512)
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
    pad = _padding_mask(pb.layout)
    assert not eng.params.cpu().numpy()[pad].any()
