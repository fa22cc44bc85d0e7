"""Full-step parity on the GPU: engine (CUDA) vs oracle (torch-CPU fp64/fp32) on identical inputs.
Writes step_check.json to the current directory.  Usage: python tools/gpu_step_check.py [tiny|g1small] ..."""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chameleon_recsys_b200.clicked_items_state import batch_clicks_for_state_update  # noqa: E402
from chameleon_recsys_b200.engine import NarEngine  # noqa: E402
from chameleon_recsys_b200.harness import make_problem, warm_state  # noqa: E402
from oracle import sampler_ref  # noqa: E402
from oracle.lstm_ref import LstmOracle  # noqa: E402
from oracle.nar_oracle import NarOracle  # noqa: E402
from oracle.residual_ref import ResidualOracle  # noqa: E402


def make_oracle(pb, dtype=torch.float64, residual=None):
    """The oracle of ``pb``'s model; ``residual`` (default: hp.rnn_residual_connections) builds the residual session
    stack of oracle/residual_ref.py."""
    hp = pb.hp
    residual = hp.rnn_residual_connections if residual is None else residual
    cls = ResidualOracle if residual else (LstmOracle if hp.rnn_cell == 'lstm' else NarOracle)
    return cls(pb.session_features_config, pb.articles_features_config, pb.internal_features_config,
                     pb.content_article_embeddings_matrix, pb.articles_metadata,
                     negative_samples=hp.train_total_negative_samples, softmax_temperature=hp.softmax_temperature,
                     reg_weight_decay=hp.reg_l2, recent_clicks_for_normalization=hp.recent_clicks_for_normalization,
                     elapsed_days_smooth_log_base=hp.elapsed_days_smooth_log_base,
                     popularity_smooth_log_base=hp.popularity_smooth_log_base,
                     CAR_embedding_size=hp.CAR_embedding_size, rnn_units=hp.rnn_units,
                     rnn_num_layers=hp.rnn_num_layers, max_cardinality_for_ohe=hp.max_cardinality_for_ohe,
                     lr=hp.learning_rate, ranking=hp.ranking, rnn_cell=hp.rnn_cell, dtype=dtype, keep_prob=hp.dropout_keep_prob,
                     novelty_reg_factor=hp.novelty_reg_factor, dropout_seed=hp.sampler_seed, int2log=pb.plan.int2log)


def make_engine(pb, **kw):
    hp = pb.hp
    return NarEngine(pb.plan, pb.layout, pb.content_article_embeddings_matrix, pb.articles_metadata,
                     negative_samples=hp.train_total_negative_samples,
                     negative_sample_from_buffer=hp.train_negative_samples_from_buffer,
                     softmax_temperature=hp.softmax_temperature, reg_weight_decay=hp.reg_l2, lr=hp.learning_rate,
                     recent_clicks_buffer_max_size=hp.recent_clicks_buffer_max_size,
                     recent_clicks_for_normalization=hp.recent_clicks_for_normalization,
                     elapsed_days_smooth_log_base=hp.elapsed_days_smooth_log_base,
                     popularity_smooth_log_base=hp.popularity_smooth_log_base, ranking=hp.ranking, rnn_cell=hp.rnn_cell,
                     sampler_seed=hp.sampler_seed, keep_prob=hp.dropout_keep_prob, novelty_reg_factor=hp.novelty_reg_factor,
                     rnn_residual=hp.rnn_residual_connections, **kw)


def rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)) if a.size else 0.0


def engine_kinks(lasts, session_size, T, n_cand):
    """The engine's leaky_relu slope choices for NarOracle's kink alignment, from the ``last`` intermediates of one step
    (or of the data-parallel shards of one step, in rank order: their positions follow each other session-major)."""
    valid = np.arange(T)[None, :] < np.clip(np.asarray(session_size) - 1, 0, T)[:, None]
    ins, cands, f1, zs = [], [], [], {}
    for last in lasts:
        L = last['F1'].shape[0]
        H1 = last['H1'].cpu().numpy() > 0
        ins.append(H1[:L]); cands.append(H1[L:].reshape(L, n_cand, -1)); f1.append(last['F1'].cpu().numpy() > 0)
        for zn in ('Z1', 'Z2', 'Z3'):
            if zn in last:
                zs.setdefault(zn, []).append((last[zn].cpu().numpy() > 0).reshape(L, n_cand, -1))
    Hc = np.concatenate(cands)
    kinks = {'valid': torch.as_tensor(valid), 'h1_in': np.concatenate(ins), 'h1_pos': Hc[:, 0], 'h1_neg': Hc[:, 1:],
             'f1': np.concatenate(f1)}
    for zn, parts in zs.items():
        Z = np.concatenate(parts)
        kinks[zn.lower() + '_pos'] = Z[:, 0]
        kinks[zn.lower() + '_neg'] = Z[:, 1:]
    return kinks


def run_case(name, profile, warm, n_steps, hp_over=None, oracle_dtype=torch.float64, sync_state=True, engine_kw=None,
             align_kinks=True, raw=False, batch_map=None, **mk):
    """``raw``: every step also starts the engine's outputs (gradients, loss accumulators, step workspace) from NaN and
    hands back, under r['raw'], the flat buffers around the step (params / adam_m / adam_v before and after the optimiser,
    the gradient), the logical gradients of both sides and the loss parts.  ``batch_map(feats, labels)`` -> (feats,
    labels) rewrites every batch before either side sees it."""
    pb = make_problem(name, profile=profile, **(hp_over or {}), **mk)
    hp = pb.hp
    if warm:
        warm_state(pb, warm)
    eng = make_engine(pb, **(engine_kw or {}))
    orc = make_oracle(pb, oracle_dtype)
    logical = pb.layout.init_logical(hp.init_seed)
    eng.set_params(logical)
    orc.set_params(logical)
    it = pb.input_fn()
    K = hp.train_total_negative_samples
    res = {'case': name, 'profile': profile, 'warm': warm, 'ranking': hp.ranking, 'layers': hp.rnn_num_layers, 'steps': []}
    for step in range(1, n_steps + 1):
        feats, labels = it.get_next()
        if batch_map is not None:
            feats, labels = batch_map(feats, labels)
        if sync_state and step > 1:
            # per-step parity: start every step from the oracle's exact state (weights + Adam slots)
            eng.load_logical_state(orc.get_params(), {k: v.numpy() for k, v in orc.adam_m.items()},
                                   {k: v.numpy() for k, v in orc.adam_v.items()}, orc.step)
        buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
        pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
        st = eng.stage(feats, labels, buf, pop)
        if raw:
            before = [t.detach().cpu().numpy().copy() for t in (eng.params, eng.adam_m, eng.adam_v)]
            t_adam = eng.global_step + 1
            eng.prepare(st, t_adam)                              # sizes the step workspace (submit then runs the step on it)
            eng.grads.fill_(float('nan')); eng.loss_dev.fill_(float('nan'))
            eng._ws.fill_(0xFF)                                   # every float of the step workspace a NaN
            w_ref = {k: v.detach().clone() for k, v in orc.params.items()}
        out = eng.result(eng.submit(st, keep=True))
        st = out['stage']
        B, T, L = st['B'], st['T'], st['L']
        neg_gpu = out['negatives'].cpu().numpy()
        allc = np.concatenate([feats['item_clicked'], labels['label_last_item']], axis=1)
        neg_ref = sampler_ref.sample_negatives(allc, buf, K, hp.train_negative_samples_from_buffer, hp.sampler_seed, step)
        params_before = {n: v.astype(np.float64) for n, v in orc.get_params().items()}
        last = eng.last
        n_cand = K + 1
        # kink alignment (see NarOracle._dense): the oracle differentiates leaky_relu with the ENGINE's slope choices
        kinks = engine_kinks([last], feats['session_size'], T, n_cand) if align_kinks and L > 0 else None
        o, grads = orc.train_step(feats, labels, neg_ref, buf, pop, kinks=kinks)
        mask = o['mask'].numpy()
        r = {'step': step, 'B': B, 'T': T, 'L': L, 'neg_equal': bool(np.array_equal(neg_gpu, neg_ref))}
        l2i = pb.plan.log2int
        X = last['X'].cpu().numpy()[:, l2i]
        E = last['E'].cpu().numpy()
        x_in = o['x_in'].detach().numpy()[mask]
        x_pos = o['x_pos'].detach().numpy()[mask]
        x_neg = o['x_neg'].detach().numpy()[mask]
        Xc = X[L:].reshape(L, n_cand, -1)
        r['x_in'] = rel(X[:L], x_in); r['x_pos'] = rel(Xc[:, 0], x_pos); r['x_neg'] = rel(Xc[:, 1:], x_neg)
        segerr = {}
        for sg in pb.plan.segments:
            sl = slice(sg.log_col, sg.log_col + sg.width)
            segerr[sg.name] = [float(np.abs(X[:L][:, sl] - x_in[:, sl]).max()), float(np.abs(Xc[:, 0][:, sl] - x_pos[:, sl]).max()),
                               float(np.abs(Xc[:, 1:][..., sl] - x_neg[..., sl]).max())]
        r['seg_abs_err'] = segerr
        r['stats'] = last['stats'].cpu().numpy().tolist()
        Ec = E[L:].reshape(L, n_cand, -1)
        r['e_in'] = rel(E[:L], o['e_in'].detach().numpy()[mask])
        r['e_pos'] = rel(Ec[:, 0], o['e_pos'].detach().numpy()[mask])
        r['e_neg'] = rel(Ec[:, 1:], o['e_neg'].detach().numpy()[mask])
        H = hp.rnn_units
        r['rnn'] = rel(last['HO'][-1].cpu().numpy()[:, :H], o['rnn_out'].detach().numpy()[mask])
        r['pred'] = rel(last['PR'].cpu().numpy(), o['pred'].detach().numpy()[mask])
        lg = last['logits'].cpu().numpy()
        lg_ref = o['logits'].detach().numpy()[mask]
        r['logits_rel_max'] = rel(lg, lg_ref)
        r['logits_rel_rms'] = float(np.sqrt(((lg - lg_ref) ** 2).mean()) / max(np.sqrt((lg_ref ** 2).mean()), 1e-30))
        r['xe_gpu'] = out['xe_loss']; r['xe_ref'] = float(o['xe_loss']); r['xe_rel'] = abs(out['xe_loss'] - float(o['xe_loss'])) / abs(float(o['xe_loss']))
        r['reg_gpu'] = out['reg_loss']; r['reg_ref'] = float(o['reg_loss'])
        r['total_rel'] = abs(out['total_loss'] - float(o['total_loss'])) / abs(float(o['total_loss']))
        # gradients: engine grads exclude the l2 term (folded into the Adam kernel)
        g_gpu = eng.get_grads()
        p_before = None
        gerr = {}
        gabs = {}
        for k, g in grads.items():
            gref = g.detach().numpy().astype(np.float64)
            if orc.reg > 0 and orc.regularised(k):
                # oracle params were already updated by Adam: recover w_before from the engine's copy is not possible;
                # compare against (grad - reg*w_before) using the logical params saved below
                gref = gref - orc.reg * params_before[k]
            gerr[k.split('/')[-2] + '/' + k.split('/')[-1]] = rel(g_gpu[k], gref)
            gabs[k.split('/')[-2] + '/' + k.split('/')[-1]] = (float(np.abs(g_gpu[k] - gref).max()), float(np.abs(gref).max()))
        gerr.pop('matching_dense_layer_4/bias', None)       # exactly zero in exact arithmetic (softmax gradient sums to 0)
        r['grad_rel_max'] = max(gerr.values()); r['grad_rel'] = gerr; r['grad_abs'] = gabs
        p_gpu = eng.get_params(); p_ref = orc.get_params()
        r['param_abs_max'] = max(float(np.abs(p_gpu[k] - p_ref[k]).max()) for k in p_ref)
        # Adam normalises: compare updates only where the gradient is far above eps/sqrt(1-b2) = 3.2e-7
        upd = []
        for k, g in grads.items():
            gref = np.abs(g.detach().numpy().astype(np.float64))
            big = gref > 1e-4 * max(gref.max(), 1e-30)
            big &= gref > 3e-5
            if big.any():
                du = (p_gpu[k] - params_before[k])[big]; dr = (p_ref[k] - params_before[k])[big]
                upd.append(float(np.abs(du - dr).max() / hp.learning_rate))
        r['update_err_over_lr'] = max(upd) if upd else 0.0
        if raw:
            g_ref = {}
            for k, g in grads.items():
                g = g.detach()
                if orc.reg > 0 and orc.regularised(k):
                    g = g - orc.reg * w_ref[k]            # the same fp64 product autograd formed: exact where only L2 acts
                g_ref[k] = g.numpy().astype(np.float64)
            after = [t.detach().cpu().numpy().copy() for t in (eng.params, eng.adam_m, eng.adam_v)]
            r['raw'] = {'grads': g_gpu, 'grads_ref': g_ref, 'flat_grads': eng.grads.detach().cpu().numpy().copy(),
                        'before': before, 'after': after, 't': t_adam, 'applied': eng.global_step == t_adam,
                        'loss': [out['xe_loss'], out['reg_loss'], out['nov_reg_loss']],
                        'loss_ref': [float(o['xe_loss']), float(o['reg_loss']), float(o['nov_reg_loss'])],
                        'logits': lg, 'logits_ref': lg_ref}
            res['layout'], res['hp'], res['regularised'] = pb.layout, hp, orc.regularised
        res['steps'].append(r)
        # host state update (hook.after_run)
        pb.clicked_items_state.update_from_batch(feats['item_clicked'], feats['event_timestamp'], labels['label_last_item'])
    return res


def run_trajectory(name, profile, warm, n_steps, hp_over=None, oracle_dtype=torch.float32, engine_kw=None):
    """UN-SYNCED trajectory: engine and oracle start from the same weights and then each follows its OWN Adam
    trajectory for n_steps (no state reload) - this is what tells whether the narrower backward GEMMs (single-pass
    TF32 vs the reference's fp32) bend the loss curve.  Returns per-step losses of both and their relative gap."""
    pb = make_problem(name, profile=profile, **(hp_over or {}))
    hp = pb.hp
    if warm:
        warm_state(pb, warm)
    eng = make_engine(pb, **(engine_kw or {}))
    orc = make_oracle(pb, oracle_dtype)
    logical = pb.layout.init_logical(hp.init_seed)
    eng.set_params(logical)
    orc.set_params(logical)
    it = pb.input_fn()
    K = hp.train_total_negative_samples
    steps = []
    for step in range(1, n_steps + 1):
        feats, labels = it.get_next()
        buf = pb.clicked_items_state.get_recent_clicks_buffer().copy()
        pop = pb.clicked_items_state.get_articles_recent_pop_norm().copy()
        out = eng.train_step(feats, labels, buf, pop)
        allc = np.concatenate([feats['item_clicked'], labels['label_last_item']], axis=1)
        neg_ref = sampler_ref.sample_negatives(allc, buf, K, hp.train_negative_samples_from_buffer, hp.sampler_seed, step)
        o, _ = orc.train_step(feats, labels, neg_ref, buf, pop)
        ref = float(o['total_loss'])
        steps.append({'step': step, 'gpu': out['total_loss'], 'ref': ref, 'rel': abs(out['total_loss'] - ref) / abs(ref),
                      'neg_equal': bool(np.array_equal(out['negatives'].cpu().numpy(), neg_ref))})
        items, ts = batch_clicks_for_state_update(feats['item_clicked'], feats['event_timestamp'], labels['label_last_item'])
        pb.clicked_items_state.update_items_state(items, ts)
    p_gpu, p_ref = eng.get_params(), orc.get_params()
    drift = max(float(np.abs(p_gpu[k] - p_ref[k]).max()) for k in p_ref)
    return {'case': name, 'steps': steps, 'max_rel': max(s['rel'] for s in steps), 'param_drift_abs_max': drift,
            'lr': hp.learning_rate}


def main():
    cases = sys.argv[1:] or ['tinyA', 'tinyB', 'tinyB_cold', 'tinyB_cos', 'tinyB_2l', 'g1small']
    report = []
    for c in cases:
        t0 = time.time()
        try:
            if c == 'tinyA':
                res = run_case('tiny', 'A', 5, 3)
            elif c == 'tinyB':
                res = run_case('tiny', 'B', 5, 3)
            elif c == 'tinyB_cold':
                res = run_case('tiny', 'B', 0, 2)
            elif c == 'tinyB_cos':
                res = run_case('tiny', 'B', 5, 2, hp_over=dict(ranking='cosine'))
            elif c == 'tinyB_2l':
                res = run_case('tiny', 'B', 5, 2, hp_over=dict(rnn_num_layers=2))
            elif c == 'g1small':
                res = run_case('g1', 'B', 30, 2, hp_over=dict(batch_size=64), oracle_dtype=torch.float32)
            elif c == 'g1':
                res = run_case('g1', 'B', 30, 1, oracle_dtype=torch.float32)
            else:
                raise ValueError(c)
            res['seconds'] = round(time.time() - t0, 1)
            report.append(res)
            for s in res['steps']:
                print(c, json.dumps({k: v for k, v in s.items() if k not in ('grad_rel', 'seg_abs_err', 'stats')}))
                print('    seg', {k: ['%.1e' % e for e in v] for k, v in s['seg_abs_err'].items() if max(v) > 1e-5})
                worst = sorted(s['grad_rel'].items(), key=lambda kv: -kv[1])[:4]
                print('    worst grads', worst)
        except Exception as e:  # noqa: BLE001
            import traceback
            report.append({'case': c, 'error': traceback.format_exc()})
            print(c, 'ERROR', traceback.format_exc())
    with open('step_check.json', 'w') as f:
        json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
