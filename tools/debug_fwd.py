"""Forward / gradient errors of full steps under both forward precisions (3 = 3xTF32, 4 = bf16x3) on the shapes the
parity suite covers.  python tools/debug_fwd.py"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from tools import gpu_step_check as g  # noqa: E402

CASES = [('tiny_cold', 'tiny', 0, 2, {}, torch.float64), ('adressa32', 'adressa', 20, 1, dict(batch_size=32), torch.float32),
         ('stress8', 'stress', 4, 1, dict(batch_size=8), torch.float32), ('g1_48', 'g1', 30, 2, dict(batch_size=48), torch.float32)]
for name, wl, warm, steps, hp, dt in CASES:
    for fwd in (3, 4):
        res = g.run_case(wl, 'B', warm, steps, hp_over=hp, oracle_dtype=dt, engine_kw=dict(fwd_precision=fwd))
        for s in res['steps']:
            worst = sorted(s['grad_rel'].items(), key=lambda kv: -kv[1])[:3]
            print(name, 'fwd', fwd, 'step', s['step'], 'L', s['L'],
                  'x %.1e e %.1e rnn %.1e pred %.1e logits %.1e xe %.1e' % (max(s['x_in'], s['x_pos'], s['x_neg']), max(s['e_in'], s['e_pos'], s['e_neg']), s['rnn'], s['pred'], s['logits_rel_max'], s['xe_rel']),
                  'grad_max %.2e upd %.2f' % (s['grad_rel_max'], s['update_err_over_lr']), [(k, '%.1e' % v) for k, v in worst])
