"""GPU diagnostics: run every kernel family in its own subprocess (a trap / hang in one does not
mask the others) and write diag.json to the current directory.  Usage:
    python tools/gpu_diag.py            # all
    python tools/gpu_diag.py gemm       # one family
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.getcwd()


def _gemm_case(a_k, b_k, prec, M, N, K, epi='none', split=1, blo=False):
    import torch
    from chameleon_recsys_b200 import ops
    torch.manual_seed(M * 7 + N * 3 + K)
    dev = 'cuda'
    lda = ((K if a_k else M) + 3) // 4 * 4
    ldb = ((K if b_k else N) + 3) // 4 * 4
    A = torch.zeros((M if a_k else K), lda, device=dev)
    B = torch.zeros((N if b_k else K), ldb, device=dev)
    A[:, :(K if a_k else M)].normal_()
    B[:, :(K if b_k else N)].normal_()
    Al = (A[:, :K] if a_k else A[:, :M].t()).double()      # [M,K]
    Bl = (B[:, :K] if b_k else B[:, :N].t()).double()      # [N,K]
    ref = Al @ Bl.t()
    ldd = (N + 3) // 4 * 4
    D = torch.full((M, ldd), 7.0, device=dev)
    bias = aux = None
    kw = {}
    if epi == 'bias_leaky':
        bias = torch.randn(ldd, device=dev)
        ref = torch.nn.functional.leaky_relu(ref + bias[:N].double(), 0.2)
        kw = dict(bias=bias, act=ops.ACT_LEAKY)
    elif epi == 'bias_tanh':
        bias = torch.randn(ldd, device=dev) * 0.1
        ref = torch.tanh(ref / 30 + bias[:N].double())
        A = A / 30
        kw = dict(bias=bias, act=ops.ACT_TANH)
    elif epi == 'dact_tanh':
        aux = torch.rand(M, ldd, device=dev) * 1.8 - 0.9
        ref = ref * (1 - aux[:, :N].double() ** 2)
        kw = dict(dact=ops.ACT_TANH, aux=aux)
    elif epi == 'accum':
        D.zero_()
        D += 1.0
        ref = ref + 1.0
        kw = dict(accumulate=True, split_k=split)
    if blo:
        Blo = torch.empty_like(B)
        ops.tf32_lo(B, B.numel(), Blo)
        kw['b_lo'] = Blo
    ops.gemm(A, B, D, M, N, K, a_kmajor=a_k, b_kmajor=b_k, lda=lda, ldb=ldb, precision=prec, **kw)
    torch.cuda.synchronize()
    got = D[:, :N].double()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    untouched = bool((D[:, N:] == (7.0 if epi != 'accum' else 1.0)).all().item()) if ldd > N else True
    return {'err': err, 'scale': scale, 'rel': err / max(scale, 1e-30), 'pad_untouched': untouched,
            'nan': bool(torch.isnan(got).any().item())}


def _fam_gemm_major(a_k, b_k):
    res = []
    shapes = [(128, 128, 32), (128, 128, 256), (300, 200, 100), (1000, 510, 1024), (257, 64, 480)]
    for prec in (1, 3):
        for (M, N, K) in shapes:
            for blo in ((False, True) if prec == 3 else (False,)):
                r = _gemm_case(a_k, b_k, prec, M, N, K, blo=blo)
                r.update(a_k=a_k, b_k=b_k, prec=prec, shape=[M, N, K], epi='none', blo=blo)
                r['ok'] = (not r['nan']) and r['rel'] < (3e-3 if prec == 1 else 2e-5) and r['pad_untouched']
                res.append(r)
    return res


def fam_gemm_kk(): return _fam_gemm_major(True, True)
def fam_gemm_km(): return _fam_gemm_major(True, False)
def fam_gemm_mk(): return _fam_gemm_major(False, True)
def fam_gemm_mm(): return _fam_gemm_major(False, False)


def fam_gemm_epi():
    res = []
    for epi in ('bias_leaky', 'bias_tanh', 'dact_tanh'):
        r = _gemm_case(True, True, 3, 333, 250, 200, epi)
        r.update(epi=epi, ok=(not r['nan']) and r['rel'] < 5e-5 and r['pad_untouched'])
        res.append(r)
    for split in (1, 4, 13, 0):
        r = _gemm_case(True, True, 1, 480, 1024, 5000, 'accum', split)
        r.update(epi='accum', split=split, ok=(not r['nan']) and r['rel'] < 3e-3)
        res.append(r)
    # big single-pass problems (many waves of 128x128 tiles), all operand majors, ragged edges
    for (a_k, b_k) in ((True, True), (True, False), (False, True), (False, False)):
        r = _gemm_case(a_k, b_k, 1, 3000, 1000, 2040)
        r.update(a_k=a_k, b_k=b_k, shape=[3000, 1000, 2040], epi='T2', ok=(not r['nan']) and r['rel'] < 3e-3 and r['pad_untouched'])
        res.append(r)
    r = _gemm_case(False, False, 1, 1024, 1000, 20000, 'accum', 0)
    r.update(epi='T2 accum auto-split', ok=(not r['nan']) and r['rel'] < 3e-3)
    res.append(r)
    r = _gemm_case(True, True, 1, 3000, 1024, 2048, 'dact_tanh')
    r.update(epi='T2 dact', ok=(not r['nan']) and r['rel'] < 3e-3)
    res.append(r)
    return res


def fam_gemm_bf16():
    """precision 4 (bf16x3 on the bf16 tensor path): D = act(A * W + b) with W given as the packed bf16 plane, against fp64.
    Expected error ~2^-16 of |a||b| per product (bf16 hi + lo keep 16 mantissa bits): 1e-4 of the result scale is the bar."""
    import torch
    from chameleon_recsys_b200 import ops
    res = []
    for (M, N, K, epi) in ((333, 250, 200, 'none'), (1000, 1024, 1024, 'bias_tanh'), (129, 64, 72, 'bias_leaky'),
                           (5000, 128, 1024, 'none'), (20000, 1024, 408, 'bias_leaky'), (77, 32, 64, 'none')):
        torch.manual_seed(M + N + K)
        lda = (K + 3) // 4 * 4
        A = torch.zeros(M, lda, device='cuda'); A[:, :K].normal_()
        W = torch.randn(K, (N + 3) // 4 * 4, device='cuda')
        if epi == 'bias_tanh':
            A /= 30
        ref = A[:, :K].double() @ W[:, :N].double()
        ldd = (N + 3) // 4 * 4
        D = torch.full((M, ldd), 7.0, device='cuda')
        kw = {}
        if epi != 'none':
            bias = torch.randn(ldd, device='cuda') * 0.1
            ref = ref + bias[:N].double()
            ref = torch.tanh(ref) if epi == 'bias_tanh' else torch.nn.functional.leaky_relu(ref, 0.2)
            kw = dict(bias=bias, act=ops.ACT_TANH if epi == 'bias_tanh' else ops.ACT_LEAKY)
        plane = ops.pack_bf16x3(W, K, N)
        ops.gemm(A, None, D, M, N, K, a_kmajor=True, b_kmajor=True, lda=lda, ldb=0, precision=4, b_bf16=plane,
                 ld_bf16=plane.stride(0), **kw)
        torch.cuda.synchronize()
        got = D[:, :N].double()
        rel = float((got - ref).abs().max() / ref.abs().max())
        r = dict(shape=[M, N, K], epi=epi, rel=rel, nan=bool(torch.isnan(D[:, :N]).any()),
                 pad_untouched=bool((D[:, N:] == 7.0).all()) if ldd > N else True)
        r['ok'] = (not r['nan']) and rel < 1e-4 and r['pad_untouched']
        res.append(r)
    return res


def fam_gather():
    import torch
    from chameleon_recsys_b200 import ops
    out = []
    for (V, E, ld, n) in [(1000, 250, 252, 5000), (46034, 250, 252, 100000), (500, 117, 120, 777), (100, 64, 64, 33)]:
        table = torch.randn(V, ld, device='cuda')
        ids = torch.randint(0, V, (n,), device='cuda')
        o = torch.zeros(n, ld, device='cuda')
        ops.gather_rows(table, ids, o, E)
        torch.cuda.synchronize()
        ok = bool(torch.equal(o[:, :E], table[ids][:, :E]))
        g = torch.zeros(V, ld, device='cuda')
        src = torch.randn(n, ld, device='cuda')
        ops.scatter_add_rows(g, ids, src, E)
        ref = torch.zeros(V, ld, device='cuda', dtype=torch.float64).index_add_(0, ids, src.double())
        err = (g[:, :E].double() - ref[:, :E]).abs().max().item()
        out.append({'V': V, 'E': E, 'n': n, 'gather_exact': ok, 'scatter_err': err, 'ok': ok and err < 1e-3})
    return out


def fam_sampler():
    import numpy as np
    import torch
    from chameleon_recsys_b200 import ops
    from oracle import sampler_ref
    out = []
    rs = np.random.RandomState(0)
    cases = [(8, 5, 10, 64, 10, 200, 0.5), (64, 5, 10, 2000, 300, 1000, 0.9), (256, 20, 50, 20000, 3000, 46034, 0.9),
             (4, 3, 5, 32, 10, 50, 0.0), (16, 8, 30, 500, 3000, 300, 1.0)]
    for ci, (B, T1, K, buf_len, nfb, V, fill) in enumerate(cases):
        allc = np.zeros((B, T1), np.int64)
        for b in range(B):
            n = rs.randint(2, T1 + 1)
            allc[b, :n - 1] = rs.choice(np.arange(1, V), n - 1, replace=False)
            allc[b, T1 - 1] = rs.randint(1, V)
        buf = np.zeros(buf_len, np.int64)
        nfill = int(buf_len * fill)
        buf[:nfill] = (rs.zipf(1.3, nfill) % (V - 1)) + 1
        for step in (1, 7):
            ref = sampler_ref.sample_negatives(allc, buf, K, nfb, 42, step)
            d_all = torch.from_numpy(allc).cuda()
            d_buf = torch.from_numpy(buf).cuda()
            o = torch.full((B, T1 - 1, K), -1, dtype=torch.int64, device='cuda')
            ws = torch.zeros(ops.sample_negatives_workspace(B, T1, buf_len, K), dtype=torch.uint8, device='cuda')
            ops.sample_negatives(d_all, 0, B, d_buf, K, nfb, 42, step, o, ws)
            torch.cuda.synchronize()
            got = o.cpu().numpy()
            eq = bool(np.array_equal(got, ref))
            # data-parallel slice: sessions [B//2, B) with the global pool
            o2 = torch.full((B - B // 2, T1 - 1, K), -1, dtype=torch.int64, device='cuda')
            ops.sample_negatives(d_all, B // 2, B - B // 2, d_buf, K, nfb, 42, step, o2, ws)
            torch.cuda.synchronize()
            eq2 = bool(np.array_equal(o2.cpu().numpy(), ref[B // 2:]))
            out.append({'case': ci, 'step': step, 'equal': eq, 'equal_dp_slice': eq2, 'mismatch': int((got != ref).sum()),
                        'nonzero_frac': float((ref != 0).mean()), 'ok': eq and eq2})
    return out


def fam_rnn():
    import torch
    from chameleon_recsys_b200 import ops
    out = []
    for (B, Hp, maxlen) in [(7, 64, 4), (64, 256, 19), (33, 256, 9)]:
        torch.manual_seed(B)
        lens = torch.randint(1, maxlen + 1, (B,))
        off = torch.zeros(B + 1, dtype=torch.int32)
        off[1:] = torch.cumsum(lens, 0).int()
        L = int(off[-1])
        gx = torch.randn(L, 2 * Hp, device='cuda') * 0.5
        Wh = torch.randn(Hp, 2 * Hp, device='cuda') / (Hp ** 0.5)
        dH = torch.randn(L, Hp, device='cuda')
        # torch reference (fp64 autograd)
        gxr = gx.double().clone().requires_grad_(True)
        Whr = Wh.double().clone().requires_grad_(True)
        hs = []
        for b in range(B):
            h = torch.zeros(Hp, dtype=torch.float64, device='cuda')
            for t in range(int(lens[b])):
                a = gxr[int(off[b]) + t] + h @ Whr
                g = torch.sigmoid(a[:Hp] + 1.0); c = torch.tanh(a[Hp:])
                h = g * h + (1 - g) * c
                hs.append(h)
        Href = torch.stack(hs)
        (Href * dH.double()).sum().backward()
        h_out = torch.zeros(L, Hp, device='cuda'); gate = torch.zeros_like(h_out); cand = torch.zeros_like(h_out)
        d_off = off.cuda()
        ops.ugrnn_fwd(gx, Wh, d_off, B, Hp, h_out, gate, cand)
        WhT = torch.zeros(2 * Hp, Hp, device='cuda')
        ops.transpose(Wh, Hp, 2 * Hp, 2 * Hp, WhT, Hp)
        d_gx = torch.zeros(L, 2 * Hp, device='cuda'); h_prev = torch.zeros(L, Hp, device='cuda')
        ops.ugrnn_bwd(dH, h_out, gate, cand, WhT, d_off, B, Hp, d_gx, h_prev)
        torch.cuda.synchronize()
        e_f = (h_out.double() - Href).abs().max().item()
        e_b = (d_gx.double() - gxr.grad).abs().max().item()
        dWh = h_prev.double().t() @ d_gx.double()
        e_w = (dWh - Whr.grad).abs().max().item()
        e_t = (WhT - Wh.t()).abs().max().item()
        out.append({'B': B, 'Hp': Hp, 'L': L, 'fwd_err': e_f, 'dgx_err': e_b, 'dWh_err': e_w, 'transpose_err': e_t,
                    'ok': e_f < 1e-4 and e_b < 1e-4 and e_w < 1e-3 and e_t == 0})
    return out


def fam_loss():
    import torch
    from chameleon_recsys_b200 import ops
    out = []
    for (n_pos, n_cand, Cdim, tau) in [(5, 11, 64, 1.0), (486, 51, 1024, 0.1), (100, 101, 256, 0.2)]:
        torch.manual_seed(n_pos)
        cand = torch.randn(n_pos * n_cand, Cdim, device='cuda') * 0.5
        pred = torch.randn(n_pos, Cdim, device='cuda') * 0.5
        prod = torch.zeros_like(cand)
        ops.mul_pred(cand, pred, n_pos, n_cand, Cdim, prod)
        ref = cand.view(n_pos, n_cand, Cdim) * pred[:, None, :]
        e1 = (prod.view(n_pos, n_cand, Cdim) - ref).abs().max().item()
        dprod = torch.randn_like(cand)
        dc = torch.zeros_like(cand); dp = torch.zeros_like(pred)
        ops.mul_pred_bwd(dprod, cand, pred, n_pos, n_cand, Cdim, dc, dp)
        e2 = (dc.view(n_pos, n_cand, Cdim) - dprod.view(n_pos, n_cand, Cdim) * pred[:, None, :]).abs().max().item()
        e3 = (dp.double() - (dprod.view(n_pos, n_cand, Cdim).double() * cand.view(n_pos, n_cand, Cdim).double()).sum(1)).abs().max().item()
        # score + softmax CE
        ld_z = 32
        z3 = torch.randn(n_pos * n_cand, ld_z, device='cuda')
        m4 = torch.zeros(32, 4, device='cuda'); m4[:, 0] = torch.randn(32, device='cuda') * 0.3
        c4 = torch.zeros(4, device='cuda'); c4[0] = 0.05
        z3r = z3.double().clone().requires_grad_(True)
        m4r = m4[:, 0].double().clone().requires_grad_(True)
        c4r = c4[:1].double().clone().requires_grad_(True)
        zl = torch.nn.functional.leaky_relu(z3r, 0.2)      # z3 given to the kernel is POST activation
        z3_post = zl.detach().float().contiguous()
        logit_r = ((zl @ m4r + c4r) / tau).view(n_pos, n_cand)
        loss_r = -(torch.log_softmax(logit_r, -1)[:, 0]).sum() / n_pos
        loss_r.backward()
        logits = torch.zeros(n_pos, n_cand, device='cuda'); loss = torch.zeros(1, device='cuda')
        dz = torch.zeros_like(z3); dm4 = torch.zeros_like(m4); dc4 = torch.zeros_like(c4)
        ops.score_softmax_ce(z3_post, ld_z, 32, m4, 4, c4, n_pos, n_cand, 1.0 / tau, 1.0 / n_pos, logits, loss, dz, dm4, dc4)
        torch.cuda.synchronize()
        e4 = (logits.double() - logit_r).abs().max().item()
        e5 = abs(loss.item() - loss_r.item())
        e6 = (dz.double() - z3r.grad).abs().max().item()      # kernel returns grad wrt PRE-activation == grad wrt z3r here
        e7 = (dm4[:, 0].double() - m4r.grad).abs().max().item()
        e8 = abs(dc4[0].item() - c4r.grad.item())
        # cosine mode
        candr = cand.double().clone().requires_grad_(True); predr = pred.double().clone().requires_grad_(True)
        cs = (torch.nn.functional.normalize(candr.view(n_pos, n_cand, Cdim), dim=-1) *
              torch.nn.functional.normalize(predr, dim=-1)[:, None, :]).sum(-1) / tau
        lc = -(torch.log_softmax(cs, -1)[:, 0]).sum() / n_pos
        lc.backward()
        logits2 = torch.zeros(n_pos, n_cand, device='cuda'); loss2 = torch.zeros(1, device='cuda')
        dcc = torch.zeros_like(cand); dpp = torch.zeros_like(pred)
        ops.cosine_softmax_ce(cand, pred, n_pos, n_cand, Cdim, 1.0 / tau, 1.0 / n_pos, logits2, loss2, dcc, dpp)
        torch.cuda.synchronize()
        e9 = (logits2.double() - cs).abs().max().item()
        e10 = abs(loss2.item() - lc.item())
        e11 = (dcc.double() - candr.grad).abs().max().item()
        e12 = (dpp.double() - predr.grad).abs().max().item()
        errs = dict(mul=e1, dcand=e2, dpred=e3, logits=e4, loss=e5, dz=e6, dm4=e7, dc4=e8, cos_logits=e9, cos_loss=e10,
                    cos_dcand=e11, cos_dpred=e12)
        out.append({'n_pos': n_pos, 'n_cand': n_cand, 'C': Cdim, **errs, 'ok': all(v < 2e-3 for v in errs.values())})
    return out


def fam_misc():
    import torch
    from chameleon_recsys_b200 import ops
    torch.manual_seed(0)
    n = 4096 * 33
    w = torch.randn(n, device='cuda'); g = torch.randn(n, device='cuda') * 0.1
    m = torch.zeros(n, device='cuda'); v = torch.zeros(n, device='cuda')
    wr, mr, vr = w.double().clone(), m.double().clone(), v.double().clone()
    reg_end = 4096 * 10
    for step in (1, 2, 3):
        ops.adam_tf(w, g, m, v, n, reg_end, 1e-3, 1e-2, step)
        gg = g.double().clone(); gg[:reg_end] += 1e-3 * wr[:reg_end]
        mr = 0.9 * mr + 0.1 * gg; vr = 0.999 * vr + 0.001 * gg * gg
        lr_t = 1e-2 * (1 - 0.999 ** step) ** 0.5 / (1 - 0.9 ** step)
        wr = wr - lr_t * mr / (vr.sqrt() + 1e-8)
    torch.cuda.synchronize()
    e_adam = (w.double() - wr).abs().max().item()
    x = torch.randn(1000, 516, device='cuda')
    cs = torch.ones(512, device='cuda')
    ops.colsum_add(x, 1000, 512, 516, cs)
    e_cs = (cs.double() - (1 + x[:, :512].double().sum(0))).abs().max().item()
    l2 = torch.zeros(1, device='cuda')
    ops.l2_loss_add(x, x.numel(), 1e-3, l2)
    torch.cuda.synchronize()
    e_l2 = abs(l2.item() - 1e-3 * (x.double() ** 2).sum().item() / 2) / l2.item()
    return [{'adam_err': e_adam, 'colsum_err': e_cs, 'l2_rel': e_l2, 'ok': e_adam < 1e-5 and e_cs < 1e-3 and e_l2 < 1e-4}]


FAMILIES = {'gemm_kk': fam_gemm_kk, 'gemm_km': fam_gemm_km, 'gemm_mk': fam_gemm_mk, 'gemm_mm': fam_gemm_mm,
            'gemm_epi': fam_gemm_epi, 'gemm_bf16': fam_gemm_bf16, 'gather': fam_gather, 'sampler': fam_sampler, 'rnn': fam_rnn, 'loss': fam_loss,
            'misc': fam_misc}


def main():
    os.makedirs(OUT, exist_ok=True)
    if len(sys.argv) > 2 and sys.argv[1] == '--child':
        fam = sys.argv[2]
        res = FAMILIES[fam]()
        print('DIAG_JSON ' + json.dumps(res))
        return
    fams = sys.argv[1:] or list(FAMILIES)
    report = {}
    for fam in fams:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', fam], capture_output=True, text=True,
                               timeout=600, cwd=ROOT)
            lines = [l for l in r.stdout.splitlines() if l.startswith('DIAG_JSON ')]
            if lines:
                report[fam] = {'results': json.loads(lines[-1][10:]), 'rc': r.returncode}
            else:
                report[fam] = {'error': (r.stdout[-2000:] + '\n' + r.stderr[-4000:]), 'rc': r.returncode}
        except subprocess.TimeoutExpired:
            report[fam] = {'error': 'timeout'}
        report[fam]['seconds'] = round(time.time() - t0, 1)
        res = report[fam].get('results')
        print(fam, 'rc', report[fam].get('rc'), 'ok' if res and all(x.get('ok') for x in res) else 'FAIL',
              report[fam]['seconds'], 's', flush=True)
        if res:
            for x in res:
                if not x.get('ok'):
                    print('   FAIL', json.dumps(x))
        else:
            print(report[fam].get('error', '')[-3000:])
    with open(os.path.join(OUT, 'diag.json'), 'w') as f:
        json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
