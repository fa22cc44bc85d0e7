"""The session-cell recurrence kernels (csrc/rnn.cu) on the GPU (pytest -m gpu): UGRNN, GRU and LSTM forward and backward
against an fp64 torch recurrence at every accepted hidden size, and the hidden sizes every entry point accepts."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

CELLS = ('ugrnn', 'gru', 'lstm')
HPS = (32, 64, 128, 256, 512, 1024)
# gx column blocks per unit: UGRNN gate | candidate, GRU r | u | candidate, LSTM i | j | f | o
GX_BLOCKS = {'ugrnn': 2, 'gru': 3, 'lstm': 4}
# session lengths per case: an empty session, single steps, mixed, long; more sessions than one CTA holds (SB = 4)
LENGTHS = {'single': [1], 'empty_and_one': [0, 1, 0], 'mixed': [3, 0, 1, 7, 2, 1, 5, 4, 20, 1, 2]}


def make_inputs(cell, Hp, lengths):
    """Seeded inputs of one case: pre-activations gx [L, nHp], recurrent weights Wh [Hp, nHp] (the GRU's Whg | Whc side by
    side), output gradient dH [L, Hp] and the session offsets."""
    import torch
    lens = LENGTHS[lengths]
    B = len(lens)
    torch.manual_seed(Hp + B)
    off = torch.zeros(B + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(torch.tensor(lens), 0).int()
    L = int(off[-1])
    n = GX_BLOCKS[cell]
    gx = torch.randn(L, n * Hp, device='cuda') * 0.5
    Wh = torch.randn(Hp, n * Hp, device='cuda') / (Hp ** 0.5)
    dH = torch.randn(L, Hp, device='cuda')
    return gx, Wh, dH, off


def reference(cell, gx, Wh, lens, dH):
    """fp64 recurrence of `cell` over pre-activations gx and its autograd backward of sum(h * dH): the saved outputs the
    kernels write, h entering each step, d(gx) and d(Wh)."""
    import torch
    H = Wh.shape[0]
    gxr = gx.double().clone().requires_grad_(True)
    Whr = Wh.double().clone().requires_grad_(True)
    saved = {}
    r = 0
    for n in lens:
        h = torch.zeros(H, dtype=torch.float64, device=gx.device)
        c = torch.zeros_like(h)
        for _ in range(n):
            out = {'h_prev': h}
            if cell == 'ugrnn':                      # tools/gpu_diag.py::fam_rnn
                a = gxr[r] + h @ Whr
                g, cd = torch.sigmoid(a[:H] + 1.0), torch.tanh(a[H:])
                h = g * h + (1 - g) * cd
                out.update(gate=g, cand=cd)
            elif cell == 'gru':                      # include/nar_b200.h, nar_gru_fwd
                a = gxr[r, :2 * H] + h @ Whr[:, :2 * H]
                rg, u = torch.sigmoid(a[:H]), torch.sigmoid(a[H:])
                rh = rg * h
                cd = torch.tanh(gxr[r, 2 * H:] + rh @ Whr[:, 2 * H:])
                h = u * h + (1 - u) * cd
                out.update(r=rg, u=u, cand=cd, rh=rh)
            else:                                    # LSTMCell, forget bias 1.0
                z = gxr[r] + h @ Whr
                i, j, f, o = torch.sigmoid(z[:H]), torch.tanh(z[H:2 * H]), torch.sigmoid(z[2 * H:3 * H] + 1.0), torch.sigmoid(z[3 * H:])
                c = f * c + i * j
                h = o * torch.tanh(c)
                out.update(c=c, act=torch.cat([i, j, f, o]))
            out['h'] = h
            for k, v in out.items():
                saved.setdefault(k, []).append(v)
            r += 1
    saved = {k: torch.stack(v) for k, v in saved.items()}
    (saved['h'] * dH.double()).sum().backward()
    saved = {k: v.detach() for k, v in saved.items()}
    saved['d_gx'], saved['dWh'] = gxr.grad, Whr.grad
    return saved


def run_kernels(cell, gx, Wh, dH, off):
    """Forward then backward kernels of `cell` on one case; returns every output they write and the dWh the engine's
    weight-gradient GEMMs form from them."""
    import torch
    from chameleon_recsys_b200 import ops
    L, Hp = dH.shape
    B = off.numel() - 1
    d_off = off.cuda()
    z = lambda *s: torch.zeros(*s, device='cuda')  # noqa: E731
    n = GX_BLOCKS[cell]
    d_gx, h_prev = z(L, n * Hp), z(L, Hp)
    WhT = z(n * Hp, Hp)
    out = {'h': z(L, Hp)}
    if cell == 'ugrnn':
        out.update(gate=z(L, Hp), cand=z(L, Hp))
        ops.ugrnn_fwd(gx, Wh, d_off, B, Hp, out['h'], out['gate'], out['cand'])
        ops.transpose(Wh, Hp, 2 * Hp, 2 * Hp, WhT, Hp)
        ops.ugrnn_bwd(dH, out['h'], out['gate'], out['cand'], WhT, d_off, B, Hp, d_gx, h_prev)
        dWh = h_prev.double().t() @ d_gx.double()
    elif cell == 'gru':
        Whg, Whc = Wh[:, :2 * Hp].contiguous(), Wh[:, 2 * Hp:].contiguous()
        out.update(r=z(L, Hp), u=z(L, Hp), cand=z(L, Hp), rh=z(L, Hp))
        ops.gru_fwd(gx, Whg, Whc, d_off, B, Hp, out['h'], out['r'], out['u'], out['cand'], out['rh'])
        WhgT, WhcT = WhT[:2 * Hp], WhT[2 * Hp:]
        ops.transpose(Whg, Hp, 2 * Hp, 2 * Hp, WhgT, Hp)
        ops.transpose(Whc, Hp, Hp, Hp, WhcT, Hp)
        ops.gru_bwd(dH, out['h'], out['r'], out['u'], out['cand'], WhgT, WhcT, d_off, B, Hp, d_gx, h_prev)
        dg, dc = d_gx[:, :2 * Hp].double(), d_gx[:, 2 * Hp:].double()
        dWh = torch.cat([h_prev.double().t() @ dg, out['rh'].double().t() @ dc], 1)
    else:
        out.update(act=gx.clone(), c=z(L, Hp))                # gx is overwritten in place with the activated gates
        ops.lstm_fwd(out['act'], Wh, d_off, B, Hp, out['h'], out['c'])
        ops.transpose(Wh, Hp, 4 * Hp, 4 * Hp, WhT, Hp)
        ops.lstm_bwd(dH, out['h'], out['c'], out['act'], WhT, d_off, B, Hp, d_gx, h_prev)
        dWh = h_prev.double().t() @ d_gx.double()
    torch.cuda.synchronize()
    out.update(h_prev=h_prev, d_gx=d_gx, dWh=dWh)
    return out


@pytest.mark.parametrize('Hp', HPS)
@pytest.mark.parametrize('lengths', sorted(LENGTHS))
@pytest.mark.parametrize('cell', CELLS)
def test_recurrence_kernels_match_fp64(cell, lengths, Hp):
    gx, Wh, dH, off = make_inputs(cell, Hp, lengths)
    ref = reference(cell, gx, Wh, LENGTHS[lengths], dH)
    got = run_kernels(cell, gx, Wh, dH, off)
    assert set(got) == set(ref)
    for k in sorted(set(ref) - {'d_gx', 'dWh'}):
        assert (got[k].double() - ref[k]).abs().max().item() < 1e-5, k
    scale = max(ref['d_gx'].abs().max().item(), 1e-30)
    assert (got['d_gx'].double() - ref['d_gx']).abs().max().item() < 1e-5 * max(scale, 1.0)
    assert (got['dWh'] - ref['dWh']).abs().max().item() < 1e-4 * max(ref['dWh'].abs().max().item(), 1.0)


def test_recurrence_kernels_accept_exactly_the_supported_sizes():
    """Every entry point accepts Hp in {32, 64, ..., 1024} and rejects every other multiple of 4 up to 2048 (B = 0: the
    shape check runs, nothing launches)."""
    import torch
    from chameleon_recsys_b200 import _lib, ops
    ctx = ops.context()
    x = ops._p(torch.zeros(16, device='cuda'))
    off = ops._p(torch.zeros(2, dtype=torch.int32, device='cuda'))
    st = ops._stream()
    lib, h = ctx.lib, ctx.handle
    calls = {
        'ugrnn_fwd': lambda Hp: lib.nar_ugrnn_fwd(h, x, x, off, 0, Hp, x, x, x, st),
        'ugrnn_bwd': lambda Hp: lib.nar_ugrnn_bwd(h, x, x, x, x, x, off, 0, Hp, x, x, st),
        'gru_fwd': lambda Hp: lib.nar_gru_fwd(h, x, x, x, off, 0, Hp, x, x, x, x, x, st),
        'gru_bwd': lambda Hp: lib.nar_gru_bwd(h, x, x, x, x, x, x, x, off, 0, Hp, x, x, st),
        'lstm_fwd': lambda Hp: lib.nar_lstm_fwd(h, x, x, off, 0, Hp, x, x, st),
        'lstm_bwd': lambda Hp: lib.nar_lstm_bwd(h, x, x, x, x, x, off, 0, Hp, x, x, st),
    }
    for name, call in calls.items():
        accepted = [Hp for Hp in range(4, 2049, 4) if call(Hp) == 0]
        assert accepted == list(HPS), name
    with pytest.raises(_lib.NarError):
        ops.lstm_fwd(torch.zeros(16, device='cuda'), torch.zeros(16, device='cuda'), torch.zeros(2, dtype=torch.int32, device='cuda'),
                     1, 16, torch.zeros(16, device='cuda'), torch.zeros(16, device='cuda'))
