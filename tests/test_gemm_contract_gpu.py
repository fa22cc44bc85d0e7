"""The wgmma GEMM (nar_gemm_tf32 / nar_gemm_tf32_dt) and nar_pack_bf16x3 against fp64, at the operand strides, offsets
and shapes the engine launches and at the edges of the kernel's tiles.

Storage.  Every operand, bias, aux and b_lo is a strided view at a 16-byte-aligned offset inside a larger buffer, and
everything outside its logical region is NaN: the floats before it, the row tails past K (past M / N for MN-major
storage) and the rows after it.  A bf16x3 plane is NaN outside the columns the pack writes; inside them, the entries
for k >= K of the last 32-k block are the pack's own zeros.  A read outside any operand therefore shows up as NaN in D.
D is a view with guard rows and columns on every side; its whole buffer is prefilled with a signalling-NaN sentinel
(bits 0x7fa5a5a5, which any arithmetic would quiet) and every guard float must keep its bits.  Overwritten outputs start
as NaN, accumulating ones from a random prefill D0.

Bar.  Each element of D is compared with the fp64 result of the same operation, with a bar of its own:

    |D - ref| <= c_mode(K) * S * G  +  c_e * T,        S = |A| |B|^T in fp64,

where G = |act'(aux)| for a dact epilogue (else 1: leaky and tanh are 1-Lipschitz) and T collects the magnitudes the
epilogue rounds: |v| + |bias| + |act(v + bias)| (times G), plus |act(.)| (1 + aux^2) for the dact factor, plus, when
accumulating, the number of splits times (|D0| + S G).  c_e = 2^-21 (8 u, u = 2^-24) covers the bias add, the leaky
multiply, tanhf's 2 ulp, the dact factor and its multiply, and each red.add.

c_mode(K) = p_mode + n_mode K 2^-23, the first-order bound of the product plus the accumulation:
  - single-pass TF32 (precision 1, mode 0): the tensor core reads A's and B's raw fp32 bits and truncates each to TF32
    (10 stored mantissa bits), a relative error below 2^-10 per operand: p_0 = 2 * 2^-10 + 2^-20.
  - 3xTF32 (precision 3, B split in-kernel or from a b_lo plane, modes 1 / 2): x = hi + lo with hi = x truncated to
    TF32 and lo exact in fp32, |lo| < 2^-10 |x|.  The MMA truncates lo to TF32 (error < 2^-20 |x|) for A_lo and B_lo,
    and A_lo B_lo is dropped: p_1 = p_2 = 3 * 2^-20.
  - bf16x3 (precision 4, mode 4): hi = bf16(x) (RNE to 8 significant bits, |x - hi| <= 2^-8 |x|), lo = bf16(x - hi)
    (|error| <= 2^-8 |x - hi| <= 2^-16 |x|), A_lo B_lo dropped: p_4 = 3 * 2^-16.
  - Accumulation: each product term passes through an fp32 accumulator that truncates to the largest exponent in play,
    at most 2^-23 of the running |sum| <= S per term: n = 1 term per k for TF32, 3 for 3xTF32 and bf16x3.
Each test's docstring gives the largest error/bar measured over its cases on an H100 80GB HBM3 (SXM, 700 W power
limit).  Where that stayed below 0.05, the test's bar is a stated fraction of this bound.
"""
import ctypes as C
import functools
import math

import pytest
import torch

from chameleon_recsys_b200 import ops
from chameleon_recsys_b200._lib import GemmEpilogue, NarError, load

pytestmark = pytest.mark.gpu

NAR_ERR_INVALID = -1
CE = 2.0 ** -21
P_MODE = {0: 2 * 2.0 ** -10 + 2.0 ** -20, 1: 3 * 2.0 ** -20, 2: 3 * 2.0 ** -20, 4: 3 * 2.0 ** -16}
N_MODE = {0: 1, 1: 3, 2: 3, 4: 3}
PRECISION = {0: 1, 1: 3, 2: 3, 4: 4}
SLOPE = float(torch.tensor(0.2, dtype=torch.float32))        # the kernel's leaky slope, 0.2f
SENTINEL = 0x7FA5A5A5
PRE = 8                                                       # floats before each view: 32 bytes
_WORST = []


@pytest.fixture(autouse=True)
def _worst_ratio(record_property):
    """Records the test's largest error/bar (junit property worst_err_over_bar)."""
    _WORST.clear()
    yield
    if _WORST:
        record_property('worst_err_over_bar', '%.4g' % max(_WORST))


def c_mode(mode, K):
    return P_MODE[mode] + N_MODE[mode] * K * 2.0 ** -23


def _ld4(n, extra=0):
    return (n + 3) // 4 * 4 + extra


# ------------------------------------------------------------------------------------------------------------ storage
def nan_view(rows, cols, ld, col0=0, dtype=torch.float32):
    """A [rows, cols] view with row stride ld starting at column col0 of a NaN buffer: PRE elements before it, NaN row
    tails and one NaN row after it."""
    assert col0 + cols <= ld
    buf = torch.full((PRE + rows * ld + ld,), float('nan'), dtype=dtype, device='cuda')
    return buf[PRE:PRE + rows * ld].view(rows, ld)[:, col0:col0 + cols]


def operand(mn, K, ld, kmajor, g, col0=0, scale=1.0):
    """Operand of logical shape [mn, K] stored K-major ([mn, ld]) or MN-major ([K, ld]) in NaN storage; returns
    (view, fp64 [mn, K])."""
    v = nan_view(mn, K, ld, col0) if kmajor else nan_view(K, mn, ld, col0)
    v.copy_(torch.randn(v.shape, device='cuda', generator=g) * scale)
    return v, (v if kmajor else v.t()).double()


def vec(n, g, scale=1.0):
    v = nan_view(1, n, _ld4(n))[0]
    v.copy_(torch.randn(n, device='cuda', generator=g) * scale)
    return v


class Dest:
    """D [rows, cols] (row stride ld, from column col0) with GR guard rows before and after, in a buffer of sentinel
    bits; the view starts NaN or at `init`."""
    GR = 2

    def __init__(self, rows, cols, ld, col0=4, init=None):
        assert col0 % 4 == 0 and col0 + cols <= ld
        n = PRE + (rows + 2 * self.GR) * ld + 64
        self.bits = torch.full((n,), SENTINEL, dtype=torch.int32, device='cuda')
        self.buf = self.bits.view(torch.float32)
        self.ld = ld
        store = self.buf[PRE:PRE + (rows + 2 * self.GR) * ld].view(rows + 2 * self.GR, ld)
        self.view = store[self.GR:self.GR + rows, col0:col0 + cols]
        self.mask = torch.ones(n, dtype=torch.bool, device='cuda')
        self.mask[PRE:PRE + (rows + 2 * self.GR) * ld].view(rows + 2 * self.GR, ld)[self.GR:self.GR + rows,
                                                                                    col0:col0 + cols] = False
        if init is None:
            self.view.fill_(float('nan'))
        else:
            self.view.copy_(init)
        self.snapshot = self.bits.clone()

    def guards_intact(self):
        return bool((self.bits[self.mask] == SENTINEL).all())

    def untouched(self):
        return torch.equal(self.bits, self.snapshot)


# ---------------------------------------------------------------------------------------------------- bf16x3 planes
_SCRATCH = {}


def pack(Ws, outs, Ks, Ns, ld_outs, scratch=None, n=None):
    """nar_pack_bf16x3 over the matrices Ws[i] (views [K, N], row stride .stride(0)) into outs[i] (bf16 / int16 views
    with row stride ld_outs[i]); returns the status code (n: the count passed, len(Ws) by default)."""
    n = len(Ws) if n is None else n
    if scratch is None:
        scratch = _SCRATCH.setdefault('s', torch.zeros(32 * 32, dtype=torch.uint8, device='cuda'))
    arr = lambda t, vals: (t * len(vals))(*vals)        # noqa: E731
    return load().nar_pack_bf16x3(arr(C.c_void_p, [w.data_ptr() for w in Ws]), arr(C.c_void_p, [o.data_ptr() for o in outs]),
                                  arr(C.c_int32, Ks), arr(C.c_int32, Ns), arr(C.c_int32, [w.stride(0) for w in Ws]),
                                  arr(C.c_int32, ld_outs), n, C.c_void_p(scratch.data_ptr()),
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))


def plane_ref(W, K, N):
    """The plane torch's round-to-nearest-even bf16 gives: [N, ceil(K/32) 64] int16 bits."""
    kt = (K + 31) // 32
    x = torch.zeros(kt * 32, N, device='cuda')
    x[:K] = W[:K, :N]
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    out = torch.empty(N, kt, 64, dtype=torch.bfloat16, device='cuda')
    out[:, :, :32] = hi.t().reshape(N, kt, 32)
    out[:, :, 32:] = lo.t().reshape(N, kt, 32)
    return out.reshape(N, kt * 64).view(torch.int16)


def make_plane(W, K, N, ld_bf16):
    """bf16x3 plane of W [K, N] in NaN storage with row stride ld_bf16."""
    plane = nan_view(N, ld_bf16, ld_bf16, dtype=torch.bfloat16)
    assert pack([W], [plane], [K], [N], [ld_bf16]) == 0
    return plane


# -------------------------------------------------------------------------------------------------------- one GEMM
def run_case(M, N, K, *, mode, a_k=True, b_k=True, lda=None, ldb=None, a_col0=0, b_col0=0, ldd=None, d_col0=4,
             bias=False, act=0, dact=0, ld_aux=None, accumulate=False, split_k=1, trans_d=False, ld_bf16=None,
             aux_special=None, scale=1.0, tighten=1.0, seed=0):
    """Runs one GEMM with NaN storage around every input and a guarded D, and checks it against fp64 (the bar times
    `tighten`)."""
    g = torch.Generator(device='cuda').manual_seed(seed * 1000003 + M * 7919 + N * 131 + K * 7 + mode)
    lda = lda or _ld4(K if a_k else M, 4)
    A, A64 = operand(M, K, lda, a_k, g, a_col0, scale)
    kw = dict(precision=PRECISION[mode])
    if mode == 4:
        assert b_k
        Wv, W64 = operand(N, K, ldb or _ld4(N, 4), False, g, b_col0)       # the weight [in, out] = MN-major B
        kt = (K + 31) // 32
        plane = make_plane(Wv, K, N, ld_bf16 or kt * 64)
        B, B64, ldb = None, W64, 0
        kw.update(b_bf16=plane, ld_bf16=plane.stride(0))
    else:
        ldb = ldb or _ld4(K if b_k else N, 8)
        B, B64 = operand(N, K, ldb, b_k, g, b_col0)
        if mode == 2:
            lo = nan_view(*B.shape, ldb, b_col0)
            hi = (B.contiguous().view(torch.int32) & -8192).view(torch.float32)
            lo.copy_(B - hi)
            kw['b_lo'] = lo
    v = A64 @ B64.t()
    S = A64.abs() @ B64.abs().t()
    out = v
    T = torch.zeros_like(v)
    G = torch.ones_like(v)
    if bias:
        b = vec(N, g)
        kw['bias'] = b
        out = out + b.double()
        T = T + b.double().abs()
    if act:
        out = torch.where(out > 0, out, SLOPE * out) if act == 1 else torch.tanh(out)
        kw['act'] = act
    if bias or act:
        T = T + v.abs() + out.abs()
    if dact:
        ld_aux = ld_aux or _ld4(N, 8)
        aux = nan_view(M, N, ld_aux)
        y = torch.randn(M, N, device='cuda', generator=g)
        if dact == 2:
            y = torch.tanh(y)
        if aux_special is not None:
            for val, step in aux_special:              # val at every step-th element, from element step // 2
                y.view(-1)[step // 2::step] = val
        aux.copy_(y)
        y64 = aux.double()
        gr = torch.where(y64 > 0, 1.0, SLOPE) if dact == 1 else 1.0 - y64 * y64
        T = T * gr.abs() + out.abs() * (1 + y64 * y64)
        G = gr.abs()
        out = out * gr
        kw.update(dact=dact, aux=aux, ld_aux=ld_aux)
    rows, cols = (N, M) if trans_d else (M, N)
    ldd = ldd or _ld4(d_col0 + cols, 4)
    D0 = None
    if accumulate:
        D0 = torch.randn(rows, cols, device='cuda', generator=g)
        kw.update(accumulate=True)
    kw['split_k'] = split_k
    dst = Dest(rows, cols, ldd, d_col0, D0)
    ops.gemm(A, B, dst.view, M, N, K, a_kmajor=a_k, b_kmajor=b_k, lda=lda, ldb=ldb, ldd=ldd, trans_d=trans_d, **kw)
    torch.cuda.synchronize()
    got = dst.view.t() if trans_d else dst.view
    bar = (c_mode(mode, K) * S * G + CE * T) * tighten
    if accumulate:
        splits = (K + 31) // 32 if split_k != 1 else 1
        d0 = (D0.t() if trans_d else D0).double()
        out = out + d0
        bar = bar + CE * splits * (d0.abs() + S * G) * tighten
    check(got, out, bar)
    assert dst.guards_intact(), 'a write landed outside D'


def check(got, ref, bar):
    err = (got.double() - ref).abs()
    bad = ~(err <= bar)                                  # NaN fails
    ratio = float((err / bar.clamp_min(1e-300)).nan_to_num(math.inf).max()) if err.numel() else 0.0
    _WORST.append(ratio)
    if bad.any():
        i = tuple(int(x) for x in bad.nonzero()[0])
        raise AssertionError('%d of %d elements outside the bar; first at %s: got %r ref %r bar %r (worst err/bar %.3g)'
                             % (int(bad.sum()), bad.numel(), i, float(got[i]), float(ref[i]), float(bar[i]), ratio))


# ------------------------------------------------------------------------------------------------ engine call table
@functools.lru_cache(maxsize=None)
def _dims(problem):
    from chameleon_recsys_b200.harness import make_problem
    pb = make_problem(problem)
    n_cand = pb.hp.train_total_negative_samples + 1
    return dict(C=pb.layout.C, Fp=pb.plan.Fp, c0=pb.plan.ctx_col0, Hp=pb.layout.Hp, K=n_cand - 1, n_cand=n_cand,
                # a small L everywhere, and G1's 23.6 K candidate rows (463 positions x 51) for layer 2 and the scorer
                L=77 if problem == 'tiny' else 200, Lr=463 if problem == 'g1' else 77)


GATES = {'ugrnn': 2, 'gru': 3, 'lstm': 4}

# Seq::fwd(X, ldx, W, ldw, b, Y, ldy, M, N, Kd, act, x_kmajor): Y = act(X W + b), W [in, out] MN-major (or its plane)
# Seq::dgrad(dY, lddy, W, ldw, dX, lddx, M, n_in, n_out, dact, aux, ld_aux, accumulate): K-major dY and W
# Seq::wgrad(X, ldx, dY, lddy, W, ldw, n_in, n_out, rows): dW += X^T dY, both MN-major, split-K chosen by the library
# Seq::wgrad_xt(XT, ldxt, dY, lddy, W, ldw, n_in, n_out, rows): dW^T += dY^T X through nar_gemm_tf32_dt
FWD_SITES = ['clicked_rows_forward:car_layer1', 'clicked_rows_forward:car_layer2',
             'clicked_rows_forward:rnn_input_ugrnn', 'clicked_rows_forward:rnn_input_gru',
             'clicked_rows_forward:rnn_input_lstm', 'clicked_rows_forward:rnn_input_layer2', 'clicked_rows_forward:fc1',
             'clicked_rows_forward:fc2', 'run_step:dedup_positives', 'run_step:dedup_item_half',
             'run_step:dedup_context_half', 'run_step:dedup_layer2_h1ct', 'run_step:car_layer1_candidates',
             'run_step:car_layer2_candidates', 'scorer:m1_product', 'scorer:m2', 'scorer:m3',
             'run_recommend:context_half', 'run_recommend:item_half', 'run_recommend:car_layer2']
BWD_SITES = ['run_step:scorer_m3_dgrad', 'run_step:scorer_m2_dgrad', 'run_step:scorer_m1_dgrad', 'run_step:fc2_dgrad',
             'run_step:fc1_dgrad', 'run_step:rnn_input_dgrad_ugrnn', 'run_step:rnn_input_dgrad_gru',
             'run_step:rnn_input_dgrad_lstm', 'run_step:rnn_layer2_dgrad', 'run_step:car_layer2_candidates_dgrad',
             'run_step:car_layer2_clicked_dgrad', 'run_step:car_layer1_dedup_dgrad',
             'run_step:car_layer1_context_negatives_dgrad', 'run_step:car_layer1_dgrad',
             'run_step:scorer_m3_wgrad', 'run_step:scorer_m2_wgrad', 'run_step:scorer_m1_wgrad',
             'run_step:car_layer2_candidates_wgrad', 'run_step:car_layer2_candidates_wgrad_xt', 'run_step:fc2_wgrad',
             'run_step:fc1_wgrad', 'run_step:rnn_wx_wgrad_ugrnn', 'run_step:rnn_wx_wgrad_gru', 'run_step:rnn_wx_wgrad_lstm',
             'run_step:rnn_wh_wgrad_ugrnn', 'run_step:rnn_wh_wgrad_lstm', 'run_step:gru_whg_wgrad',
             'run_step:gru_whc_wgrad', 'run_step:car_layer2_clicked_wgrad', 'run_step:car_layer1_dedup_wgrad',
             'run_step:car_layer1_context_negatives_wgrad', 'run_step:car_layer1_wgrad']


def fwd(mode, ldx, ldw, has_bias, ldy, M, N, Kd, act, x_kmajor=True, x_col0=0):
    run_case(M, N, Kd, mode=mode, a_k=x_kmajor, b_k=mode == 4, lda=ldx, ldb=ldw, a_col0=x_col0, ldd=ldy, d_col0=0,
             bias=has_bias, act=act, scale=0.25)


def dgrad(mode, lddy, ldw, lddx, M, n_in, n_out, dact, ld_aux=None, accumulate=False, dx_col0=0):
    run_case(M, n_in, n_out, mode=mode, a_k=True, b_k=True, lda=lddy, ldb=ldw, ldd=lddx, d_col0=dx_col0, dact=dact,
             ld_aux=ld_aux, accumulate=accumulate, split_k=0 if accumulate else 1)


def wgrad(mode, ldx, lddy, ldw, n_in, n_out, rows, x_col0=0, dy_col0=0):
    run_case(n_in, n_out, rows, mode=mode, a_k=False, b_k=False, lda=ldx, ldb=lddy, a_col0=x_col0, b_col0=dy_col0,
             ldd=ldw, d_col0=0, accumulate=True, split_k=0)


def wgrad_xt(mode, ldxt, lddy, ldw, n_in, n_out, rows):
    run_case(n_out, n_in, rows, mode=mode, a_k=False, b_k=True, lda=lddy, ldb=ldxt, ldd=ldw, d_col0=0, accumulate=True,
             split_k=0, trans_d=True)


def fwd_site(site, mode, d):
    C, Fp, c0, Hp, L, n_cand = d['C'], d['Fp'], d['c0'], d['Hp'], d['L'], d['n_cand']
    U, Rc, ldr = d['K'] * 20 + 1, d['Lr'] * n_cand, (d['Lr'] * n_cand + 31) // 32 * 32
    LK, TH, NONE = 1, 2, 0
    gw = {k: g * Hp for k, g in GATES.items()}
    P = 3 * 70                                           # recommend: 3 queries x a 70-candidate chunk
    calls = {
        'clicked_rows_forward:car_layer1': lambda: fwd(mode, Fp, C, True, C, L, C, Fp, LK),
        'clicked_rows_forward:car_layer2': lambda: fwd(mode, C, C, True, C, L, C, C, TH),
        'clicked_rows_forward:rnn_input_ugrnn': lambda: fwd(mode, C, gw['ugrnn'], True, gw['ugrnn'], L, gw['ugrnn'], C, NONE),
        'clicked_rows_forward:rnn_input_gru': lambda: fwd(mode, C, gw['gru'], True, gw['gru'], L, gw['gru'], C, NONE),
        'clicked_rows_forward:rnn_input_lstm': lambda: fwd(mode, C, gw['lstm'], True, gw['lstm'], L, gw['lstm'], C, NONE),
        'clicked_rows_forward:rnn_input_layer2': lambda: fwd(mode, Hp, gw['ugrnn'], True, gw['ugrnn'], L, gw['ugrnn'], Hp, NONE),
        'clicked_rows_forward:fc1': lambda: fwd(mode, Hp, 512, True, 512, L, 512, Hp, LK),
        'clicked_rows_forward:fc2': lambda: fwd(mode, 512, C, True, C, L, C, 512, TH),
        'run_step:dedup_positives': lambda: fwd(mode, Fp, C, True, C, L, C, Fp, NONE),
        'run_step:dedup_item_half': lambda: fwd(mode, Fp, C, False, C, U, C, c0, NONE),
        'run_step:dedup_context_half': lambda: fwd(mode, Fp, C, True, C, L, C, Fp - c0, NONE, x_col0=c0),
        'run_step:dedup_layer2_h1ct': lambda: fwd(mode, ldr, C, True, C, Rc, C, C, TH, x_kmajor=False),
        'run_step:car_layer1_candidates': lambda: fwd(mode, Fp, C, True, C, L * n_cand, C, Fp, LK),
        'run_step:car_layer2_candidates': lambda: fwd(mode, C, C, True, C, Rc, C, C, TH),
        'scorer:m1_product': lambda: fwd(mode, C, 128, True, 128, Rc, 128, C, LK),
        'scorer:m2': lambda: fwd(mode, 128, 64, True, 64, Rc, 64, 128, LK),
        'scorer:m3': lambda: fwd(mode, 64, 32, True, 32, Rc, 32, 64, LK),
        'run_recommend:context_half': lambda: fwd(mode, Fp, C, True, C, L, C, Fp - c0, NONE, x_col0=c0),
        'run_recommend:item_half': lambda: fwd(mode, Fp, C, False, C, 70, C, c0, NONE),
        'run_recommend:car_layer2': lambda: fwd(mode, C, C, True, C, P, C, C, TH),
    }
    calls[site]()


def bwd_site(site, mode, d):
    C, Fp, c0, Hp, L, n_cand = d['C'], d['Fp'], d['c0'], d['Hp'], d['L'], d['n_cand']
    U, Rc, ldr = d['K'] * 20 + 1, d['Lr'] * n_cand, (d['Lr'] * n_cand + 31) // 32 * 32
    NB, R = 2 * L + U, L + L * n_cand
    LK, TH, NONE = 1, 2, 0
    gw = {k: g * Hp for k, g in GATES.items()}
    calls = {
        'run_step:scorer_m3_dgrad': lambda: dgrad(mode, 32, 32, 64, Rc, 64, 32, LK, 64),
        'run_step:scorer_m2_dgrad': lambda: dgrad(mode, 64, 64, 128, Rc, 128, 64, LK, 128),
        'run_step:scorer_m1_dgrad': lambda: dgrad(mode, 128, 128, C, Rc, C, 128, NONE),
        'run_step:fc2_dgrad': lambda: dgrad(mode, C, C, 512, L, 512, C, LK, 512),
        'run_step:fc1_dgrad': lambda: dgrad(mode, 512, 512, Hp, L, Hp, 512, NONE),
        'run_step:rnn_input_dgrad_ugrnn': lambda: dgrad(mode, gw['ugrnn'], gw['ugrnn'], C, L, C, gw['ugrnn'], TH, C),
        'run_step:rnn_input_dgrad_gru': lambda: dgrad(mode, gw['gru'], gw['gru'], C, L, C, gw['gru'], TH, C),
        'run_step:rnn_input_dgrad_lstm': lambda: dgrad(mode, gw['lstm'], gw['lstm'], C, L, C, gw['lstm'], TH, C),
        'run_step:rnn_layer2_dgrad': lambda: dgrad(mode, gw['ugrnn'], gw['ugrnn'], Hp, L, Hp, gw['ugrnn'], NONE),
        'run_step:car_layer2_candidates_dgrad': lambda: dgrad(mode, C, C, C, Rc, C, C, LK, C),
        'run_step:car_layer2_clicked_dgrad': lambda: dgrad(mode, C, C, C, L, C, C, LK, C),
        'run_step:car_layer1_dedup_dgrad': lambda: dgrad(mode, C, C, Fp, NB, Fp, C, NONE),
        'run_step:car_layer1_context_negatives_dgrad':
            lambda: dgrad(mode, C, C, Fp, L, Fp - c0, C, NONE, accumulate=True, dx_col0=c0),
        'run_step:car_layer1_dgrad': lambda: dgrad(mode, C, C, Fp, R, Fp, C, NONE),
        'run_step:scorer_m3_wgrad': lambda: wgrad(mode, 64, 32, 32, 64, 32, Rc),
        'run_step:scorer_m2_wgrad': lambda: wgrad(mode, 128, 64, 64, 128, 64, Rc),
        'run_step:scorer_m1_wgrad': lambda: wgrad(mode, C, 128, 128, C, 128, Rc),
        'run_step:car_layer2_candidates_wgrad': lambda: wgrad(mode, C, C, C, C, C, Rc),
        'run_step:car_layer2_candidates_wgrad_xt': lambda: wgrad_xt(mode, ldr, C, C, C, C, Rc),
        'run_step:fc2_wgrad': lambda: wgrad(mode, 512, C, C, 512, C, L),
        'run_step:fc1_wgrad': lambda: wgrad(mode, Hp, 512, 512, Hp, 512, L),
        'run_step:rnn_wx_wgrad_ugrnn': lambda: wgrad(mode, C, gw['ugrnn'], gw['ugrnn'], C, gw['ugrnn'], L),
        'run_step:rnn_wx_wgrad_gru': lambda: wgrad(mode, C, gw['gru'], gw['gru'], C, gw['gru'], L),
        'run_step:rnn_wx_wgrad_lstm': lambda: wgrad(mode, C, gw['lstm'], gw['lstm'], C, gw['lstm'], L),
        'run_step:rnn_wh_wgrad_ugrnn': lambda: wgrad(mode, Hp, gw['ugrnn'], gw['ugrnn'], Hp, gw['ugrnn'], L),
        'run_step:rnn_wh_wgrad_lstm': lambda: wgrad(mode, Hp, gw['lstm'], gw['lstm'], Hp, gw['lstm'], L),
        'run_step:gru_whg_wgrad': lambda: wgrad(mode, Hp, gw['gru'], 2 * Hp, Hp, 2 * Hp, L),
        'run_step:gru_whc_wgrad': lambda: wgrad(mode, Hp, gw['gru'], Hp, Hp, Hp, L, dy_col0=2 * Hp),
        'run_step:car_layer2_clicked_wgrad': lambda: wgrad(mode, C, C, C, C, C, L),
        'run_step:car_layer1_dedup_wgrad': lambda: wgrad(mode, Fp, C, C, Fp, C, NB),
        'run_step:car_layer1_context_negatives_wgrad': lambda: wgrad(mode, Fp, C, C, Fp - c0, C, L, x_col0=c0),
        'run_step:car_layer1_wgrad': lambda: wgrad(mode, Fp, C, C, Fp, C, R),
    }
    calls[site]()


@pytest.mark.parametrize('fwd_precision', [3, 4])
@pytest.mark.parametrize('problem', ['tiny', 'g1'])
@pytest.mark.parametrize('site', FWD_SITES)
def test_engine_forward_calls(site, problem, fwd_precision):
    """Each forward GEMM call form of engine.cu (Seq::fwd at its call sites in the step, the scorer and
    run_recommend) with that site's offsets, leading dimensions, majors, bias and activation, at fwd_precision 3 (with
    the weights' b_lo plane) and 4 (bf16x3 plane), dimensions from the 'tiny' and 'g1' problems.  Bar: the module's
    per-element bound.  Largest error/bar measured: 0.071 (g1 scorer M3, bf16x3)."""
    fwd_site(site, 2 if fwd_precision == 3 else 4, _dims(problem))


@pytest.mark.parametrize('bwd_precision', [1, 3])
@pytest.mark.parametrize('problem', ['tiny', 'g1'])
@pytest.mark.parametrize('site', BWD_SITES)
def test_engine_backward_calls(site, problem, bwd_precision):
    """Each backward GEMM call form of engine.cu (Seq::dgrad, Seq::wgrad, Seq::wgrad_xt at their call sites in the
    step) with that site's offsets, leading dimensions, majors, dact / accumulate and automatic split-K, at
    bwd_precision 1 and 3.  Bar: the module's per-element bound.  Largest error/bar measured: 0.46 (g1 scorer M3
    dgrad, single-pass TF32)."""
    bwd_site(site, 0 if bwd_precision == 1 else 1, _dims(problem))


# ------------------------------------------------------------------------------------------------------ edge shapes
MS = (1, 3, 63, 64, 65, 127)
NS = (1, 3, 4, 5, 31, 127)
KS = (1, 3, 4, 31, 33)
MAJORS = [(True, True), (True, False), (False, True), (False, False)]
INSTANTIATIONS = ([('plain', m, ak, bk) for m in (0, 1, 2) for ak, bk in MAJORS] +
                  [('plain', 4, True, True), ('plain', 4, False, True), ('trans_d', 0, False, True), ('trans_d', 1, False, True)])
EPIS = ['none', 'bias_leaky', 'bias_tanh', 'dact_leaky', 'dact_tanh', 'accumulate']


def _edge_cases():
    out = []
    for j, (kind, mode, ak, bk) in enumerate(INSTANTIATIONS):
        ms = MS + ((2, 66) if kind == 'trans_d' else ())          # TRANS_D: M = 1, 2, 3 (mod 4) tails
        for i, M in enumerate(ms):
            N = NS[(i + j) % len(NS)]
            K = KS[(i + 2 * j) % len(KS)]
            epi = 'accumulate' if (kind == 'trans_d' and i % 2) else ('none' if kind == 'trans_d' else EPIS[(i + j) % 6])
            if mode == 4 and epi == 'accumulate':
                epi = 'bias_leaky'
            out.append(pytest.param(kind, mode, ak, bk, M, N, K, epi,
                                    id='%s-m%d-%s%s-%dx%dx%d-%s' % (kind, mode, 'K' if ak else 'MN', 'K' if bk else 'MN',
                                                                   M, N, K, epi)))
    return out


@pytest.mark.parametrize('kind,mode,a_k,b_k,M,N,K,epi', _edge_cases())
def test_edge_shapes(kind, mode, a_k, b_k, M, N, K, epi):
    """A covering set of M in {1, 3, 63, 64, 65, 127}, N in {1, 3, 4, 5, 31, 127} and K in {1, 3, 4, 31, 33}: every
    kernel instantiation (4 majors x modes 0 / 1 / 2, bf16x3 with either A major, transposed D in modes 0 / 1, which
    also runs M = 2 and 66) meets every value of each.  Leading dimensions run 4-12 floats past the minimum, and bf16x3
    planes 8 or 64 columns past it, all NaN.  The epilogue rotates through none, bias + leaky, bias + tanh, dact leaky,
    dact tanh and accumulate (with the library's split).  Bar: the module's per-element bound.  Largest error/bar
    measured: 0.91 (single-pass TF32, 127 x 127 x 1, accumulate)."""
    kw = dict(bias=epi.startswith('bias'), act={'bias_leaky': 1, 'bias_tanh': 2}.get(epi, 0),
              dact={'dact_leaky': 1, 'dact_tanh': 2}.get(epi, 0), accumulate=epi == 'accumulate',
              split_k=0 if epi == 'accumulate' else 1)
    extra = 4 * (1 + (M + N + K) % 3)
    lda = _ld4(K if a_k else M, extra)
    ld_bf16 = (K + 31) // 32 * 64 + (8 if M % 2 else 64)
    run_case(M, N, K, mode=mode, a_k=a_k, b_k=b_k, lda=lda, trans_d=kind == 'trans_d', ld_bf16=ld_bf16,
             d_col0=4 * (1 + M % 2), **kw)


# -------------------------------------------------------------------------------------------------------- epilogues
EPILOGUE_CASES = [
    ('bias', dict(bias=True)),
    ('bias_leaky', dict(bias=True, act=1)),
    ('bias_tanh', dict(bias=True, act=2)),
    ('leaky', dict(act=1)),
    ('tanh', dict(act=2)),
    ('dact_leaky_signed_zeros', dict(dact=1, aux_special=[(0.0, 3), (-0.0, 5)])),
    ('dact_tanh_saturated', dict(dact=2, aux_special=[(1.0, 3), (-1.0, 5), (0.0, 7)])),
    ('accumulate', dict(accumulate=True, split_k=1)),
    ('accumulate_split', dict(accumulate=True, split_k=3)),
]


@pytest.mark.parametrize('N', [133, 70, 127])
@pytest.mark.parametrize('mode', [0, 1, 2, 4])
@pytest.mark.parametrize('name,epi', EPILOGUE_CASES, ids=[c[0] for c in EPILOGUE_CASES])
def test_epilogues_both_store_paths(name, epi, mode, N):
    """N = 1, 2, 3 (mod 4): each row's last 1-3 columns take epilogue_store4's scalar tail and the rest its float4
    path, in one launch.  Bias, leaky and tanh; leaky' with aux holding exact +0 and -0 (derivative 0.2f, not 1);
    tanh' with aux at +1, -1 and 0; accumulate without and with an explicit split.  The leaky reference uses the slope
    float32(0.2).  Bar: the module's per-element bound.  Largest error/bar measured: 0.26 (dact tanh, single-pass TF32,
    N = 133)."""
    if mode == 4 and epi.get('accumulate'):
        pytest.skip('bf16x3 does not accumulate (rejected by the argument checks)')
    run_case(150, N, 32 * 3 + 7, mode=mode, a_k=N != 70, b_k=N != 127 or mode == 4, scale=0.5, **epi)


# --------------------------------------------------------------------------------------------- split-K and the epilogue
def _plain_inputs(M, N, K, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    A, A64 = operand(M, K, _ld4(K), True, g, scale=0.1)
    B, B64 = operand(N, K, _ld4(K), True, g, scale=0.1)
    return g, A, A64, B, B64


@pytest.mark.parametrize('split_k', [2, 4])
@pytest.mark.parametrize('epi', ['bias', 'act_leaky', 'bias_tanh'])
def test_split_k_rejects_bias_and_act(epi, split_k):
    """An explicit split_k > 1 with a bias or an activation would apply them once per split: NarError, D untouched
    (bit for bit)."""
    M = N = 128
    K = 1024
    g, A, _, B, _ = _plain_inputs(M, N, K)
    kw = dict(bias=vec(N, g) if 'bias' in epi else None, act=2 if 'tanh' in epi else (1 if 'leaky' in epi else 0))
    dst = Dest(M, N, _ld4(N + 8), 4, torch.randn(M, N, device='cuda', generator=g))
    with pytest.raises(NarError):
        ops.gemm(A, B, dst.view, M, N, K, lda=A.stride(0), ldb=B.stride(0), ldd=dst.ld, precision=1, accumulate=True,
                 split_k=split_k, **kw)
    torch.cuda.synchronize()
    assert dst.untouched()


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('act', [1, 2])
def test_auto_split_with_bias_and_act(act, mode):
    """accumulate + split_k = 0 + bias + act at M = N = 128, K = 4096 (one tile, 128 k-tiles: the library's automatic
    split alone would pick 16): D = D0 + act(A B^T + b) within the bar, i.e. one split.  Bar: a quarter of the
    module's bound (with the whole bound the largest error/bar measured was 0.030); largest measured against it: 0.12."""
    run_case(128, 128, 4096, mode=mode, bias=True, act=act, accumulate=True, split_k=0, scale=0.05, tighten=0.25)


@pytest.mark.parametrize('field,value', [('act', 3), ('act', -1), ('act', 7), ('dact', 3), ('dact', -2)])
def test_act_outside_nar_act_rejected(field, value):
    """act / dact values outside nar_act (0, 1, 2) are rejected, not treated as none."""
    M = N = K = 64
    g, A, _, B, _ = _plain_inputs(M, N, K)
    aux = torch.randn(M, N, device='cuda', generator=g)
    dst = Dest(M, N, 72, 4)
    kw = {field: value}
    if field == 'dact':
        kw['aux'] = aux
    with pytest.raises(NarError):
        ops.gemm(A, B, dst.view, M, N, K, lda=A.stride(0), ldb=B.stride(0), ldd=dst.ld, precision=1, **kw)
    torch.cuda.synchronize()
    assert dst.untouched()


@pytest.mark.parametrize('a_k,b_k', [(True, True), (False, False)])
@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('k_tiles', [3, 5, 7])
def test_two_splits_bit_exact(k_tiles, mode, a_k, b_k):
    """split_k = 2 over an odd number of k-tiles splits them ceil / floor (the first split takes ceil(k_tiles / 2)).
    Onto a zero D, two red.adds give the same bits in either order, fl(p0 + p1), and each partial p_s is the same
    MMA sequence as a non-split GEMM over that split's k-range: the result must match those bits exactly.  It is also
    held to the module's bound: largest error/bar measured 0.27."""
    M, N, K = 200, 136, 32 * k_tiles
    g = torch.Generator(device='cuda').manual_seed(k_tiles)
    A, A64 = operand(M, K, _ld4(K if a_k else M, 4), a_k, g)
    B, B64 = operand(N, K, _ld4(K if b_k else N, 4), b_k, g)
    per = (k_tiles + 1) // 2
    kw = dict(a_kmajor=a_k, b_kmajor=b_k, lda=A.stride(0), ldb=B.stride(0), precision=PRECISION[mode])
    D = torch.zeros(M, N, device='cuda')
    ops.gemm(A, B, D, M, N, K, accumulate=True, split_k=2, **kw)
    parts = []
    for k0, k1 in ((0, 32 * per), (32 * per, K)):
        Ap = A[:, k0:k1] if a_k else A[k0:k1]
        Bp = B[:, k0:k1] if b_k else B[k0:k1]
        P = torch.full((M, N), float('nan'), device='cuda')
        ops.gemm(Ap, Bp, P, M, N, k1 - k0, **kw)
        parts.append(P)
    torch.cuda.synchronize()
    assert torch.equal((parts[0] + parts[1]).view(torch.int32), D.view(torch.int32))
    check(D, A64 @ B64.t(), c_mode(mode, K) * (A64.abs() @ B64.abs().t()) * 1.0 + CE * 2 * (A64.abs() @ B64.abs().t()))


# ---------------------------------------------------------------------------------------------- nar_pack_bf16x3
PACK_SENTINEL = 0x7FA5


def _pack_set(g, shapes, special=False):
    """Matrices W [K, N] (row stride N + 4 * (i % 3), NaN past N) and sentinel-filled plane storages with ld_out
    8 * (i % 3) past the minimum and two rows past N."""
    Ws, outs, stores, lds = [], [], [], []
    for i, (K, N) in enumerate(shapes):
        W = nan_view(K, N, N + 4 * (i % 3))
        x = torch.randn(K, N, device='cuda', generator=g) * (10.0 ** (i % 5 - 2))
        if special:
            vals = torch.tensor([0.0, -0.0, 1e-40, -3e-39, 1.4e-45, 1e38, -2.5e38, 3.0e-38, 1.0 + 2 ** -20, -65504.0],
                                device='cuda')
            x.view(-1)[:min(x.numel(), vals.numel())] = vals[:x.numel()]
        W.copy_(x)
        ld = (K + 31) // 32 * 64 + 8 * (i % 3)
        store = torch.full((N + 2, ld), PACK_SENTINEL, dtype=torch.int16, device='cuda')
        Ws.append(W)
        outs.append(store)
        stores.append(store)
        lds.append(ld)
    return Ws, outs, lds


def _pack_check(Ws, outs, shapes):
    for W, store, (K, N) in zip(Ws, outs, shapes):
        w = (K + 31) // 32 * 64
        assert torch.equal(store[:N, :w], plane_ref(W, K, N)), (K, N)
        assert bool((store[:N, w:] == PACK_SENTINEL).all()) and bool((store[N:] == PACK_SENTINEL).all()), (K, N)


def _shapes(n, seed):
    g = torch.Generator().manual_seed(seed)
    Ks = [1, 31, 33, 70, 100, 5, 64, 200]
    Ns = [1, 5, 33, 67, 130, 32, 3]
    return [(Ks[int(torch.randint(len(Ks), (1,), generator=g))], Ns[int(torch.randint(len(Ns), (1,), generator=g))])
            for _ in range(n)]


@pytest.mark.parametrize('n', [1, 3, 32])
def test_pack_bit_exact(n):
    """n matrices in one call, mixed K and N off the 32 grid, ldw > N (NaN past N): row n of each plane holds, per 32-k
    block, the 32 bf16(x) then the 32 bf16(x - bf16(x)), round-to-nearest-even as torch rounds; k >= K in the last block
    is 0; plane columns past ceil(K/32) 64 and rows past N keep their sentinel.  ±0, subnormal and large values."""
    g = torch.Generator(device='cuda').manual_seed(n)
    shapes = _shapes(n, n)
    Ws, outs, lds = _pack_set(g, shapes, special=True)
    assert pack(Ws, outs, [k for k, _ in shapes], [m for _, m in shapes], lds) == 0
    torch.cuda.synchronize()
    _pack_check(Ws, outs, shapes)


def test_pack_descriptor_cache():
    """The descriptor table is cached by contents: P1, P2, P1 on one scratch buffer are each packed correctly (P1's
    outputs are reset to the sentinel before it runs again)."""
    g = torch.Generator(device='cuda').manual_seed(5)
    scratch = torch.zeros(32 * 32, dtype=torch.uint8, device='cuda')
    s1, s2 = _shapes(3, 11), _shapes(5, 12)
    P1, P2 = _pack_set(g, s1), _pack_set(g, s2)
    for (Ws, outs, lds), shapes in ((P1, s1), (P2, s2), (P1, s1)):
        for o in outs:
            o.fill_(PACK_SENTINEL)
        assert pack(Ws, outs, [k for k, _ in shapes], [m for _, m in shapes], lds, scratch) == 0
        torch.cuda.synchronize()
        _pack_check(Ws, outs, shapes)


@pytest.mark.parametrize('case', ['n0', 'n33', 'k0', 'k_negative', 'ld_out_short'])
def test_pack_rejects(case):
    """n = 0, n = 33, K <= 0 and an ld_out shorter than ceil(K/32) 64: NAR_ERR_INVALID, nothing written."""
    g = torch.Generator(device='cuda').manual_seed(3)
    shapes = [(70, 33)] * (33 if case == 'n33' else 2)
    Ws, outs, lds = _pack_set(g, shapes)
    Ks = [k for k, _ in shapes]
    if case == 'k0':
        Ks[1] = 0
    if case == 'k_negative':
        Ks[1] = -5
    if case == 'ld_out_short':
        lds[1] = 3 * 64 - 8
    before = [o.clone() for o in outs]
    rc = pack(Ws, outs, Ks, [m for _, m in shapes], lds, n=0 if case == 'n0' else None)
    torch.cuda.synchronize()
    assert rc == NAR_ERR_INVALID
    assert all(torch.equal(a, b) for a, b in zip(outs, before))


# ---------------------------------------------------------------------------------------------- argument checks
class Call:
    """A valid nar_gemm_tf32(_dt) call that argument-check rows modify one field of."""

    def __init__(self, kind='plain'):
        g = torch.Generator(device='cuda').manual_seed(1)
        self.M, self.N, self.K = 64, 68, 70
        r = lambda *s: torch.randn(*s, device='cuda', generator=g)        # noqa: E731
        self.keep = []
        self.epi = GemmEpilogue()
        self.epi.precision, self.epi.split_k = 1, 1
        self.a_k, self.b_k, self.trans_d = 1, 1, False
        self.A, self.B = r(64, 72), r(68, 72)
        self.lda = self.ldb = 72
        self.dst = Dest(64, 68, 76, 4)
        self.D, self.ldd = self.dst.view.data_ptr(), 76
        self.t = {}
        if kind == 'trans_d':
            self.a_k, self.trans_d = 0, True
            self.A = r(70, 64)
            self.lda = 64
            self.dst = Dest(68, 64, 72, 4)
            self.D, self.ldd = self.dst.view.data_ptr(), 72
        elif kind == 'bf16':
            W = r(70, 68)
            self.t['plane'] = ops.pack_bf16x3(W, 70, 68)
            self.epi.precision, self.epi.b_bf16, self.epi.ld_bf16 = 4, self.t['plane'].data_ptr(), 192
        elif kind == 'scale':            # single-pass TF32 weight gradient with A scaled per (k group, m)
            self.a_k = self.b_k = 0
            self.A, self.B = r(70, 64), r(70, 68)
            self.lda, self.ldb = 64, 68
            self.t['scale'] = r(10, 64)
            self.epi.a_scale, self.epi.ld_a_scale, self.epi.a_scale_group = self.t['scale'].data_ptr(), 64, 7
        elif kind == 'pred':             # scorer-product backward: positions of 8 rows
            for k, s in (('pred', (8, 68)), ('d_pred', (8, 68)), ('aux', (64, 68))):
                self.t[k] = r(*s)
            self.epi.dact, self.epi.aux, self.epi.ld_aux = 2, self.t['aux'].data_ptr(), 68
            self.epi.pred, self.epi.d_pred, self.epi.ld_pred, self.epi.pred_group = \
                self.t['pred'].data_ptr(), self.t['d_pred'].data_ptr(), 68, 8
            self.dst = Dest(64, 68, 68, 0)
            self.D, self.ldd = self.dst.view.data_ptr(), 68
        elif kind == 'car':              # CAR layer-1 backward: 32 positions x (1 + 1) rows, no D
            for k in ('pp', 'pc', 'pi', 'dpp', 'dpc', 'dpi'):
                self.t[k] = torch.zeros(32, 68, device='cuda') if k.startswith('d') else r(32, 68)
                setattr(self.epi, 'car_' + k, self.t[k].data_ptr())
            self.t['pos_idx'] = torch.arange(32, dtype=torch.int32, device='cuda')
            self.t['neg_uidx'] = torch.zeros(32, dtype=torch.int32, device='cuda')
            self.epi.car_pos_idx, self.epi.car_neg_uidx = self.t['pos_idx'].data_ptr(), self.t['neg_uidx'].data_ptr()
            self.epi.ld_car, self.epi.car_k, self.epi.dact = 68, 1, 1
            self.D, self.ldd = None, 0

    def keep_plane(self):
        self.t['plane'] = ops.pack_bf16x3(torch.zeros(70, 68, device='cuda'), 70, 68)
        return self.t['plane']

    def __call__(self):
        fn = load().nar_gemm_tf32_dt if self.trans_d else load().nar_gemm_tf32
        from chameleon_recsys_b200.ops import context, _stream
        ctx = context()
        rc = fn(ctx.handle, self.M, self.N, self.K, C.c_void_p(self.A if isinstance(self.A, int) else self.A.data_ptr()),
                self.lda, self.a_k, C.c_void_p(self.B if isinstance(self.B, int) or self.B is None else self.B.data_ptr()),
                self.ldb, self.b_k, C.c_void_p(self.D), self.ldd, None if self.epi is None else C.byref(self.epi), _stream())
        torch.cuda.synchronize()
        return rc


def _addr(t, off=4):
    return t.data_ptr() + off


def _set(**kw):
    def f(c):
        for k, v in kw.items():
            if k.startswith('epi.'):
                v = v(c) if callable(v) else v
                setattr(c.epi, k[4:], v)
            else:
                setattr(c, k, v(c) if callable(v) else v)
    return f


ARG_ROWS = [
    # plain
    ('plain', 'A_null', _set(A=0)),
    ('plain', 'epi_null', _set(epi=None)),
    ('plain', 'B_null', _set(B=0)),
    ('plain', 'D_null', _set(D=None)),
    ('plain', 'ldd_not_multiple_of_4', _set(ldd=74)),
    ('plain', 'D_misaligned', _set(D=lambda c: c.D + 4)),
    ('plain', 'bias_misaligned', _set(**{'epi.bias': lambda c: _addr(c.A)})),
    ('plain', 'dact_without_aux', _set(**{'epi.dact': 1, 'epi.ld_aux': 68})),
    ('plain', 'ld_aux_not_multiple_of_4', _set(**{'epi.dact': 1, 'epi.aux': lambda c: c.B.data_ptr(), 'epi.ld_aux': 70})),
    ('plain', 'aux_misaligned', _set(**{'epi.dact': 1, 'epi.aux': lambda c: _addr(c.B), 'epi.ld_aux': 72})),
    ('plain', 'precision_0', _set(**{'epi.precision': 0})),
    ('plain', 'precision_2', _set(**{'epi.precision': 2})),
    ('plain', 'act_3', _set(**{'epi.act': 3})),
    ('plain', 'act_negative', _set(**{'epi.act': -1})),
    ('plain', 'dact_3', _set(**{'epi.dact': 3, 'epi.aux': lambda c: c.B.data_ptr(), 'epi.ld_aux': 72})),
    ('plain', 'split_without_accumulate', _set(**{'epi.split_k': 2})),
    ('plain', 'split_with_bias', _set(**{'epi.split_k': 2, 'epi.accumulate': 1, 'epi.bias': lambda c: c.A.data_ptr()})),
    ('plain', 'split_with_act', _set(**{'epi.split_k': 2, 'epi.accumulate': 1, 'epi.act': 1})),
    ('plain', 'A_misaligned', _set(A=lambda c: _addr(c.A))),
    ('plain', 'lda_not_multiple_of_4', _set(lda=70)),
    ('plain', 'lda_zero', _set(lda=0)),
    ('plain', 'B_misaligned', _set(B=lambda c: _addr(c.B))),
    ('plain', 'ldb_not_multiple_of_4', _set(ldb=71)),
    ('plain', 'b_lo_misaligned', _set(**{'epi.precision': 3, 'epi.b_lo': lambda c: _addr(c.B)})),
    ('plain', 'a_scale_group_without_a_scale', _set(**{'epi.a_scale_group': 4})),
    ('plain', 'ld_a_scale_without_a_scale', _set(**{'epi.ld_a_scale': 64})),
    ('plain', 'd_pred_without_pred', _set(**{'epi.d_pred': lambda c: c.A.data_ptr()})),
    ('plain', 'pred_group_without_pred', _set(**{'epi.pred_group': 8})),
    ('plain', 'ld_pred_without_pred', _set(**{'epi.ld_pred': 68})),
    ('plain', 'car_pc_without_car_pp', _set(**{'epi.car_pc': lambda c: c.A.data_ptr()})),
    ('plain', 'car_k_without_car_pp', _set(**{'epi.car_k': 1})),
    ('plain', 'ld_car_without_car_pp', _set(**{'epi.ld_car': 68})),
    # bf16x3
    ('bf16', 'no_plane', _set(**{'epi.b_bf16': None})),
    ('bf16', 'accumulate', _set(**{'epi.accumulate': 1})),
    ('bf16', 'plane_misaligned', _set(**{'epi.b_bf16': lambda c: c.epi.b_bf16 + 2})),
    ('bf16', 'ld_bf16_not_multiple_of_8', _set(**{'epi.ld_bf16': 196})),
    ('bf16', 'ld_bf16_short', _set(**{'epi.ld_bf16': 128})),
    # transposed D
    ('trans_d', 'b_lo', _set(**{'epi.precision': 3, 'epi.b_lo': lambda c: c.B.data_ptr()})),
    ('trans_d', 'bf16', _set(**{'epi.precision': 4, 'epi.b_bf16': lambda c: c.keep_plane().data_ptr(), 'epi.ld_bf16': 192})),
    ('trans_d', 'dact', _set(**{'epi.dact': 1, 'epi.aux': lambda c: c.B.data_ptr(), 'epi.ld_aux': 64})),
    ('trans_d', 'aux', _set(**{'epi.aux': lambda c: c.B.data_ptr(), 'epi.ld_aux': 64})),
    ('trans_d', 'a_scale', _set(**{'epi.a_scale': lambda c: c.A.data_ptr(), 'epi.ld_a_scale': 64, 'epi.a_scale_group': 1})),
    # A scale
    ('scale', 'b_kmajor', _set(b_k=1, B=lambda c: torch.zeros(68, 72, device='cuda'), ldb=72)),
    ('scale', 'precision_3', _set(**{'epi.precision': 3})),
    ('scale', 'group_0', _set(**{'epi.a_scale_group': 0})),
    ('scale', 'group_past_rows', _set(**{'epi.a_scale_group': 71})),
    ('scale', 'ld_a_scale_short', _set(**{'epi.ld_a_scale': 60})),
    ('scale', 'ld_a_scale_not_multiple_of_4', _set(**{'epi.ld_a_scale': 66})),
    ('scale', 'a_scale_misaligned', _set(**{'epi.a_scale': lambda c: c.epi.a_scale + 4})),
    ('scale', 'with_pred', _set(**{'epi.pred': lambda c: c.A.data_ptr(), 'epi.d_pred': lambda c: c.B.data_ptr(),
                                   'epi.ld_pred': 68, 'epi.pred_group': 7})),
    # scorer-product backward
    ('pred', 'precision_3', _set(**{'epi.precision': 3})),
    ('pred', 'a_mn_major', _set(a_k=0)),
    ('pred', 'b_mn_major', _set(b_k=0)),
    ('pred', 'accumulate', _set(**{'epi.accumulate': 1})),
    ('pred', 'bias', _set(**{'epi.bias': lambda c: c.A.data_ptr()})),
    ('pred', 'act', _set(**{'epi.act': 1})),
    ('pred', 'rows_not_whole_groups', _set(M=60)),
    ('pred', 'no_d_pred', _set(**{'epi.d_pred': None})),
    ('pred', 'no_aux', _set(**{'epi.aux': None})),
    ('pred', 'ld_aux_short', _set(**{'epi.ld_aux': 64})),
    ('pred', 'ld_pred_short', _set(**{'epi.ld_pred': 64})),
    # CAR layer-1 backward
    ('car', 'a_mn_major', _set(a_k=0)),
    ('car', 'b_mn_major', _set(b_k=0)),
    ('car', 'act', _set(**{'epi.act': 1})),
    ('car', 'a_scale', _set(**{'epi.a_scale': lambda c: c.A.data_ptr(), 'epi.ld_a_scale': 72, 'epi.a_scale_group': 1})),
    ('car', 'n_not_multiple_of_4', _set(N=66)),
    ('car', 'ld_car_short', _set(**{'epi.ld_car': 64})),
    ('car', 'ld_car_not_multiple_of_4', _set(**{'epi.ld_car': 70})),
    ('car', 'car_pc_misaligned', _set(**{'epi.car_pc': lambda c: c.epi.car_pc + 4})),
    ('car', 'no_pos_idx', _set(**{'epi.car_pos_idx': None})),
    ('car', 'no_neg_uidx', _set(**{'epi.car_neg_uidx': None})),
]


@pytest.mark.parametrize('kind', ['plain', 'bf16', 'trans_d', 'scale', 'pred', 'car'])
def test_argument_check_bases_run(kind):
    """Each base call the argument-check rows modify is itself valid (so each row violates exactly one restriction)."""
    c = Call(kind)
    assert c() == 0


@pytest.mark.parametrize('kind,name,mutate', ARG_ROWS, ids=['%s-%s' % (r[0], r[1]) for r in ARG_ROWS])
def test_argument_checks(kind, name, mutate):
    """One restriction of gemm()'s host checks violated: NAR_ERR_INVALID, and D (with its guards) bit-identical."""
    c = Call(kind)
    mutate(c)
    assert c() == NAR_ERR_INVALID
    assert c.dst.untouched()
    if kind == 'car':
        assert all(bool((c.t[k] == 0).all()) for k in ('dpp', 'dpc', 'dpi'))


@pytest.mark.parametrize('trans_d', [False, True])
@pytest.mark.parametrize('dim', ['M0', 'N0', 'K0', 'M-1', 'K-3'])
def test_empty_problem(dim, trans_d):
    """M, N or K <= 0: returns 0 and writes nothing."""
    c = Call('trans_d' if trans_d else 'plain')
    setattr(c, dim[0], int(dim[1:]))
    assert c() == 0
    assert c.dst.untouched()
