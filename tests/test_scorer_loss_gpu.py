"""The scorer tail, the ranking and the optimizer helpers against plain fp64 references written here (pytest -m gpu).

Every entry point of csrc/loss.cu and the helpers of csrc/misc.cu are called directly through ops: the MLP scorer's
last layer with its softmax cross-entropy and gradient, the cosine scorer, the novelty regulariser fused into both,
the evaluation ranking, the scorer product and its backward, Adam, the bias-gradient column sums, the l2 loss, the
activation backward, the transpose, the TF32 lo plane and in-place dropout.  The references follow oracle/nar_oracle.py
(scorer, loss and novelty: NarOracle.scorer / forward; ranking: rank_and_metrics) in torch / numpy float64.

Bars are first-order rounding-error bounds of the operation each kernel performs, in units of u = 2^-24 times the
absolute sum of the terms of the entry (the derivations are in the helpers and docstrings below).  Every accumulating
output starts from a nonzero prefill and must come back as prefill + contribution; every overwritten output starts as
NaN.  The softmax gradients and the losses are evaluated at the logits the kernel wrote (whose own bar is checked
first): a logit rounding of d moves every softmax probability by a factor e^d, which is a property of the logits, not
of the loss kernel.

The agreement measured on one H100 SXM (80 GB, 700 W), as the largest error / bar, is in each test's docstring.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

gpu = pytest.mark.gpu

U = 2.0 ** -24                      # unit roundoff of float32
TINY = 2.0 ** -126                  # smallest normal float32: results in the subnormal range carry this absolute error
COS_EPS = float(np.float32(1e-12))  # the kernel's norm floor, as a float32
ACT_NONE, ACT_LEAKY, ACT_TANH = 0, 1, 2

N_POS = [1, 3, 5, 486]
N_CAND = [1, 6, 32, 33, 51, 101, 501]
TAUS = [1.0, 0.1, 0.05]
WIDTHS = [32, 33, 64]


def _f32(x):
    return float(np.float32(x))


def _check(name, err, bar):
    """err <= bar everywhere; prints the largest ratio."""
    err = np.asarray(err, dtype=np.float64)
    bar = np.asarray(bar, dtype=np.float64)
    assert np.isfinite(err).all(), (name, 'non-finite error')
    r = err / np.maximum(bar, 1e-300)
    worst = int(np.argmax(r)) if r.size else 0
    assert (err <= bar).all(), (name, worst, float(err.reshape(-1)[worst]), float(bar.reshape(-1)[worst]))
    print('ratio %-40s %.3g' % (name, float(r.max()) if r.size else 0.0))


# ============================================================================================== fp64 references
def softmax_bound(lg):
    """Per position: a first-order bound R on the relative error of every probability the loss kernels form from the
    float32 logits lg [n_pos, n] (and, since R covers it, on the absolute error of their log-sum-exp).
    expf and logf are within 2 and 1 ulp (<= 4u, 2u); lg - max and lg - lse round once, which expf turns into a relative
    error |lg - max| u; the sum of exponentials is a per-lane chain of ceil(n/32) terms and a 5-level shuffle tree.
    With A = max |lg|: R = u (5A + 4 ln n + 2 ceil(n/32) + 24)."""
    n = lg.shape[1]
    A = np.abs(lg).max(axis=1)
    return U * (5.0 * A + 4.0 * math.log(max(n, 1)) + 2.0 * math.ceil(n / 32) + 24.0)


def novelty_of(pop_norm, cand_ids, log_base):
    """nov = -log_base(pop_norm[id]) (nar_model.py:531-544) in fp64 on the float32 popularity."""
    return -np.log(pop_norm.astype(np.float64)[cand_ids]) / math.log(log_base)


def loss_grad_ref(lg, inv_count, nov=None, factor=0.0):
    """fp64 softmax cross-entropy of candidate 0 plus the novelty regulariser, at the logits lg [n_pos, n]:
    xe_l = (lse_l - lg_l0) inv_count; nov_l = factor * sum_{j>=1} q_j nov_j * inv_count with q = softmax over the
    negatives only (nar_model.py:517); the training loss is xe - nov.
    Returns xe terms [n_pos], nov terms [n_pos], dL/dlg [n_pos, n], and |.| magnitudes of the gradient's terms."""
    lg = lg.astype(np.float64)
    n_pos, n = lg.shape
    mx = lg.max(axis=1, keepdims=True)
    e = np.exp(lg - mx)
    se = e.sum(axis=1, keepdims=True)
    p = e / se
    lse = (mx + np.log(se))[:, 0]
    xe = (lse - lg[:, 0]) * inv_count
    delta = np.zeros_like(lg)
    delta[:, 0] = 1.0
    g = (p - delta) * inv_count
    mag = (p + np.abs(p - delta)) * inv_count
    nov_terms = np.zeros(n_pos)
    if factor > 0.0 and n > 1:
        ln = lg[:, 1:]
        en = np.exp(ln - ln.max(axis=1, keepdims=True))
        q = en / en.sum(axis=1, keepdims=True)
        nv = nov[:, 1:]
        nbar = (q * nv).sum(axis=1, keepdims=True)
        nov_terms = factor * nbar[:, 0] * inv_count
        g[:, 1:] -= factor * inv_count * q * (nv - nbar)
        mag[:, 1:] += factor * inv_count * q * (np.abs(nv) + 2.0 * (q * np.abs(nv)).sum(axis=1, keepdims=True))
    return xe, nov_terms, g, mag


def cosine_ref(cand, pred, eps=COS_EPS):
    """F.normalize(cand) . F.normalize(pred) (nar_oracle.py scorer, ranking='cosine') in fp64, and the pieces of its
    gradient.  cand [n_pos, n, C], pred [n_pos, C]."""
    e = cand.astype(np.float64)
    p = pred.astype(np.float64)
    en_raw = np.sqrt((e * e).sum(-1))
    pn_raw = np.sqrt((p * p).sum(-1))
    en = np.maximum(en_raw, eps)
    pn = np.maximum(pn_raw, eps)
    dot = (e * p[:, None, :]).sum(-1)
    cos = dot / (en * pn[:, None])
    a = (np.abs(e) * np.abs(p[:, None, :])).sum(-1) / (en * pn[:, None])
    return dict(e=e, p=p, en=en, pn=pn, cos=cos, a=a, e_live=en_raw >= eps, p_live=pn_raw >= eps)


def cosine_grad_ref(ref, ds):
    """Hand-written gradient of sum_lj ds_lj cos_lj: d/de = p/(|e||p|) - cos e/|e|^2, d/dp = sum_j e/(|e||p|) -
    cos p/|p|^2, where a norm at the floor is a constant (no second term)."""
    e, p, en, pn, cos = ref['e'], ref['p'], ref['en'], ref['pn'], ref['cos']
    ce = np.where(ref['e_live'], cos, 0.0)
    cp = np.where(ref['p_live'][:, None], cos, 0.0)
    t1 = p[:, None, :] / (en * pn[:, None])[..., None]
    t2 = (ce / (en * en))[..., None] * e
    d_cand = ds[..., None] * (t1 - t2)
    u1 = e / (en * pn[:, None])[..., None]
    u2 = (cp / (pn * pn)[:, None])[..., None] * p[:, None, :]
    d_pred = (ds[..., None] * (u1 - u2)).sum(1)
    return d_cand, d_pred, (t1, t2, u1, u2)


def rank_ref(p):
    """tf.nn.top_k order of one row of probabilities: rank of i = #{j: p_j > p_i or (p_j == p_i and j < i)}."""
    p = np.asarray(p, dtype=np.float64)
    gt = p[None, :] > p[:, None]
    eq = (p[None, :] == p[:, None]) & (np.arange(p.size)[None, :] < np.arange(p.size)[:, None])
    return (gt | eq).sum(axis=1)


# ====================================================================== checks of the references (no GPU needed)
def test_loss_gradient_reference_matches_autograd():
    """loss_grad_ref's hand-written dL/dlogit (cross-entropy minus the novelty regulariser, negatives-only softmax)
    against torch.autograd of the same loss in fp64: within 1e-12 (measured on CPU: ~1e-17)."""
    rs = np.random.RandomState(0)
    for n_pos, n, factor in ((3, 1, 0.5), (4, 7, 2.0), (2, 40, 0.0), (5, 33, 0.5)):
        lg = rs.standard_normal((n_pos, n)) * 4.0
        nov = rs.uniform(0.0, 9.0, size=(n_pos, n))
        inv_count = 1.0 / 7.0
        xe, nv, g, _ = loss_grad_ref(lg, inv_count, nov, factor)
        t = torch.from_numpy(lg).requires_grad_(True)
        loss = -(torch.log_softmax(t, -1)[:, 0]).sum() * inv_count
        if factor > 0.0 and n > 1:
            q = torch.softmax(t[:, 1:], -1)
            loss = loss - factor * (q * torch.from_numpy(nov[:, 1:])).sum() * inv_count
        loss.backward()
        assert abs(float(loss.detach()) - (xe.sum() - nv.sum())) < 1e-12
        assert np.abs(t.grad.numpy() - g).max() < 1e-12


def test_cosine_gradient_reference_matches_autograd():
    """cosine_grad_ref's hand-written gradient against torch.autograd through F.normalize (eps on the norm), with a
    candidate row and a prediction row held at the norm floor: within 1e-12 relative to the largest entry (measured
    on CPU: ~1e-16)."""
    rs = np.random.RandomState(1)
    n_pos, n, C = 3, 5, 100
    cand = rs.standard_normal((n_pos, n, C))
    pred = rs.standard_normal((n_pos, C))
    cand[0, 2] *= 3e-13 / np.linalg.norm(cand[0, 2])
    pred[2] *= 5e-13 / np.linalg.norm(pred[2])
    ds = rs.standard_normal((n_pos, n))
    ref = cosine_ref(cand, pred)
    assert not ref['e_live'][0, 2] and not ref['p_live'][2]
    d_cand, d_pred, _ = cosine_grad_ref(ref, ds)
    e = torch.from_numpy(cand).requires_grad_(True)
    p = torch.from_numpy(pred).requires_grad_(True)
    cos = (torch.nn.functional.normalize(e, dim=-1, eps=COS_EPS) *
           torch.nn.functional.normalize(p, dim=-1, eps=COS_EPS)[:, None, :]).sum(-1)
    assert np.abs(cos.detach().numpy() - ref['cos']).max() < 1e-12
    (cos * torch.from_numpy(ds)).sum().backward()
    for got, want in ((d_cand, e.grad.numpy()), (d_pred, p.grad.numpy())):
        scale = np.abs(want).reshape(want.shape[0], -1).max(axis=1)
        err = np.abs(got - want).reshape(want.shape[0], -1).max(axis=1)
        assert (err <= 1e-12 * scale).all(), (err, scale)


def test_rank_reference_tie_rule_matches_stable_argsort():
    """rank_ref (higher probability first, equal probabilities in index order, as tf.nn.top_k) gives the same order as
    np.argsort(-p, kind='stable') on rows with exact ties, including ties with candidate 0."""
    rs = np.random.RandomState(2)
    for n in (1, 2, 7, 33, 100):
        for _ in range(20):
            p = rs.choice(rs.uniform(0.0, 1.0, size=max(1, n // 3)), size=n)
            order = np.argsort(-p, kind='stable')
            rank = rank_ref(p)
            assert np.array_equal(np.argsort(rank), order)
            assert np.array_equal(np.sort(rank), np.arange(n))


# ================================================================================================ GPU helpers
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


class _Nov:
    """Novelty regulariser inputs: a popularity table of V items (some at the floor 1/500, some 1) and candidate ids
    drawn with repeats."""

    def __init__(self, rs, n_rows, factor, log_base, V=50):
        pop = rs.uniform(1e-3, 1.0, size=V).astype(np.float32)
        pop[:5] = np.float32(1.0 / 500.0)
        pop[5] = 1.0
        self.pop = pop
        self.ids = rs.randint(0, V, size=n_rows).astype(np.int64)
        self.factor, self.log_base = factor, log_base
        self.prefill = np.float32(rs.uniform(-2, 2))
        self.pop_d, self.ids_d = _dev(pop), _dev(self.ids)
        self.loss_d = _dev(np.array([self.prefill], np.float32))

    def struct(self):
        from chameleon_recsys_b200 import ops
        return ops.novelty_reg(self.factor, self.log_base, self.pop_d, self.ids_d, self.loss_d)

    def nov(self, n_pos, n_cand):
        return novelty_of(self.pop, self.ids, self.log_base).reshape(n_pos, n_cand)


def _mlp_cases():
    cases = []
    for i, (n_pos, n_cand) in enumerate((a, b) for a in N_POS for b in N_CAND):
        tau = TAUS[i % 3]
        width = WIDTHS[(i // 3) % 3]
        ld_z = width + (5 if i % 2 else 0)
        ld_m4 = (4, 1, 7)[(i // 2) % 3]
        nov = (0.5, 2.0)[(i // 2) % 2] if i % 2 else 0.0
        log_base = (2.0, 10.0)[(i // 4) % 2]
        cases.append(pytest.param(n_pos, n_cand, tau, width, ld_z, ld_m4, nov, log_base, 1.0,
                                  id='p%d-c%d-t%g-w%d-ld%d-m%d-nov%g-b%g' % (n_pos, n_cand, tau, width, ld_z, ld_m4, nov, log_base)))
    # logits spread above 100 at tau 0.05: expf underflows for the far candidates
    cases.append(pytest.param(5, 101, 0.05, 33, 40, 4, 2.0, 10.0, 4.0, id='spread'))
    return cases


def _mlp_inputs(rs, n_pos, n_cand, width, ld_z, ld_m4, zscale):
    R = n_pos * n_cand
    pre = rs.standard_normal((R, width)) * zscale
    z = np.where(pre > 0, pre, 0.2 * pre).astype(np.float32)          # z3 is the leaky layer's OUTPUT
    z[rs.rand(R, width) < 0.05] = 0.0                                # exact zeros: leaky' is 0.2 there, as TF's
    zbuf = np.full((R, ld_z), np.nan, np.float32)
    zbuf[:, :width] = z
    m = (rs.standard_normal(width) * 0.3).astype(np.float32)
    mbuf = np.full(width * ld_m4, 7.5, np.float32)
    mbuf[::ld_m4] = m
    c4 = np.array([0.05, 3.0, 3.0, 3.0], np.float32)
    return z, zbuf, m, mbuf, c4


# ================================================================================================== MLP scorer
@gpu
@pytest.mark.parametrize('n_pos,n_cand,tau,width,ld_z,ld_m4,factor,log_base,zscale', _mlp_cases())
def test_score_softmax_ce(n_pos, n_cand, tau, width, ld_z, ld_m4, factor, log_base, zscale):
    """nar_score_softmax_ce: logits, the cross-entropy and the novelty loss, d_z3, d_m4 and d_c4 against fp64.
    Bars (R = softmax_bound of the position, mag = the absolute sum of the terms of the entry, prefill included):
    logits (width+1) u (sum|z m| + |b|) inv_temp (a width-long fma chain, then the multiply by inv_temp); d_z3
    (R + 3u) |ds| |m| leaky'; d_m4 (R + (n_cand + n_pos + 2) u) mag (a per-lane chain over the candidates, then an
    atomic per position); d_c4 (R + (ceil(n_cand/32) + n_pos + 7) u) mag; both losses sum_l R inv_count + (n_pos + 2)
    u mag; entries in the subnormal range get 2^-126 more.  d_z3 columns width..ld_z keep their prefill exactly; the
    other d_m4 entries of its ld_m4 stride too.  The logit bar has one rounding more than width u: the multiply by
    inv_temp.  The gradient bars replace a flat 1e-5 of the absolute sum by R, which is about 1e-5 at these logits but
    grows with |logit| (the kernel's exp arguments round in proportion to it) and with n_cand.
    Measured: logits 0.15, loss 0.10, loss_nov 0.018, d_z3 0.26, d_m4 0.034, d_c4 0.026 of their bars."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(n_pos * 1000 + n_cand)
    R = n_pos * n_cand
    z, zbuf, m, mbuf, c4 = _mlp_inputs(rs, n_pos, n_cand, width, ld_z, ld_m4, zscale)
    inv_t, inv_count = _f32(1.0 / tau), _f32(1.0 / max(1, n_pos - 1))
    nv = _Nov(rs, R, factor, log_base) if factor > 0 else None
    pre = dict(loss=np.float32(0.75), dc4=rs.uniform(-1, 1, 4).astype(np.float32),
               dm4=rs.uniform(-1, 1, width * ld_m4).astype(np.float32))
    dz_pre = np.full((R, ld_z), 12345.0, np.float32)
    dz_pre[:, :width] = np.nan
    logits, loss = _dev(np.full((n_pos, n_cand), np.nan, np.float32)), _dev(pre['loss'][None])
    dz, dm4, dc4 = _dev(dz_pre), _dev(pre['dm4']), _dev(pre['dc4'])
    ops.score_softmax_ce(_dev(zbuf), ld_z, width, _dev(mbuf), ld_m4, _dev(c4), n_pos, n_cand, inv_t, inv_count,
                         logits, loss, dz, dm4, dc4, nv.struct() if nv else None)
    lg_k = _host(logits)
    # logits
    z64, m64 = z.astype(np.float64), m.astype(np.float64)
    lg_ref = ((z64 @ m64 + float(c4[0])) * inv_t).reshape(n_pos, n_cand)
    lbar = (width + 1) * U * ((np.abs(z64) @ np.abs(m64)) + abs(float(c4[0]))).reshape(n_pos, n_cand) * inv_t
    _check('logits', np.abs(lg_k - lg_ref), lbar)
    if zscale > 1:
        assert (lg_k.max(1) - lg_k.min(1)).max() > 100.0
    # loss and gradient at the kernel's logits
    Rb = softmax_bound(lg_k)
    nov = nv.nov(n_pos, n_cand) if nv else None
    xe, nov_terms, g, gmag = loss_grad_ref(lg_k, inv_count, nov, factor)
    ds, dsmag = g.reshape(-1) * inv_t, gmag.reshape(-1) * inv_t
    Rr = np.repeat(Rb, n_cand)
    _check('loss', abs(float(_host(loss)[0]) - (float(pre['loss']) + xe.sum())),
           (Rb * inv_count).sum() + (n_pos + 2) * U * (abs(float(pre['loss'])) + np.abs(xe).sum()))
    if nv:
        got = float(_host(nv.loss_d)[0])
        _check('loss_nov', abs(got - (float(nv.prefill) + nov_terms.sum())),
               (Rb * factor * inv_count * np.abs(nov).max(1)).sum()
               + (n_pos + 2) * U * (abs(float(nv.prefill)) + np.abs(nov_terms).sum()))
        if n_cand == 1:
            assert got == nv.prefill
    slope = np.where(z > 0, 1.0, 0.2)
    dz_k = _host(dz)
    assert (dz_k[:, width:] == 12345.0).all(), 'd_z3 padding columns changed'
    want = ds[:, None] * m64[None, :] * slope
    _check('d_z3', np.abs(dz_k[:, :width] - want),
           (Rr + 3 * U)[:, None] * dsmag[:, None] * np.abs(m64)[None, :] * slope + TINY)
    dm4_k = _host(dm4)
    other = np.ones(width * ld_m4, bool)
    other[::ld_m4] = False
    assert (dm4_k[other] == pre['dm4'][other]).all(), 'd_m4 entries off the ld_m4 stride changed'
    pm = pre['dm4'][::ld_m4].astype(np.float64)
    _check('d_m4', np.abs(dm4_k[::ld_m4] - (pm + ds @ z64)),
           (Rb.max() + (n_cand + n_pos + 2) * U) * (np.abs(pm) + dsmag @ np.abs(z64)) + TINY)
    dc4_k = _host(dc4)
    assert (dc4_k[1:] == pre['dc4'][1:]).all()
    _check('d_c4', abs(float(dc4_k[0]) - (float(pre['dc4'][0]) + ds.sum())),
           (Rb.max() + (math.ceil(n_cand / 32) + n_pos + 7) * U) * (abs(float(pre['dc4'][0])) + dsmag.sum()) + TINY)


@gpu
@pytest.mark.parametrize('factor', [0.0, 2.0])
def test_score_softmax_ce_forward_only(factor):
    """The recommend call: d_z3 = None and inv_count = 0.  The logits match fp64 (bar of test_score_softmax_ce), and
    loss_sum, loss_nov, d_m4 and d_c4 keep their prefill bit for bit.
    Measured: logits at most 0.079 of the bar."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(5)
    n_pos, n_cand, width, ld_z, ld_m4 = 7, 51, 32, 32, 4
    z, zbuf, m, mbuf, c4 = _mlp_inputs(rs, n_pos, n_cand, width, ld_z, ld_m4, 1.0)
    nv = _Nov(rs, n_pos * n_cand, factor, 2.0) if factor > 0 else None
    logits = _dev(np.full((n_pos, n_cand), np.nan, np.float32))
    loss = _dev(np.array([0.75], np.float32))
    dm4, dc4 = _dev(np.full(width * ld_m4, 0.5, np.float32)), _dev(np.full(4, -0.25, np.float32))
    inv_t = _f32(1 / 0.1)
    ops.score_softmax_ce(_dev(zbuf), ld_z, width, _dev(mbuf), ld_m4, _dev(c4), n_pos, n_cand, inv_t, 0.0, logits, loss,
                         None, dm4, dc4, nv.struct() if nv else None)
    lg_k = _host(logits)
    z64, m64 = z.astype(np.float64), m.astype(np.float64)
    lg_ref = ((z64 @ m64 + float(c4[0])) * inv_t).reshape(n_pos, n_cand)
    lbar = (width + 1) * U * ((np.abs(z64) @ np.abs(m64)) + abs(float(c4[0]))).reshape(n_pos, n_cand) * inv_t
    _check('forward-only logits', np.abs(lg_k - lg_ref), lbar)
    assert _host(loss)[0] == np.float32(0.75)
    assert (_host(dm4) == 0.5).all() and (_host(dc4) == -0.25).all()
    if nv:
        assert _host(nv.loss_d)[0] == nv.prefill


@gpu
def test_score_softmax_ce_argument_checks():
    """d_z3 without d_m4 or d_c4, and a novelty log_base <= 1, raise NarError; cosine's d_cand without d_pred too."""
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import NarError
    rs = np.random.RandomState(6)
    z, zbuf, m, mbuf, c4 = _mlp_inputs(rs, 2, 3, 32, 32, 4, 1.0)
    Z, M, Cb = _dev(zbuf), _dev(mbuf), _dev(c4)
    lg, loss = torch.zeros(2, 3, device='cuda'), torch.zeros(1, device='cuda')
    dz, dm4, dc4 = torch.zeros(6, 32, device='cuda'), torch.zeros(128, device='cuda'), torch.zeros(4, device='cuda')
    for a, b in ((None, dc4), (dm4, None), (None, None)):
        with pytest.raises(NarError):
            ops.score_softmax_ce(Z, 32, 32, M, 4, Cb, 2, 3, 1.0, 0.5, lg, loss, dz, a, b)
    for base in (1.0, 0.5):
        nv = _Nov(rs, 6, 0.5, base)
        with pytest.raises(NarError):
            ops.score_softmax_ce(Z, 32, 32, M, 4, Cb, 2, 3, 1.0, 0.5, lg, loss, dz, dm4, dc4, nv.struct())
        with pytest.raises(NarError):
            ops.cosine_softmax_ce(torch.zeros(6, 4, device='cuda'), torch.ones(2, 4, device='cuda'), 2, 3, 4, 1.0, 0.5,
                                  lg, loss, None, None, nv.struct())
    with pytest.raises(NarError):
        ops.cosine_softmax_ce(torch.ones(6, 4, device='cuda'), torch.ones(2, 4, device='cuda'), 2, 3, 4, 1.0, 0.5, lg, loss,
                              torch.zeros(6, 4, device='cuda'), None)


# =============================================================================================== cosine scorer
def _cos_cases():
    cases = []
    for i, (C, n_cand) in enumerate((a, b) for a in (4, 64, 100, 1024) for b in N_CAND):
        n_pos = N_POS[i % 4]
        if n_pos * n_cand * C > (1 << 24):          # keep the candidate tensor under 64 MB
            n_pos = 3
        tau = TAUS[i % 3]
        nov = (0.5, 2.0)[(i // 2) % 2] if i % 2 else 0.0
        log_base = (2.0, 10.0)[(i // 4) % 2]
        cases.append(pytest.param(n_pos, n_cand, C, tau, nov, log_base,
                                  id='p%d-c%d-C%d-t%g-nov%g-b%g' % (n_pos, n_cand, C, tau, nov, log_base)))
    return cases


def _cos_inputs(rs, n_pos, n_cand, C):
    cand = (rs.standard_normal((n_pos, n_cand, C)) * 0.5).astype(np.float32)
    pred = (rs.standard_normal((n_pos, C)) * 0.5).astype(np.float32)
    j = min(2, n_cand - 1)
    cand[0, j] *= np.float32(3e-13 / np.linalg.norm(cand[0, j].astype(np.float64)))      # below the norm floor
    pred[n_pos - 1] *= np.float32(5e-13 / np.linalg.norm(pred[n_pos - 1].astype(np.float64)))
    return cand, pred


def _cos_bars(ref, C, n_cand, inv_t):
    """kc = ceil(C/32) + 5 bounds the dot products and squared norms (per-lane chains plus the shuffle tree; the
    prediction norm adds the 3-term sum over warps).  Logits: inv_temp u (kc a + (kc + 7) |cos|), a = sum|e p| / (|e||p|)."""
    kc = math.ceil(C / 32) + 5
    return kc, inv_t * U * (kc * ref['a'] + (kc + 7) * np.abs(ref['cos']))


@gpu
@pytest.mark.parametrize('n_pos,n_cand,C,tau,factor,log_base', _cos_cases())
def test_cosine_softmax_ce(n_pos, n_cand, C, tau, factor, log_base):
    """nar_cosine_softmax_ce against fp64 F.normalize (eps 1e-12 on the norm) with one candidate row and one prediction
    row below the floor: logits, both losses, d_cand and d_pred.
    Bars (R, mag as in test_score_softmax_ce; kc from _cos_bars): logits as _cos_bars; d_cand (R + (2 kc + 16) u) |ds|
    (|t1| + |t2|) with t1 = p / (|e||p|), t2 = a e / |e|^2 (0 for a floored norm); d_pred (R + (n_cand + 2 kc + 16) u)
    sum_j |ds| (|e| / (|e||p|) + a |p| / |p|^2); the losses as in test_score_softmax_ce.  A floored norm is a constant
    of F.normalize, so its row's gradient has no normalisation term.
    Measured: logits 0.22, loss 0.058, loss_nov 0.010, d_cand 0.11, d_pred 0.039 of their bars."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(n_pos * 7 + n_cand * 13 + C)
    cand, pred = _cos_inputs(rs, n_pos, n_cand, C)
    inv_t, inv_count = _f32(1.0 / tau), _f32(1.0 / (n_pos + 2))
    nv = _Nov(rs, n_pos * n_cand, factor, log_base) if factor > 0 else None
    logits = _dev(np.full((n_pos, n_cand), np.nan, np.float32))
    loss = _dev(np.array([-1.5], np.float32))
    dc = _dev(np.full((n_pos, n_cand, C), np.nan, np.float32))
    dp = _dev(np.full((n_pos, C), np.nan, np.float32))
    ops.cosine_softmax_ce(_dev(cand), _dev(pred), n_pos, n_cand, C, inv_t, inv_count, logits, loss, dc, dp,
                          nv.struct() if nv else None)
    lg_k = _host(logits)
    ref = cosine_ref(cand, pred)
    kc, lbar = _cos_bars(ref, C, n_cand, inv_t)
    _check('cos logits', np.abs(lg_k - ref['cos'] * inv_t), lbar)
    Rb = softmax_bound(lg_k)
    nov = nv.nov(n_pos, n_cand) if nv else None
    xe, nov_terms, g, gmag = loss_grad_ref(lg_k, inv_count, nov, factor)
    _check('cos loss', abs(float(_host(loss)[0]) - (-1.5 + xe.sum())),
           (Rb * inv_count).sum() + (n_pos + 2) * U * (1.5 + np.abs(xe).sum()))
    if nv:
        got = float(_host(nv.loss_d)[0])
        _check('cos loss_nov', abs(got - (float(nv.prefill) + nov_terms.sum())),
               (Rb * factor * inv_count * np.abs(nov).max(1)).sum()
               + (n_pos + 2) * U * (abs(float(nv.prefill)) + np.abs(nov_terms).sum()))
    ds, dsmag = g * inv_t, gmag * inv_t
    d_cand, d_pred, (t1, t2, u1, u2) = cosine_grad_ref(ref, ds)
    t2m = np.where(ref['e_live'], ref['a'] / (ref['en'] ** 2), 0.0)[..., None] * np.abs(ref['e'])
    u2m = np.where(ref['p_live'][:, None], ref['a'], 0.0)[..., None] * np.abs(ref['p'])[:, None, :] / (ref['pn'] ** 2)[:, None, None]
    _check('cos d_cand', np.abs(_host(dc) - d_cand),
           (Rb[:, None, None] + (2 * kc + 16) * U) * dsmag[..., None] * (np.abs(t1) + t2m) + TINY)
    _check('cos d_pred', np.abs(_host(dp) - d_pred),
           (Rb[:, None] + (n_cand + 2 * kc + 16) * U) * (dsmag[..., None] * (np.abs(u1) + u2m)).sum(1) + TINY)


@gpu
@pytest.mark.parametrize('factor', [0.0, 0.5])
def test_cosine_softmax_ce_forward_only(factor):
    """d_cand = d_pred = None and inv_count = 0: the logits match fp64 (bar of test_cosine_softmax_ce) and loss_sum and
    loss_nov keep their prefill bit for bit.  Measured: logits at most 0.060 of the bar."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(8)
    n_pos, n_cand, C = 5, 33, 100
    cand, pred = _cos_inputs(rs, n_pos, n_cand, C)
    nv = _Nov(rs, n_pos * n_cand, factor, 10.0) if factor > 0 else None
    logits = _dev(np.full((n_pos, n_cand), np.nan, np.float32))
    loss = _dev(np.array([0.75], np.float32))
    inv_t = _f32(1 / 0.05)
    ops.cosine_softmax_ce(_dev(cand), _dev(pred), n_pos, n_cand, C, inv_t, 0.0, logits, loss, None, None,
                          nv.struct() if nv else None)
    ref = cosine_ref(cand, pred)
    _, lbar = _cos_bars(ref, C, n_cand, inv_t)
    _check('cos forward-only logits', np.abs(_host(logits) - ref['cos'] * inv_t), lbar)
    assert _host(loss)[0] == np.float32(0.75)
    if nv:
        assert _host(nv.loss_d)[0] == nv.prefill


@gpu
@pytest.mark.parametrize('C', [64, 1024])
def test_cosine_shared_memory_limit(C):
    """The kernel stages C + 3 n_cand floats in 48 KB of shared memory: n_cand = (12288 - C) // 3 runs and matches
    fp64 (bars of test_cosine_softmax_ce), one more raises NarError.  The engine's cosine_chunk_cap (engine.cu) is
    this same n_cand: it splits recommend's candidate sets into chunks the kernel accepts.  The kernel's 32 bytes of
    static shared memory put the top of that range past the 48 KB a launch gets without opting in, so the wrapper opts
    in there (without it, a launch at the cap fails with cudaErrorInvalidValue).
    Measured: logits 0.14, d_cand 0.029 of their bars."""
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import NarError
    n_pos, n_cand = 3, (12288 - C) // 3
    rs = np.random.RandomState(C)
    cand, pred = _cos_inputs(rs, n_pos, n_cand, C)
    inv_t, inv_count = _f32(1 / 0.1), _f32(1 / 3)
    logits, loss = _dev(np.full((n_pos, n_cand), np.nan, np.float32)), torch.zeros(1, device='cuda')
    dc, dp = torch.full((n_pos, n_cand, C), float('nan'), device='cuda'), torch.full((n_pos, C), float('nan'), device='cuda')
    cand_d, pred_d = _dev(cand), _dev(pred)
    ops.cosine_softmax_ce(cand_d, pred_d, n_pos, n_cand, C, inv_t, inv_count, logits, loss, dc, dp)
    lg_k = _host(logits)
    ref = cosine_ref(cand, pred)
    kc, lbar = _cos_bars(ref, C, n_cand, inv_t)
    _check('cos limit logits', np.abs(lg_k - ref['cos'] * inv_t), lbar)
    Rb = softmax_bound(lg_k)
    _, _, g, gmag = loss_grad_ref(lg_k, inv_count)
    d_cand, d_pred, (t1, t2, u1, u2) = cosine_grad_ref(ref, g * inv_t)
    t2m = np.where(ref['e_live'], ref['a'] / (ref['en'] ** 2), 0.0)[..., None] * np.abs(ref['e'])
    _check('cos limit d_cand', np.abs(_host(dc) - d_cand),
           (Rb[:, None, None] + (2 * kc + 16) * U) * (gmag * inv_t)[..., None] * (np.abs(t1) + t2m) + TINY)
    big = torch.zeros(n_pos * (n_cand + 1), C, device='cuda')
    with pytest.raises(NarError):
        ops.cosine_softmax_ce(big, pred_d, n_pos, n_cand + 1, C, inv_t, inv_count, torch.zeros(n_pos, n_cand + 1, device='cuda'),
                              loss, None, None)


# ===================================================================================================== ranking
def _rank_inputs(rs, n_pos, n_cand):
    lg = (rs.standard_normal((n_pos, n_cand)) * 3.0).astype(np.float32)
    if n_cand > 1:
        for l in range(n_pos):
            k = min(n_cand, 2 + l % 4)
            grp = rs.choice(n_cand, size=k, replace=False)
            if l % 3 == 0:
                grp[0] = 0                                      # the positive among the tied candidates
            src = lg[l].max() if l % 2 == 0 else lg[l, rs.randint(n_cand)]
            lg[l, grp] = src                                    # bit-equal logits: bit-equal probabilities
    ids = (np.arange(n_pos * n_cand, dtype=np.int64) * 3 + 1).reshape(n_pos, n_cand)
    return lg, ids


def _prob_bound(lg, p64):
    """Relative bound on each probability of the ranking kernel, u (|lg - max| + E + ceil(n/32) + 14): lg - max rounds
    once (|lg - max| u after expf), expf is within 2 ulp, the sum of exponentials carries the p-weighted mean E of those
    errors plus its chain of ceil(n/32) terms and 5 shuffle levels, and the division rounds once."""
    x = np.abs(lg.astype(np.float64) - lg.max(axis=1, keepdims=True))
    E = (p64 * x).sum(axis=1, keepdims=True)
    return U * (x + E + math.ceil(lg.shape[1] / 32) + 14)


def _softmax64(lg):
    x = lg.astype(np.float64)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


def _check_ranking(lg, ids, pid, pp, name):
    """pid / pp: the kernel's pred_ids / pred_probs.  Returns the kernel's 0-based rank of candidate 0 per position."""
    n_pos, n_cand = lg.shape
    idx = (pid - 1) // 3 - np.arange(n_pos)[:, None] * n_cand            # candidate index at each rank
    assert ((pid - 1) % 3 == 0).all() and (np.sort(idx, axis=1) == np.arange(n_cand)).all(), (name, 'not a permutation')
    p64 = _softmax64(lg)
    bar = _prob_bound(lg, p64)
    rows = np.arange(n_pos)[:, None]
    _check(name + ' probs', np.abs(pp - p64[rows, idx]), bar[rows, idx] * p64[rows, idx] + TINY)
    assert (np.diff(pp, axis=1) <= 0).all(), (name, 'pred_probs increase')
    tie = pp[:, 1:] == pp[:, :-1]
    assert (idx[:, 1:][tie] > idx[:, :-1][tie]).all(), (name, 'equal probabilities out of index order')
    # against the fp64 stable order wherever neighbouring probabilities are further apart than their bars
    order = np.argsort(-p64, axis=1, kind='stable')
    ps, bs = p64[rows, order], (bar * p64)[rows, order]
    d = np.abs(np.diff(ps, axis=1))
    amb = (d > 0) & (d <= bs[:, 1:] + bs[:, :-1] + 2 * TINY)
    bad = np.zeros((n_pos, n_cand), bool)
    bad[:, 1:] |= amb
    bad[:, :-1] |= amb
    assert (idx[~bad] == order[~bad]).all(), (name, 'order differs from fp64')
    return np.argmax(idx == 0, axis=1)


@gpu
@pytest.mark.parametrize('n_pos', [1, 3, 4, 5, 1000])
@pytest.mark.parametrize('n_cand', [1, 2, 31, 32, 33, 51, 501, 3072])
def test_rank_candidates(n_cand, n_pos):
    """nar_rank_candidates at top_n in {0, 1, 10, n_cand, n_cand + 5}, with bit-equal logits tying candidates (the
    positive among them in every third row): pred_ids is a permutation in descending probability, equal probabilities in
    candidate-index order (tf.nn.top_k), the same order as the fp64 stable argsort wherever neighbouring probabilities
    differ by more than their bars, probabilities within _prob_bound of fp64 softmax; metrics (prefilled) add exactly the
    hits and the count, and the reciprocal ranks of the kernel's own ranks within 1e-12 relative.
    The probability bar is not a flat (n_cand + 4) u: that leaves out the rounding of lg - max, which expf turns into
    |lg - max| u, and it overstates the sum of exponentials, which runs in 32 lanes.
    Measured: probabilities at most 0.58 of the bar."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(n_cand * 10 + n_pos)
    lg, ids = _rank_inputs(rs, n_pos, n_cand)
    lg_d, ids_d = _dev(lg), _dev(ids)
    for top_n in sorted({0, 1, 10, n_cand, n_cand + 5}):
        pid = torch.full((n_pos, n_cand), -1, dtype=torch.int64, device='cuda')
        pp = torch.full((n_pos, n_cand), float('nan'), device='cuda')
        pre = np.array([3.0, 0.75, 11.0])
        met = _dev(pre)
        ops.rank_candidates(lg_d, ids_d, n_pos, n_cand, top_n, pid, pp, met)
        rank = _check_ranking(lg, ids, _host(pid), _host(pp), 'rank n_cand=%d top_n=%d' % (n_cand, top_n))
        got = _host(met)
        hit = rank < top_n
        assert got[0] == pre[0] + hit.sum() and got[2] == pre[2] + n_pos, (got, pre, hit.sum())
        want = pre[1] + (1.0 / (rank[hit] + 1.0)).sum()
        assert abs(got[1] - want) <= 1e-12 * want, (got[1], want)


@gpu
@pytest.mark.parametrize('missing', ['pred_ids', 'pred_probs', 'metrics'])
def test_rank_candidates_optional_outputs(missing):
    """Each of pred_ids, pred_probs and metrics may be None: the other two come out bit-identical to the full call."""
    from chameleon_recsys_b200 import ops
    n_pos, n_cand, top_n = 37, 51, 10
    lg, ids = _rank_inputs(np.random.RandomState(9), n_pos, n_cand)
    lg_d, ids_d = _dev(lg), _dev(ids)

    def run(skip):
        out = dict(pred_ids=torch.full((n_pos, n_cand), -1, dtype=torch.int64, device='cuda'),
                   pred_probs=torch.full((n_pos, n_cand), float('nan'), device='cuda'),
                   metrics=torch.tensor([1.0, 0.5, 2.0], dtype=torch.float64, device='cuda'))
        args = {k: (None if k == skip else v) for k, v in out.items()}
        ops.rank_candidates(lg_d, ids_d, n_pos, n_cand, top_n, args['pred_ids'], args['pred_probs'], args['metrics'])
        return {k: _host(v) for k, v in out.items()}

    full, part = run(None), run(missing)
    for k in full:
        if k == missing:
            untouched = {'pred_ids': -1, 'metrics': np.array([1.0, 0.5, 2.0])}.get(k)
            if untouched is not None:
                assert (part[k] == untouched).all()
            else:
                assert np.isnan(part[k]).all()
        else:
            assert np.array_equal(part[k], full[k]), k


@gpu
def test_rank_candidates_limits():
    """n_cand = 3072 fills the 48 KB of shared memory of four warps (covered in test_rank_candidates); 3073 raises
    NarError, as do n_cand = 0 and a negative top_n."""
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import NarError
    for n_cand, top_n in ((3073, 10), (0, 10), (5, -1)):
        lg = torch.zeros(2, max(1, n_cand), device='cuda')
        ids = torch.zeros(2, max(1, n_cand), dtype=torch.int64, device='cuda')
        with pytest.raises(NarError):
            ops.rank_candidates(lg, ids, 2, n_cand, top_n, None, None, None)


# ============================================================================================ scorer product
@gpu
@pytest.mark.parametrize('act', [ACT_NONE, ACT_LEAKY, ACT_TANH])
@pytest.mark.parametrize('n_cand', [1, 51])
@pytest.mark.parametrize('C', [4, 100, 1024])
def test_mul_pred(C, n_cand, act):
    """nar_mul_pred bit-exact against the numpy float32 product; nar_mul_pred_bwd with cand_act: d_cand within
    3u |d p| (1 + e^2) of fp64 (two or three roundings; tanh' = 1 - e^2 rounds e^2 and the difference), d_pred within
    n_cand u sum_j |d e| (an fma chain over the candidates).  Candidates are the activation's outputs: leaky ones with
    exact zeros and negatives, tanh ones up to +-(1 - 2^-24).
    Measured: d_cand at most 0.78, d_pred 1.0 of the bar (at n_cand = 1 d_pred is one rounding, which attains u)."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(C + n_cand + act)
    n_pos = 67
    x = rs.standard_normal((n_pos, n_cand, C)) * 2.0
    if act == ACT_TANH:
        e = np.tanh(x).astype(np.float32)
        e.reshape(-1)[::17] = np.float32(1 - 2 ** -24) * np.sign(e.reshape(-1)[::17])
    elif act == ACT_LEAKY:
        e = np.where(x > 0, x, 0.2 * x).astype(np.float32)
        e.reshape(-1)[::13] = 0.0
    else:
        e = x.astype(np.float32)
    p = rs.standard_normal((n_pos, C)).astype(np.float32)
    d = rs.standard_normal((n_pos, n_cand, C)).astype(np.float32)
    e_d, p_d = _dev(e), _dev(p)
    prod = torch.full((n_pos, n_cand, C), float('nan'), device='cuda')
    ops.mul_pred(e_d, p_d, n_pos, n_cand, C, prod)
    assert np.array_equal(_host(prod), e * p[:, None, :])
    dc = torch.full((n_pos, n_cand, C), float('nan'), device='cuda')
    dp = torch.full((n_pos, C), float('nan'), device='cuda')
    ops.mul_pred_bwd(_dev(d), e_d, p_d, n_pos, n_cand, C, dc, dp, act)
    e64, p64, d64 = e.astype(np.float64), p.astype(np.float64)[:, None, :], d.astype(np.float64)
    slope = {ACT_NONE: 1.0, ACT_LEAKY: np.where(e64 > 0, 1.0, 0.2), ACT_TANH: 1.0 - e64 * e64}[act]
    _check('mul_pred_bwd d_cand', np.abs(_host(dc) - d64 * p64 * slope), 3 * U * np.abs(d64 * p64) * (1 + e64 * e64) + TINY)
    _check('mul_pred_bwd d_pred', np.abs(_host(dp) - (d64 * e64).sum(1)), n_cand * U * np.abs(d64 * e64).sum(1) + TINY)


# ===================================================================================================== misc.cu
def _adam_cases():
    out = []
    for n in (4, 1020, 2 ** 21 + 12):
        for reg_end in sorted({0, 4, (n // 8) * 4, n}):
            out.append(pytest.param(n, reg_end, id='n%d-reg%d' % (n, reg_end)))
    return out


@gpu
@pytest.mark.parametrize('n,reg_end', _adam_cases())
def test_adam_tf(n, reg_end):
    """nar_adam_tf at steps 1, 2 and 1000 (beta1 0.8, beta2 0.99, eps 1e-6, reg_l2 0.3), each step from the kernel's
    previous state.  n = 2^21 + 12 takes more than one grid-stride pass (the grid holds 132 * 8 CTAs of 256 threads,
    4 floats each: 1,081,344 floats).  Bars: m within 3u (|b1 m| + |(1-b1) gg|) (fma of the regulariser, two products,
    the sum); v within 5u (|b2 v| + (1-b2) gg^2); w within 6u |dw| + u |w| of w - lr_t m' / (sqrt(v') + eps) at the
    kernel's own m', v' (lr_t cast to float, product, sqrt, + eps, division, final subtraction).  params_lo is bit-exact
    w' - (w' & 0xFFFFE000) of the new w'.  The m and v bars are in terms of the two terms rather than 2u of the result,
    which cancellation between them would break, and count the rounding of the regularised gradient; the w bar counts
    the cast of lr_t and the sqrt.  Measured: m 0.89, v 0.71, w 0.999 of the bar (the final subtraction, one rounding,
    attains u |w|)."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(n + reg_end)
    lr, b1, b2, eps, reg = _f32(0.01), _f32(0.8), _f32(0.99), _f32(1e-6), _f32(0.3)
    w = _dev(rs.standard_normal(n).astype(np.float32))
    m = _dev((rs.standard_normal(n) * 0.1).astype(np.float32))
    v = _dev(rs.uniform(0, 0.1, n).astype(np.float32))
    lo = torch.full((n,), float('nan'), device='cuda')
    r = np.where(np.arange(n) < reg_end, reg, 0.0)
    for step in (1, 2, 1000):
        g_h = (rs.standard_normal(n) * np.where(rs.rand(n) < 0.1, 1e-4, 1.0)).astype(np.float32)
        w0, m0, v0 = (_host(t).astype(np.float64) for t in (w, m, v))
        ops.adam_tf(w, _dev(g_h), m, v, n, reg_end, reg, lr, step, beta1=b1, beta2=b2, eps=eps, params_lo=lo)
        w1, m1, v1 = _host(w), _host(m), _host(v)
        gg = g_h.astype(np.float64) + r * w0
        _check('adam m', np.abs(m1 - (b1 * m0 + (1 - b1) * gg)), 3 * U * (np.abs(b1 * m0) + np.abs((1 - b1) * gg)))
        _check('adam v', np.abs(v1 - (b2 * v0 + (1 - b2) * gg * gg)), 5 * U * (np.abs(b2 * v0) + (1 - b2) * gg * gg))
        lr_t = lr * math.sqrt(1.0 - b2 ** step) / (1.0 - b1 ** step)           # the host's double, before the cast
        dw = lr_t * m1.astype(np.float64) / (np.sqrt(v1.astype(np.float64)) + eps)
        _check('adam w', np.abs(w1 - (w0 - dw)), 6 * U * np.abs(dw) + U * np.abs(w0))
        bits = w1.view(np.uint32) & np.uint32(0xFFFFE000)
        assert np.array_equal(_host(lo).view(np.uint32), (w1 - bits.view(np.float32)).view(np.uint32)), step


@gpu
def test_adam_tf_argument_checks():
    """n % 4, reg_end % 4 and step 0 raise NarError and leave the state untouched."""
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200._lib import NarError
    w = torch.ones(16, device='cuda')
    g, m, v = torch.ones_like(w), torch.zeros_like(w), torch.zeros_like(w)
    for n, reg_end, step in ((14, 0, 1), (16, 6, 1), (16, 0, 0)):
        with pytest.raises(NarError):
            ops.adam_tf(w, g, m, v, n, reg_end, 0.1, 0.01, step)
    assert (_host(w) == 1).all() and (_host(m) == 0).all()


@gpu
@pytest.mark.parametrize('cols', [1, 255, 257])
@pytest.mark.parametrize('rows', [1, 7, 64, 65, 261121])
def test_colsum_add(rows, cols):
    """nar_colsum_add onto a prefill, ld = cols + 3 (NaN in the padding, never read): within (ceil(rows/64) + 17) u
    (|prefill| + sum|x|) per column: 8 partial sums of at most 14 terms per 64-row slab, a 3-level combine, one atomic
    per slab.  rows 7, 65 and 261121 leave a tail that is not a multiple of 8.  Measured: at most 0.11 of the bar."""
    from chameleon_recsys_b200 import ops
    gen = torch.Generator(device='cuda').manual_seed(rows * 3 + cols)
    ld = cols + 3
    x = torch.randn(rows, ld, device='cuda', generator=gen)
    x[:, cols:] = float('nan')
    pre = torch.rand(cols + 2, device='cuda', generator=gen) * 4 - 2
    out = pre.clone()
    ops.colsum_add(x, rows, cols, ld, out)
    torch.cuda.synchronize()
    x64 = x[:, :cols].double()
    want = pre[:cols].double() + x64.sum(0)
    mag = pre[:cols].double().abs() + x64.abs().sum(0)
    assert torch.equal(out[cols:], pre[cols:])
    _check('colsum', (out[:cols].double() - want).abs().cpu().numpy(),
           ((math.ceil(rows / 64) + 17) * U * mag).cpu().numpy())


@gpu
@pytest.mark.parametrize('n', [1, 255, 270337, 4_000_000])
def test_l2_loss_add(n):
    """nar_l2_loss_add onto a prefill: scale/2 sum x^2 within (ceil(n/(256 G)) + G + 14) u (|prefill| + scale/2 sum x^2),
    G = min(ceil(n/1024), 1056) CTAs: a per-thread fma chain, the warp and CTA sums, the scale, one atomic per CTA.
    270337 is one element more than one grid-stride pass.  Measured: at most 0.036 of the bar."""
    from chameleon_recsys_b200 import ops
    gen = torch.Generator(device='cuda').manual_seed(n)
    x = torch.randn(n, device='cuda', generator=gen)
    scale = _f32(3e-3)
    out = torch.tensor([0.125], device='cuda')
    ops.l2_loss_add(x, n, scale, out)
    torch.cuda.synchronize()
    s = scale / 2 * float((x.double() ** 2).sum())
    G = min(math.ceil(n / 1024), 1056)
    _check('l2', abs(float(out[0]) - (0.125 + s)), (math.ceil(n / (256 * G)) + G + 14) * U * (0.125 + s))


@gpu
@pytest.mark.parametrize('inplace', [False, True])
@pytest.mark.parametrize('n', [1, 1001, 541235])
@pytest.mark.parametrize('act', [ACT_NONE, ACT_LEAKY, ACT_TANH])
def test_act_bwd(act, n, inplace):
    """nar_act_bwd, out of place and in place (dx is dy, as the engine calls it): none and leaky bit-exact against numpy
    float32 (y with exact zeros and negatives), tanh within 2^-23 |dy| (1 + y^2) of fp64 dy (1 - y^2), whether or not
    1 - y y is contracted.  Measured: tanh at most 0.72 of the bar."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(n + act)
    x = rs.standard_normal(n) * 2
    y = (np.tanh(x) if act == ACT_TANH else np.where(x > 0, x, 0.2 * x)).astype(np.float32)
    y[::7] = 0.0
    dy = rs.standard_normal(n).astype(np.float32)
    dy_d, y_d = _dev(dy), _dev(y)
    dx = dy_d if inplace else torch.full((n,), float('nan'), device='cuda')
    ops.act_bwd(dy_d, y_d, n, act, dx)
    got = _host(dx)
    if act == ACT_NONE:
        assert np.array_equal(got, dy)
    elif act == ACT_LEAKY:
        assert np.array_equal(got, dy * np.where(y > 0, np.float32(1), np.float32(0.2)))
    else:
        y64 = y.astype(np.float64)
        _check('act_bwd tanh', np.abs(got - dy * (1 - y64 * y64)), 2.0 ** -23 * np.abs(dy) * (1 + y64 * y64) + TINY)


_TSHAPES = [(hp, k * hp) for hp in (64, 256) for k in (2, 3, 4)] + [(1, 1), (33, 65), (100, 7)]


@gpu
@pytest.mark.parametrize('pad', [0, 3])
@pytest.mark.parametrize('rows,cols', _TSHAPES)
def test_transpose(rows, cols, pad):
    """nar_transpose_f32 bit-exact, with ld_src = cols + pad (NaN in the padding, never read) and ld_dst = rows + pad
    (a sentinel in the padding, never written).  The Hp x {2,3,4}Hp shapes are the recurrent weights BPTT reads."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(rows * 7 + cols)
    src = np.full((rows, cols + pad), np.nan, np.float32)
    src[:, :cols] = rs.standard_normal((rows, cols))
    dst = _dev(np.full((cols, rows + pad), -7.25, np.float32))
    ops.transpose(_dev(src), rows, cols, cols + pad, dst, rows + pad)
    got = _host(dst)
    assert np.array_equal(got[:, :rows].view(np.uint32), np.ascontiguousarray(src[:, :cols].T).view(np.uint32))
    assert (got[:, rows:] == -7.25).all()


@gpu
def test_tf32_lo():
    """nar_tf32_lo: x - (x & 0xFFFFE000) bit-exact, for normals of every sign and scale, subnormals and +-0, over more
    than one grid-stride pass."""
    from chameleon_recsys_b200 import ops
    rs = np.random.RandomState(10)
    n = 300_001
    x = (rs.standard_normal(n) * np.exp(rs.uniform(-30, 30, n))).astype(np.float32)
    x[:6] = [0.0, -0.0, 1e-40, -3e-42, np.float32(2 ** -149), -np.float32(1.1754942e-38)]
    x[6::5] = rs.randint(0, 2 ** 32, size=x[6::5].size, dtype=np.uint64).astype(np.uint32).view(np.float32)
    x[~np.isfinite(x)] = 1.5
    lo = torch.full((n,), float('nan'), device='cuda')
    ops.tf32_lo(_dev(x), n, lo)
    want = x - (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    assert np.array_equal(_host(lo).view(np.uint32), want.view(np.uint32))


@gpu
@pytest.mark.parametrize('inplace', [False, True])
def test_dropout_rows_inplace_and_padded(inplace):
    """nar_dropout_rows with ld > cols, out of place and in place (dst is src, as the engine calls it for the feature
    rows): the kept entries are bit-exact src * float32(1/keep_prob) where oracle/dropout_ref.py keeps them, the rest
    0, and the padding columns keep their sentinel."""
    from chameleon_recsys_b200 import ops
    from oracle import dropout_ref
    L, K, F, ld = 9, 4, 24, 28
    n_cand = K + 1
    R = L + L * n_cand
    rs = np.random.RandomState(11)
    pos = np.sort(rs.choice(5000, L, replace=False)).astype(np.int32) + (1 << 21)
    row_pos = np.concatenate([pos, np.repeat(pos, n_cand)]).astype(np.int32)
    x = np.full((R, ld), -3.5, np.float32)
    x[:, :F] = rs.standard_normal((R, F))
    src = _dev(x)
    dst = src if inplace else _dev(np.full((R, ld), -3.5, np.float32))
    seed, step, keep = 987654321012, 17, 0.8
    ops.dropout_rows(src, dst, R, F, ld, _dev(row_pos), L, n_cand, K, 0, keep, seed, step)
    got = _host(dst)
    mask = np.zeros((R, F), bool)
    mask[:L] = dropout_ref.keep_mask(seed, step, 1, pos.astype(np.int64), F, keep)
    cm = mask[L:].reshape(L, n_cand, F)
    cm[:, 0] = dropout_ref.keep_mask(seed, step, 2, pos.astype(np.int64), F, keep)
    cm[:, 1:] = dropout_ref.keep_mask(seed, step, 3, pos.astype(np.int64)[:, None] * K + np.arange(K), F, keep)
    want = np.where(mask, x[:, :F] * (np.float32(1) / np.float32(keep)), np.float32(0))
    assert np.array_equal(got[:, :F].view(np.uint32), want.view(np.uint32))
    assert (got[:, F:] == -3.5).all()
