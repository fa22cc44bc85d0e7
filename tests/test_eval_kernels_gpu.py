"""The kernels ``Estimator.evaluate`` and ``Estimator.predict`` run after scoring, driven directly through their C entry
points at every list length, position count and shared-memory edge: the list metrics and their reduction, the coverage
bitmaps (csrc/eval_metrics.cu), hit rate by session position (same file), the packed per-session logs
(csrc/session_logs.cu) and the top-n of a candidate set (csrc/recommend.cu).

References: oracle/eval_metrics_ref.list_values (fp64), oracle/by_position_ref.ByPositionRef, oracle/session_logs_ref
and oracle/recommend_ref.topn_rule, plus numpy restatements of the kernels' fixed summation orders and of the documented
packed-log layout.  Every output starts from a sentinel (a NaN bit pattern for floats, a fixed value for integers) and
carries guard space past its end that must keep it; rows a call must not write must keep it too.  Accumulators start
from a nonzero prefill and must grow by exactly the reference's amount.  A rejected call returns before any launch and
leaves every output untouched.

Errors were measured on one H100 80GB HBM3 at its 700 W power limit; each test's docstring states its bar and the worst
error seen there.  The list values came within 5.6e-16 relative of fp64 (bar 1e-12), the top-n probabilities within
9.5e-8 relative (bar 1e-6); everything else matched bit for bit.

list_kernel holds 1552 bytes of static shared memory, so a dynamic size in (48 KB - 1552, 48 KB] also needs the
opt-in.  Before nar_eval_metrics_lists raised the attribute whenever it launched, those sizes failed to launch with
cudaErrorInvalidValue (top_n 64 with acr_dim 58 .. 64, top_n 32 with acr_dim 308 .. 320, top_n 10 with acr_dim
1171 .. 1208).
"""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.by_position_ref import ByPositionRef
from oracle.eval_metrics_ref import list_values
from oracle.recommend_ref import topn_rule
from oracle.session_logs_ref import session_logs_ref

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAR_ERR_INVALID, NAR_ERR_UNSUPPORTED = -1, -2
NAN64 = 0x7FF8DEAD5A5A5A5A                  # quiet NaN with a payload: no kernel computes it
NAN32 = 0x7FC05A5A
SENT64 = 0x5A5A5A5A5A5A5A5A
SENT32 = 0x5A5A5A5A
GUARD = 64
LIST_BAR = 1e-12                            # per-query list values: relative to fp64
PROB_BAR = 1e-6                             # top-n probabilities: relative to fp64
N_VALUES = 6


def _i64(x):
    """a 64-bit mask as the signed int64 the C ABI takes"""
    return x - (1 << 64) if x >= 1 << 63 else x


def _torch():
    import torch
    return torch


def _lib():
    from chameleon_recsys_b200._lib import load
    return load()


def _s():
    return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


def _p(t, byte_offset=0):
    return C.c_void_p(0 if t is None else t.data_ptr() + byte_offset)


_ALIVE = []                                 # device inputs of the calls in flight: freed only after a synchronize


def _dev(a):
    t = _torch().from_numpy(np.ascontiguousarray(a)).cuda()
    _ALIVE.append(t)
    return t


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
    if _ALIVE:
        _torch().cuda.synchronize()
        _ALIVE.clear()


def _filled(n, bits, width):
    """n elements (+ GUARD) of ``bits`` as a device int tensor of ``width`` bits"""
    torch = _torch()
    dt = {64: torch.int64, 32: torch.int32}[width]
    t = torch.full((n + GUARD,), _i64(bits) if width == 64 else (bits - (1 << 32) if bits >= 1 << 31 else bits),
                   dtype=dt, device='cuda')
    _ALIVE.append(t)
    return t


def _bits(t, width):
    _torch().cuda.synchronize()
    return t.cpu().numpy().view(np.uint64 if width == 64 else np.uint32)


def _rel(got, want):
    """worst |got - want| / |want| (want == 0 demands got == 0 exactly: returns inf otherwise)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    nz = want != 0
    if np.any(got[~nz] != 0):
        return math.inf
    return float(np.max(np.abs(got[nz] - want[nz]) / np.abs(want[nz]), initial=0.0))


# ================================================================================================ list metrics
def _norms(acr, dim):
    x = np.asarray(acr, np.float64)[:, :dim]
    return np.sqrt((x * x).sum(axis=1))


def _lists_run(ids, labels, pop, acr, dim, top_n, rows, nq, length, q_stride, row_stride, label_stride=1,
               row_mask=None, neg_rel=0.1, bits0=None, seed=0):
    """One nar_eval_metrics_lists call on sentinel-filled outputs.  ``ids`` / ``labels`` flat int64 laid out with the
    given strides; ``acr`` [V, ld] float32.  -> (rc, per_query bits [rows * nq * 6 + GUARD], bitmaps [rows * words +
    GUARD], err, the bitmap prefill, the norms)."""
    torch = _torch()
    lib = _lib()
    V, ld = acr.shape
    words = (V + 31) // 32
    norms = _norms(acr, dim)
    mask = (1 << rows) - 1 if row_mask is None else row_mask
    if bits0 is None:
        rs = np.random.RandomState(seed + 99)
        bits0 = np.where(rs.rand(rows * words) < 0.2, rs.randint(0, 1 << 31, rows * words), 0).astype(np.uint32)
    pq = _filled(rows * nq * N_VALUES, NAN64, 64)
    bm = _dev(np.concatenate([bits0, np.full(GUARD, SENT32, np.uint32)]).view(np.int32))
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    rc = lib.nar_eval_metrics_lists(_p(_dev(ids)), row_stride, q_stride, rows, _i64(mask), nq, length, top_n,
                                    _p(_dev(labels)), label_stride, _p(_dev(pop)), _p(_dev(acr)), dim, ld,
                                    _p(_dev(norms)), V, neg_rel, _p(pq), _p(bm), _p(err), _s())
    return rc, _bits(pq, 64), _bits(bm, 32), int(_bits(err, 32)[0]), bits0, norms


def _lists_ref(ids, labels, pop, acr, dim, top_n, rows, nq, length, q_stride, row_stride, label_stride, row_mask,
               neg_rel, bits0, norms):
    """-> (values [rows, nq, 6] with nan where the sentinel must stay, bitmaps, err)"""
    V = acr.shape[0]
    words = (V + 31) // 32
    m = min(top_n, length)
    x = np.asarray(acr, np.float64)[:, :dim]
    want = np.full((rows, nq, N_VALUES), np.nan)
    bits = bits0.copy()
    err = 0
    for r in range(rows):
        if not (row_mask >> r) & 1:
            continue
        for q in range(nq):
            label = int(labels[q * label_stride])
            if label == 0:
                want[r, q] = 0.0
                continue
            row = ids[r * row_stride + q * q_stride: r * row_stride + q * q_stride + length]
            if not 0 <= label < V or np.any((row[:m] < 0) | (row[:m] >= V)):
                err = 1
                want[r, q] = 0.0
                continue
            want[r, q, :5] = list_values(row, label, top_n, pop, x, norms, neg_rel)
            want[r, q, 5] = 1.0
            for i in row[:m].tolist():
                bits[r * words + (i >> 5)] |= np.uint32(1 << (i & 31))
    return want, bits, err


def _lists_check(args, kw=None, expect_err=None):
    """Run one call and compare everything with the reference; -> worst relative error of the per-query values."""
    kw = dict(kw or {})
    rc, pq, bm, err, bits0, norms = _lists_run(*args, **kw)
    assert rc == 0, rc
    ids, labels, pop, acr, dim, top_n, rows, nq, length, q_stride, row_stride = args
    mask = kw.get('row_mask', (1 << rows) - 1)
    want, wbits, werr = _lists_ref(ids, labels, pop, acr, dim, top_n, rows, nq, length, q_stride, row_stride,
                                   kw.get('label_stride', 1), mask, kw.get('neg_rel', 0.1), bits0, norms)
    n = rows * nq * N_VALUES
    assert np.all(pq[n:] == NAN64), 'per_query guard written'
    assert np.array_equal(bm, np.concatenate([wbits, np.full(GUARD, SENT32, np.uint32)])), 'bitmaps'
    assert err == werr if expect_err is None else err == expect_err
    got = pq[:n].view(np.float64).reshape(rows, nq, N_VALUES)
    keep = np.isnan(want[:, :, 0])
    assert np.all(pq[:n].reshape(rows, nq, N_VALUES)[keep] == NAN64), 'a masked row was written'
    zero = ~keep & (want[:, :, 5] == 0)
    assert np.all(pq[:n].reshape(rows, nq, N_VALUES)[zero] == 0), 'a label-0 or bad query is not six zeros'
    live = ~keep & (want[:, :, 5] == 1)
    worst = _rel(got[live], want[live]) if live.any() else 0.0
    assert worst <= LIST_BAR, worst
    return worst


def _list_problem(rs, V, dim, ld, rows, nq, length, q_stride, row_stride, label_stride=1, zero_frac=0.2, int_acr=False):
    acr = np.zeros((V, ld), np.float32)
    acr[:, :dim] = rs.randint(-3, 4, size=(V, dim)) if int_acr else rs.randn(V, dim)
    pop = rs.uniform(1e-4, 1.0, V).astype(np.float32)
    ids = np.full(max(row_stride * rows, 1), -77, np.int64)         # stride gaps hold ids no call may read
    for r in range(rows):
        for q in range(nq):
            o = r * row_stride + q * q_stride
            ids[o:o + length] = rs.randint(0, V, length)
    labels = np.full(max(nq * label_stride, 1), -55, np.int64)
    lab = rs.randint(1, V, nq)
    lab[rs.rand(nq) < zero_frac] = 0
    # plant the label inside many lists (row 0's layout; other rows draw their own ids)
    for q in range(nq):
        if lab[q] and rs.rand() < 0.7:
            for r in range(rows):
                o = r * row_stride + q * q_stride
                ids[o + rs.randint(0, length)] = lab[q]
    labels[::label_stride][:nq] = lab
    return ids, labels, pop, acr


M_CASES = [(m, rel) for m in (2, 3, 31, 32, 33, 63, 64) for rel in ('len<top_n', 'len=top_n', 'len>top_n')]


@gpu
@pytest.mark.parametrize('m,rel', M_CASES)
def test_lists_every_list_length(m, rel):
    """Per-query values of every query, m = min(top_n, len) = 2 .. 64 with len below, at and above top_n, two rows.
    Bar: 1e-12 relative to fp64 (the kernel's fp64 sums differ from the oracle's only in order, FMA contraction and
    log2); worst on the H100 5.6e-16."""
    rs = np.random.RandomState(m * 3 + len(rel))
    top_n, length = {'len<top_n': (m + 3, m), 'len=top_n': (m, m), 'len>top_n': (m, m + 5)}[rel]
    nq, rows, V, dim = 5, 2, 300, 24
    # integer ACR rows at m <= 3: a list of one repeated id has distance 0 on both sides, not 0 against 1e-16
    ids, labels, pop, acr = _list_problem(rs, V, dim, dim, rows, nq, length, length, nq * length, int_acr=m <= 3)
    worst = _lists_check((ids, labels, pop, acr, dim, top_n, rows, nq, length, length, nq * length), dict(seed=m))
    print('lists m=%d %s worst rel %.3g' % (m, rel, worst))


@gpu
def test_lists_rejected_calls_leave_outputs_untouched():
    """m < 2 (top_n 1, or len 1) is NAR_ERR_INVALID, m = 65 and shared memory above 200 KB NAR_ERR_UNSUPPORTED, and so
    are bad strides, row counts and relevance; none of them writes an output or err."""
    rs = np.random.RandomState(5)
    V, dim, nq = 100, 8, 3
    ids, labels, pop, acr = _list_problem(rs, V, dim, dim, 1, nq, 70, 70, nq * 70)
    base = (ids, labels, pop, acr, dim)
    cases = [
        (dict(top_n=1, length=5), NAR_ERR_INVALID),
        (dict(top_n=5, length=1), NAR_ERR_INVALID),
        (dict(top_n=65, length=70), NAR_ERR_UNSUPPORTED),
        (dict(top_n=64, length=70, q_stride=69), NAR_ERR_INVALID),
        (dict(top_n=8, length=10, rows=64), NAR_ERR_INVALID),
        (dict(top_n=8, length=10, rows=0), NAR_ERR_INVALID),
        (dict(top_n=8, length=10, label_stride=0), NAR_ERR_INVALID),
        (dict(top_n=8, length=10, neg_rel=0.0), NAR_ERR_INVALID),
        (dict(top_n=8, length=10, neg_rel=float('nan')), NAR_ERR_INVALID),
    ]
    for kw, want in cases:
        top_n, length = kw['top_n'], kw['length']
        rows = kw.get('rows', 1)
        rc, pq, bm, err, bits0, _ = _lists_run(ids, labels, pop, acr, dim, top_n, rows, nq, length,
                                               kw.get('q_stride', 70), nq * 70, label_stride=kw.get('label_stride', 1),
                                               row_mask=1, neg_rel=kw.get('neg_rel', 0.1))
        assert rc == want, (kw, rc)
        assert np.all(pq == NAN64) and err == 0, kw
        assert np.array_equal(bm[:bits0.size], bits0) and np.all(bm[bits0.size:] == SENT32), kw
    # acr_ld < acr_dim, and 8 m^2 + 4 m dim = 200 KB + 256 (m 64, dim 673)
    for dim_, ld_, want in ((9, 8, NAR_ERR_INVALID), (673, 673, NAR_ERR_UNSUPPORTED)):
        a = np.zeros((V, ld_), np.float32)
        rc = _lib().nar_eval_metrics_lists(_p(_dev(ids)), nq * 70, 70, 1, 1, nq, 70, 64, _p(_dev(labels)), 1,
                                           _p(_dev(pop)), _p(_dev(a)), dim_, ld_, _p(_dev(np.ones(V))), V, 0.1,
                                           _p(_filled(nq * 6, NAN64, 64)), _p(_filled(4, 0, 32)),
                                           _p(_filled(1, 0, 32)), _s())
        assert rc == want, (dim_, ld_, rc)


# shared-memory sizes 8 m^2 + 4 m dim around the 48 KB a launch gets without opting in.  list_kernel holds 1552 bytes of
# static shared memory (s_id, s_er, s_err, s_occ, s_bad), so dynamic sizes in (48 KB - 1552, 48 KB] need the opt-in too.
# Cases up to 48 KB come first: an earlier opt-in would leave the attribute raised for them.
SMEM_CASES = [(64, 57), (50, 137), (50, 138), (10, 1170), (32, 307),     # <= 48 KB - 1552
              (64, 58), (32, 308), (50, 139), (10, 1171),                # just above 48 KB - 1552
              (10, 1208), (32, 320), (64, 64),                           # up to exactly 48 KB
              (64, 65), (10, 1209),                                      # just above 48 KB
              (64, 250),                                                 # 96.8 KB (the G1 ACR width)
              (64, 672),                                                 # exactly 200 KB
              (64, 250), (64, 65)]                                       # smaller calls after the largest


def smem_cases():
    """Run SMEM_CASES in order in this process; -> [(m, dim, smem, rc, worst)] and the rc of m 64 x dim 673."""
    out = []
    for i, (m, dim) in enumerate(SMEM_CASES):
        rs = np.random.RandomState(1000 + i)
        V, nq, length = 160, 3, m + 2
        ids, labels, pop, acr = _list_problem(rs, V, dim, dim, 1, nq, length, length, nq * length, zero_frac=0.0)
        args = (ids, labels, pop, acr, dim, m, 1, nq, length, length, nq * length)
        try:
            worst = _lists_check(args, dict(seed=i))
            rc = 0
        except AssertionError as e:
            rc, worst = _lists_run(*args)[0], str(e)
        out.append((m, dim, 8 * m * m + 4 * m * dim, rc, worst))
    rs = np.random.RandomState(7)
    ids, labels, pop, acr = _list_problem(rs, 50, 673, 673, 1, 2, 64, 64, 128)
    rc = _lists_run(ids, labels, pop, acr, 673, 64, 1, 2, 64, 64, 128)[0]
    return out, rc


@gpu
def test_lists_shared_memory_edges_in_a_fresh_process():
    """Every size around 48 KB - 1552 and 48 KB, 96.8 KB and exactly 200 KB launches and matches fp64 (bar 1e-12
    relative, worst on the H100 4.8e-16), including a smaller size after the largest; 200 KB + 256 bytes is
    NAR_ERR_UNSUPPORTED.  A fresh interpreter runs them so that no earlier call in the session has raised the kernel's
    shared-memory attribute."""
    code = ('import json, sys, importlib.util; sys.path.insert(0, %r); '
            'spec = importlib.util.spec_from_file_location("eval_kernels", %r); '
            'mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod); '
            'print("RESULT " + json.dumps(mod.smem_cases()))') % (ROOT, os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-s', '-c', code], capture_output=True, text=True, cwd=ROOT, env=env,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith('RESULT ')][-1]
    cases, rc_over = json.loads(line[len('RESULT '):])
    for m, dim, smem, rc, worst in cases:
        print('lists smem m=%d dim=%d %d B: rc %d worst %s' % (m, dim, smem, rc, worst))
    bad = [(m, dim, smem, rc, worst) for m, dim, smem, rc, worst in cases if rc != 0 or not worst <= LIST_BAR]
    assert not bad, bad
    assert rc_over == NAR_ERR_UNSUPPORTED


ROW_CASES = [(1, 1 | (1 << 40)), (2, 0b10 | (1 << 10)), (63, (1 << 0) | (1 << 5) | (1 << 33) | (1 << 62) | (1 << 63))]


@gpu
@pytest.mark.parametrize('rows,mask', ROW_CASES)
def test_lists_rows_masks_and_strides(rows, mask):
    """Rows 1, 2 and 63 with sparse masks (bit 62 included; bits >= rows ignored), q_stride > len, a row stride with a
    gap, label_stride 3 and acr_ld > acr_dim.  Bar 1e-12 relative (worst on the H100 below 6e-16); unmasked rows keep
    the sentinel and their bitmaps the prefill."""
    rs = np.random.RandomState(rows)
    V, dim, ld, nq, length, top_n = 200, 12, 17, 4, 9, 6
    q_stride, row_stride, ls = length + 3, nq * (length + 3) + 5, 3
    ids, labels, pop, acr = _list_problem(rs, V, dim, ld, rows, nq, length, q_stride, row_stride, label_stride=ls)
    worst = _lists_check((ids, labels, pop, acr, dim, top_n, rows, nq, length, q_stride, row_stride),
                         dict(label_stride=ls, row_mask=mask, seed=rows))
    print('lists rows=%d worst rel %.3g' % (rows, worst))
    # a mask with no bit below rows: nothing is written
    rc, pq, bm, err, bits0, _ = _lists_run(ids, labels, pop, acr, dim, top_n, rows, nq, length, q_stride, row_stride,
                                           label_stride=ls, row_mask=1 << 63 if rows == 63 else 1 << rows)
    assert rc == 0 and np.all(pq == NAN64) and err == 0 and np.array_equal(bm[:bits0.size], bits0)


@gpu
@pytest.mark.parametrize('nq', [1, 66000])
def test_lists_one_query_and_a_grid_past_65535(nq):
    """nq = 1, and nq = 66 000 (a grid x dimension above 65 535) at m = 2.  Bar 1e-12 relative (worst on the H100
    below 6e-16)."""
    rs = np.random.RandomState(nq % 97)
    V, dim, length, top_n = 500, 5, 3, 2
    ids, labels, pop, acr = _list_problem(rs, V, dim, dim, 1, nq, length, length, nq * length, int_acr=True)
    worst = _lists_check((ids, labels, pop, acr, dim, top_n, 1, nq, length, length, nq * length), dict(seed=nq))
    print('lists nq=%d worst rel %.3g' % (nq, worst))


def _value_table(dim):
    """V = 64 integer ACR rows of width ``dim`` (exact dots and norms in any order): id 1 all zero, ids 2 and 3 identical
    (their cosine rounds above 1 and is clipped), id 4 = -id 2 (cosine below -1, distance 1)."""
    rs = np.random.RandomState(dim)
    V = 64
    acr = rs.randint(-3, 4, size=(V, dim)).astype(np.float32)
    acr[1] = 0.0
    acr[2] = 0.0
    acr[2, :min(3, dim)] = 1.0                       # dot 3 over norm product 2.9999999999999996
    acr[3] = acr[2]
    acr[4] = -acr[2]
    pop = rs.uniform(0.01, 0.9, V).astype(np.float32)
    pop[5] = 1.0                                     # -log2(1) = 0
    pop[6] = np.float32(1.0 / 2500)                  # the empty-buffer floor 1 / recent_clicks_for_normalization
    pop[7] = np.finfo(np.float32).tiny
    return acr, pop


def _value_lists():
    """(list of 12 ids, label) per query at top_n 8: the label at rank 0, at rank m - 1 and only past m; repeated inside
    and beyond m; more occurrences than m (the ideal DCG is clamped to m); id 0 in the list; the zero, identical and
    antiparallel rows with pop 1, the floor and FLT_MIN; a label-0 query; a bad label; a bad id inside m."""
    L = []
    L.append(([9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20], 9))
    L.append(([10, 11, 12, 13, 14, 15, 16, 9, 17, 18, 19, 20], 9))
    L.append(([10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 9, 20], 9))
    L.append(([10, 9, 11, 9, 12, 13, 14, 15, 16, 9, 17, 18], 9))
    L.append(([9, 9, 10, 9, 9, 9, 11, 9, 9, 9, 9, 9], 9))
    L.append(([0, 10, 0, 11, 12, 0, 13, 14, 15, 0, 16, 17], 12))
    L.append(([1, 2, 3, 4, 5, 6, 7, 2, 1, 3, 4, 5], 3))
    L.append(([2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3], 2))
    L.append(([21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32], 0))
    L.append(([40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51], 64))
    L.append(([52, 53, -1, 54, 55, 56, 57, 58, 59, 60, 61, 62], 52))
    L.append(([33, 34, 35, 36, 37, 38, 39, 33, 34, 35, 36, 37], 39))
    return L


@gpu
@pytest.mark.parametrize('neg_rel', [1e-6, 0.1, 1.0])
@pytest.mark.parametrize('dim', [1, 5])
def test_lists_values_at_their_edges(neg_rel, dim):
    """Hand-made queries (see _value_lists) on integer ACR rows, acr_dim 1 and 5, neg_relevance 1e-6, 0.1 and 1.  Bar
    1e-12 relative (worst on the H100 below 6e-16); NDCG of a single label occurrence within one log2 ulp (2 ulp of the
    quotient); a bad label or id sets err, writes six zeros and marks none of its ids."""
    acr, pop = _value_table(dim)
    Ls = _value_lists()
    nq, length, top_n = len(Ls), 12, 8
    ids = np.array([v for row, _ in Ls for v in row], np.int64)
    labels = np.array([lab for _, lab in Ls], np.int64)
    worst = _lists_check((ids, labels, pop, acr, dim, top_n, 1, nq, length, length, nq * length),
                         dict(neg_rel=neg_rel), expect_err=1)
    rc, pq, bm, err, bits0, norms = _lists_run(ids, labels, pop, acr, dim, top_n, 1, nq, length, length, nq * length,
                                               neg_rel=neg_rel, bits0=np.zeros(2, np.uint32))
    got = pq[:nq * N_VALUES].view(np.float64).reshape(nq, N_VALUES)
    for q in (0, 1, 11):                             # one occurrence inside m, at rank 0, m - 1 and 6
        k = Ls[q][0].index(Ls[q][1])
        want = 1.0 / math.log2(k + 2)
        assert abs(got[q, 0] - want) <= 2 * np.spacing(want), (q, got[q, 0], want)
    assert got[2, 0] == 0.0                          # the label only past m
    for q in (9, 10):                                # bad queries: none of their ids is marked
        for i in Ls[q][0][:top_n]:
            if 0 <= i < 64 and i not in {v for r, _ in Ls[:9] + Ls[11:] for v in r[:top_n]}:
                assert not (bm[i >> 5] >> (i & 31)) & 1, (q, i)
    print('lists values dim=%d neg_rel=%g worst rel %.3g' % (dim, neg_rel, worst))


# ================================================================================================ reduce, mark, popcount
def _reduce_emul(pq):
    """reduce_kernel's order: thread t sums q = t, t + 256, ... in turn, then a tree over halves 128, 64, ..., 1"""
    part = np.zeros((256, N_VALUES))
    for k in range(0, pq.shape[0], 256):
        blk = pq[k:k + 256]
        part[:blk.shape[0]] = part[:blk.shape[0]] + blk
    h = 128
    while h:
        part[:h] = part[:h] + part[h:2 * h]
        h >>= 1
    return part[0]


@gpu
@pytest.mark.parametrize('nq', [0, 1, 255, 256, 257, 100003])
def test_reduce_bit_for_bit(nq):
    """acc[row] += the kernel's fixed-order sum of per_query[row], bit for bit against a numpy emulation of that order;
    rows outside the mask and the guard keep their prefill; nq = 0 writes nothing."""
    torch = _torch()
    rs = np.random.RandomState(nq % 1000)
    rows, mask = 3, 0b101 | (1 << 7)
    pq = (rs.randn(rows, nq, N_VALUES) * 10.0 ** rs.uniform(-4, 4, (rows, nq, N_VALUES))).astype(np.float64)
    acc0 = rs.randn(rows * N_VALUES + GUARD) * 1e3
    acc = _dev(acc0)
    assert _lib().nar_eval_metrics_reduce(_p(_dev(pq.reshape(-1) if nq else np.zeros(1))), rows, mask, nq, _p(acc),
                                          _s()) == 0
    torch.cuda.synchronize()
    got = acc.cpu().numpy()
    want = acc0.copy()
    if nq:
        for r in (0, 2):
            want[r * N_VALUES:(r + 1) * N_VALUES] = acc0[r * N_VALUES:(r + 1) * N_VALUES] + _reduce_emul(pq[r])
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    for bad in (dict(rows=0), dict(rows=64), dict(nq=-1)):
        a = dict(rows=rows, nq=nq)
        a.update(bad)
        assert _lib().nar_eval_metrics_reduce(_p(_dev(np.zeros(8))), a['rows'], mask, a['nq'], _p(acc), _s()) == \
            NAR_ERR_INVALID
    assert np.array_equal(acc.cpu().numpy().view(np.uint64), want.view(np.uint64))


@gpu
@pytest.mark.parametrize('num_items', [1, 31, 32, 33, 46034])
@pytest.mark.parametrize('skip_zero', [0, 1])
def test_mark_bit_for_bit(num_items, skip_zero):
    """The bits of every id OR the prefill, id 0 skipped only with skip_zero, the guard words untouched; ids -1 and
    num_items set err and no bit; n = 0 writes nothing."""
    torch = _torch()
    rs = np.random.RandomState(num_items + skip_zero)
    words = (num_items + 31) // 32
    n = min(3 * num_items + 5, 50000)
    ids = rs.randint(0, num_items, n).astype(np.int64)
    ids[::7] = 0
    b0 = np.where(rs.rand(words) < 0.3, rs.randint(0, 1 << 31, words), 0).astype(np.uint32)
    b0[0] &= ~np.uint32(1)                           # bit 0 clear, so skip_zero shows
    pre = np.concatenate([b0, np.full(GUARD, SENT32, np.uint32)])
    want = pre.copy()
    for i in ids.tolist():
        if i or not skip_zero:
            want[i >> 5] |= np.uint32(1 << (i & 31))
    bm = _dev(pre.view(np.int32))
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    lib = _lib()
    assert lib.nar_eval_metrics_mark(_p(_dev(ids)), n, num_items, skip_zero, _p(bm), _p(err), _s()) == 0
    assert np.array_equal(_bits(bm, 32), want) and int(_bits(err, 32)[0]) == 0
    assert lib.nar_eval_metrics_mark(_p(_dev(ids)), 0, num_items, skip_zero, _p(bm), _p(err), _s()) == 0
    assert lib.nar_eval_metrics_mark(_p(None), 0, num_items, skip_zero, _p(bm), _p(err), _s()) == 0
    assert np.array_equal(_bits(bm, 32), want) and int(_bits(err, 32)[0]) == 0
    for bad in (-1, num_items):
        b2 = _dev(pre.view(np.int32))
        assert lib.nar_eval_metrics_mark(_p(_dev(np.array([bad], np.int64))), 1, num_items, skip_zero, _p(b2), _p(err),
                                         _s()) == 0
        assert np.array_equal(_bits(b2, 32), pre) and int(_bits(err, 32)[0]) == 1
        err.zero_()
    assert lib.nar_eval_metrics_mark(_p(_dev(ids)), n, 0, skip_zero, _p(bm), _p(err), _s()) == NAR_ERR_INVALID
    assert lib.nar_eval_metrics_mark(_p(_dev(ids)), -1, num_items, skip_zero, _p(bm), _p(err), _s()) == NAR_ERR_INVALID
    assert np.array_equal(_bits(bm, 32), want)


@gpu
@pytest.mark.parametrize('words', [1, 2, 255, 256, 257, 1439, 5000])
def test_popcount_exact(words):
    """counts[i] = the set bits of bitmap i, for words below, at and above the CTA's 256 threads (strided)."""
    rs = np.random.RandomState(words)
    n_maps = 5
    b = rs.randint(0, 1 << 32, size=(n_maps, words), dtype=np.uint64).astype(np.uint32)
    b[1] = 0
    b[2] = 0xFFFFFFFF
    cnt = _filled(n_maps, SENT64, 64)
    assert _lib().nar_eval_metrics_popcount(_p(_dev(b.view(np.int32))), n_maps, words, _p(cnt), _s()) == 0
    got = _bits(cnt, 64)
    want = np.array([sum(bin(int(v)).count('1') for v in row) for row in b], np.uint64)
    assert np.array_equal(got[:n_maps], want) and np.all(got[n_maps:] == SENT64)
    assert _lib().nar_eval_metrics_popcount(_p(_dev(b.view(np.int32))), 0, words, _p(cnt), _s()) == NAR_ERR_INVALID
    assert _lib().nar_eval_metrics_popcount(_p(_dev(b.view(np.int32))), n_maps, 0, _p(cnt), _s()) == NAR_ERR_INVALID


# ================================================================================================ hit rate by position
def _bp_batch(rs, B, T, V, rows, length, q_extra=0, label_stride=1, full_frac=0.3):
    """Compact session-major rows: session b has n_b <= T rows at positions b * T + t.  -> (ids [rows, nq, q_stride],
    labels [nq * label_stride], pos_idx, sess_off, lengths)"""
    n = rs.randint(0, T + 1, B)
    n[rs.rand(B) < full_frac] = T
    sess_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
    nq = int(sess_off[-1])
    pos = np.concatenate([b * T + np.arange(n[b]) for b in range(B)]).astype(np.int32) if nq else np.zeros(0, np.int32)
    lab = rs.randint(1, V, nq).astype(np.int64)
    lab[rs.rand(nq) < 0.15] = 0
    labels = np.full(max(nq * label_stride, 1), -9, np.int64)
    labels[:nq * label_stride:label_stride] = lab
    q_stride = length + q_extra
    ids = np.full((rows, max(nq, 1), q_stride), -3, np.int64)
    ids[:, :nq, :length] = rs.randint(0, V, (rows, nq, length))
    hit = rs.rand(rows, nq) < 0.4
    where = rs.randint(0, length, (rows, nq))
    for r in range(rows):
        ids[r, np.flatnonzero(hit[r]), where[r, hit[r]]] = lab[hit[r]]
    return ids, labels, pos, sess_off, n


class _BP:
    """Sentinel / prefilled by-position outputs carried over batches, and their reference."""

    def __init__(self, rs, rows, T, ld, top_n, num_items):
        self.rows, self.T, self.ld, self.top_n, self.num_items = rows, T, ld, top_n, num_items
        self.h0 = rs.randint(1, 1000, rows * ld + GUARD).astype(np.int64)
        self.t0 = self.h0 + rs.randint(0, 1000, rows * ld + GUARD)
        self.np0 = rs.uniform(0.5, 3.0, T + GUARD).astype(np.float32)
        self.hits, self.total, self.norm_pop = _dev(self.h0), _dev(self.t0), _dev(self.np0)
        self.err = _torch().zeros(1, dtype=_torch().int32, device='cuda')
        self.ref = ByPositionRef(rows, top_n)
        self.ref.begin()
        self.pref = ByPositionRef(1, top_n)
        self.pref.begin()
        for t in range(T):
            self.pref.norm_pop[0][t + 1] = self.np0[t]

    def add(self, ids, labels, nq, length, mask, pos=None, sess_off=None, pop=None, label_stride=1):
        rows = self.rows
        rc = _lib().nar_eval_by_position(
            _p(_dev(ids)), ids.shape[1] * ids.shape[2], ids.shape[2], rows, _i64(mask), nq, length, self.top_n,
            _p(_dev(labels)), label_stride, _p(None if pos is None else _dev(pos)), self.T,
            _p(None if sess_off is None else _dev(sess_off)), 0 if sess_off is None else sess_off.size - 1,
            _p(None if pop is None else _dev(pop)), self.num_items, _p(self.hits), _p(self.total), self.ld,
            _p(self.norm_pop), _p(self.err), _s())
        if rc:
            return rc
        lab = labels[:nq * label_stride:label_stride]
        for r in range(rows):
            if (mask >> r) & 1:
                self.ref.add(r, ids[r, :nq, :length], lab, self.T, pos)
        if pop is not None:
            self.pref.add(0, ids[0, :nq, :length], lab, self.T, pos, pop)
        return rc

    def check(self):
        h, t, npop = _bits(self.hits, 64).view(np.int64), _bits(self.total, 64).view(np.int64), \
            _bits(self.norm_pop, 32)
        wh, wt = self.h0.copy(), self.t0.copy()
        for r in range(self.rows):
            for p, v in self.ref.total[r].items():
                wt[r * self.ld + p - 1] += v
            for p, v in self.ref.hits[r].items():
                wh[r * self.ld + p - 1] += v
        assert np.array_equal(h, wh), 'hits'
        assert np.array_equal(t, wt), 'total'
        wn = self.np0.copy()
        for p, v in self.pref.norm_pop[0].items():
            wn[p - 1] = v
        assert np.array_equal(npop, wn.view(np.uint32)), 'norm_pop'
        assert int(_bits(self.err, 32)[0]) == 0


BP_T = [(1, 9000), (2, 5000), (255, 40), (256, 37), (257, 33), (1000, 11), (1024, 9)]


@gpu
@pytest.mark.parametrize('T,B', BP_T)
def test_by_position_every_position_count(T, B):
    """T = 1 .. 1024 (257 and 1000 do not divide POP_CHUNK = 4096), n_sess * T spanning several 4096-cell chunks with a
    partial last one, two batches: hits and total grow from a nonzero prefill by exactly the oracle's counts (columns
    past T keep it), norm_pop equals the oracle's sequential float32 sum from a nonzero prefill bit for bit."""
    rs = np.random.RandomState(T)
    V, rows, length, top_n = 5000, 3, 7, 5
    st = _BP(rs, rows, T, T + 3, top_n, V)
    pop = rs.uniform(0, 1, V).astype(np.float32)
    for batch in range(2):
        Bb = B if batch == 0 else max(1, B // 3)
        ids, labels, pos, sess_off, _ = _bp_batch(rs, Bb, T, V, rows, length, q_extra=2)
        nq = pos.size
        assert st.add(ids, labels, nq, length, 0b101, pos, sess_off, pop) == 0
    st.check()


@gpu
def test_by_position_grid_form_rows_and_strides():
    """pos_idx null (nq = B * T, query q at q % T), 63 rows with a sparse mask (bit 62 in, bits >= rows ignored),
    ld > T, top_n > len, label_stride 2, q_stride > len: exact counts, untouched columns and rows."""
    rs = np.random.RandomState(11)
    V, rows, T, B, length, top_n = 300, 63, 7, 40, 4, 9
    st = _BP(rs, rows, T, T + 5, top_n, V)
    nq = B * T
    lab = rs.randint(0, V, nq).astype(np.int64)
    labels = np.full(2 * nq, -9, np.int64)
    labels[::2] = lab
    ids = rs.randint(0, V, (rows, nq, length + 3)).astype(np.int64)
    ids[:, :, 1] = np.where(rs.rand(rows, nq) < 0.5, lab, ids[:, :, 1])
    mask = (1 << 0) | (1 << 9) | (1 << 31) | (1 << 62) | (1 << 63)
    assert st.add(ids, labels, nq, length, mask, label_stride=2) == 0
    st.check()


@gpu
def test_by_position_rejected_calls():
    """T = 1025 is NAR_ERR_UNSUPPORTED; ld < T, nq not a multiple of T without pos_idx, pop without sess_off are
    NAR_ERR_INVALID; none writes an output."""
    rs = np.random.RandomState(3)
    V, length = 100, 4
    for T, kw, want in ((1025, {}, NAR_ERR_UNSUPPORTED), (8, dict(ld=7), NAR_ERR_INVALID),
                        (8, dict(grid=True, nq=9), NAR_ERR_INVALID), (8, dict(no_off=True), NAR_ERR_INVALID)):
        st = _BP(rs, 2, T, kw.get('ld', T), 3, V)
        ids, labels, pos, sess_off, _ = _bp_batch(rs, 3, T, V, 2, length)
        pop = rs.uniform(0, 1, V).astype(np.float32)
        nq = kw.get('nq', pos.size)
        if kw.get('grid'):
            rc = st.add(ids, labels, nq, length, 3)
        else:
            rc = st.add(ids, labels, nq, length, 3, pos, None if kw.get('no_off') else sess_off, pop)
        assert rc == want, (T, kw, rc)
        st.ref.begin()
        st.pref.begin()
        for t in range(T):
            st.pref.norm_pop[0][t + 1] = st.np0[t]
        st.check()


# ================================================================================================ session logs
def _round_up(x, m):
    return (x + m - 1) // m * m


def _layout(B, rows, K, flags):
    """the documented packed-log layout: byte offsets of counts, neg, labels, ids, probs, pops, the total, Kp, Wp"""
    Kp, Wp = _round_up(K, 2), _round_up(K + 1, 4)
    off = _round_up(16 + 4 * B, 16)
    o = [16]
    for bit, size in ((1, rows * Kp * 8), (2, _round_up(rows * 8, 16)), (2, rows * Wp * 8), (2, rows * Wp * 4),
                      (2, rows * Wp * 4)):
        o.append(off)
        off += size if flags & bit else 0
    return o + [off, Kp, Wp]


def test_session_logs_layout_offsets():
    """CPU: nar_eval_session_logs_layout returns the documented offsets for every K residue, B, rows and flags, and
    rejects bad arguments without writing."""
    lib = _lib()
    for B in (0, 1, 3, 4, 1000):
        for rows in (0, 1, 15, 33):
            for K in (1, 2, 3, 4, 5, 100):
                for flags in (0, 1, 2, 3):
                    out = (C.c_int64 * 9)()
                    assert lib.nar_eval_session_logs_layout(B, rows, K, flags, out) == 0
                    assert list(out) == _layout(B, rows, K, flags), (B, rows, K, flags)
    for args in ((-1, 1, 1, 1), (1, -1, 1, 1), (1, 1, 0, 1), (1, 1, 1, 4)):
        out = (C.c_int64 * 9)(*([7] * 9))
        assert lib.nar_eval_session_logs_layout(*args, out) == NAR_ERR_INVALID
        assert list(out) == [7] * 9


def _sl_problem(rs, B, L, K, V, T=48):
    n = rs.multinomial(L, np.ones(B) / B) if B else np.zeros(0, np.int64)
    while np.any(n > T):
        n = rs.multinomial(L, np.ones(B) / B)
    sess_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
    pos = np.concatenate([b * T + np.arange(n[b]) for b in range(B)] + [np.zeros(0, np.int64)]).astype(np.int32)
    label_next = np.zeros(B * T, np.int64)
    lab = rs.randint(1, V, L)
    lab[rs.rand(L) < 0.3] = 0
    label_next[pos] = lab
    W = K + 1
    pred_ids = rs.randint(0, V, (max(L, 1), W)).astype(np.int64)
    probs = rs.uniform(0, 1, (max(L, 1), W)).astype(np.float32)
    probs[:, 0] = np.float32(0.12345675)             # a tie of rint
    neg = rs.randint(1, V, (B * T, K)).astype(np.int64)
    cs = 3
    cand = np.full(max(L, 1) * cs, -1, np.int64)
    cand[:L * cs:cs] = label_next[pos]
    pop = rs.uniform(0, 1, V).astype(np.float32)
    return dict(n=n, sess_off=sess_off, pos=pos, label_next=label_next, pred_ids=pred_ids, probs=probs, neg=neg,
                cand=cand, cs=cs, pop=pop, T=T, W=W)


def _sl_expected(pb, B, L, K, flags, size):
    """the packed buffer a call must leave: the zeroed header gets Q, the rest of the buffer starts as 0x5A bytes"""
    o = _layout(B, L, K, flags)
    Kp, Wp = o[7], o[8]
    buf = np.full(size, 0x5A, np.uint8)
    buf[:16] = 0
    T = pb['T']
    labels2 = pb['label_next'].reshape(B, T)
    neg_log, rec_log = session_logs_ref(np.arange(B), labels2, pb['neg'].reshape(B, T, K) if flags & 1 else None,
                                        pb['pred_ids'][:L] if flags & 2 else None,
                                        pb['probs'][:L] if flags & 2 else None, pb['pop'], pb['pos'])
    counts = np.array([int(np.count_nonzero(labels2[b, :pb['n'][b]])) for b in range(B)], np.int32)
    Q = int(counts.sum())
    buf[:4] = np.array([Q], np.int32).view(np.uint8)
    buf[16:16 + 4 * B] = counts.view(np.uint8)
    if flags & 1:
        neg = np.zeros((Q, Kp), np.int64)
        neg[:, :K] = np.array([v for s in neg_log for v in s['negative_items']], np.int64).reshape(Q, K)
        buf[o[1]:o[1] + Q * Kp * 8] = neg.reshape(-1).view(np.uint8)
    if flags & 2:
        def cat(key, dt):
            return np.array([v for s in rec_log for v in s[key]], dt)
        buf[o[2]:o[2] + Q * 8] = cat('next_click_labels', np.int64).view(np.uint8)
        for k, key, dt in ((3, 'predicted_item_ids', np.int64), (4, 'predicted_item_probs', np.float32),
                           (5, 'predicted_item_norm_pop', np.float32)):
            a = np.zeros((Q, Wp), dt)
            a[:, :K + 1] = cat(key, dt).reshape(Q, K + 1)
            buf[o[k]:o[k] + a.nbytes] = a.reshape(-1).view(np.uint8)
    return buf


def _sl_run(pb, B, L, K, V, flags, misalign=0):
    torch = _torch()
    o = _layout(B, L, K, flags)
    size = o[6] + GUARD
    raw = torch.full((size + 32,), 0x5A, dtype=torch.uint8, device='cuda')
    raw[:16].zero_()
    rc = _lib().nar_eval_session_logs_pack(
        _p(_dev(pb['pred_ids'])), _p(_dev(pb['probs'])), _p(_dev(pb['cand'])), pb['cs'],
        _p(_dev(pb['pos'] if L else np.zeros(1, np.int32))),
        _p(_dev(pb['sess_off'])), _p(_dev(pb['pop'])), _p(_dev(pb['neg'])), _p(_dev(pb['label_next'])), B, K, L, V,
        flags, _p(raw, misalign), _s())
    torch.cuda.synchronize()
    return rc, raw.cpu().numpy()[:size], size


@gpu
@pytest.mark.parametrize('K', [1, 2, 3, 4, 5, 100])
def test_session_logs_pack_byte_for_byte(K):
    """L = 0, 1, 15, 16, 17 and 33 compact rows over flags 1, 2 and 3: the packed buffer equals a numpy build of the
    documented layout from the oracle's logs byte for byte - padding columns exactly 0, the bytes no section owns and
    the rows past Q keep the 0x5A fill, and so does the guard."""
    V = 700
    for L in (0, 1, 15, 16, 17, 33):
        for flags in (1, 2, 3):
            rs = np.random.RandomState(K * 100 + L * 3 + flags)
            B = 3 if L < 16 else 5
            pb = _sl_problem(rs, B, L, K, V)
            rc, got, size = _sl_run(pb, B, L, K, V, flags)
            assert rc == 0
            want = _sl_expected(pb, B, L, K, flags, size)
            assert np.array_equal(got, want), (L, flags, np.flatnonzero(got != want)[:8])


@gpu
def test_session_logs_header_over_many_sessions():
    """B = 1000 sessions with L = 10 rows: one CTA, so the per-session count loop takes four strides of 256."""
    rs = np.random.RandomState(17)
    B, L, K, V = 1000, 10, 4, 300
    pb = _sl_problem(rs, B, L, K, V)
    for flags in (1, 3):
        rc, got, size = _sl_run(pb, B, L, K, V, flags)
        assert rc == 0
        assert np.array_equal(got, _sl_expected(pb, B, L, K, flags, size)), flags


@gpu
def test_session_logs_rejects_an_unaligned_buffer():
    """An out pointer off 16-byte alignment is NAR_ERR_INVALID and leaves the buffer untouched."""
    rs = np.random.RandomState(2)
    pb = _sl_problem(rs, 3, 5, 3, 50)
    for mis in (4, 8):
        rc, got, size = _sl_run(pb, 3, 5, 3, 50, 3, misalign=mis)
        assert rc == NAR_ERR_INVALID
        want = np.full(size, 0x5A, np.uint8)
        want[:16] = 0
        assert np.array_equal(got, want)


# ================================================================================================ top n
def bloom_slot(i):
    return ((int(i) & 0xFFFFFFFF) * 2654435761 & 0xFFFFFFFF) >> 20


def _topn(lg, cand, top_n, ic=None, q_pos=None, T=0, scores=True, probs=True):
    Q = lg.shape[0]
    ids = _filled(Q * top_n, SENT64, 64)
    sc = _filled(Q * top_n, NAN32, 32) if scores else None
    pr = _filled(Q * top_n, NAN32, 32) if probs else None
    rc = _lib().nar_topn_candidates(_p(_dev(lg)), _p(_dev(cand)), Q, lg.shape[1], top_n,
                                    _p(None if ic is None else _dev(ic)), _p(None if q_pos is None else _dev(q_pos)), T,
                                    _p(ids), _p(sc), _p(pr), _s())
    return rc, _bits(ids, 64), None if sc is None else _bits(sc, 32), None if pr is None else _bits(pr, 32)


def _topn_check(lg, cand, top_n, ic=None, q_pos=None, T=0, scores=True, probs=True):
    """-> worst probability error relative to the bar"""
    Q = lg.shape[0]
    rc, ids, sc, pr = _topn(lg, cand, top_n, ic, q_pos, T, scores, probs)
    assert rc == 0, rc
    ex = None
    if ic is not None:
        ex = [set(ic[(p // T) * T:(p // T) * T + p % T + 1].tolist()) for p in q_pos.tolist()]
    wid, wsc, wpr = topn_rule(lg, cand, top_n, ex)
    n = Q * top_n
    assert np.all(ids[n:] == SENT64)
    assert np.array_equal(ids[:n].view(np.int64).reshape(Q, top_n), wid), 'ids'
    worst = 0.0
    if scores:
        assert np.all(sc[n:] == NAN32)
        assert np.array_equal(sc[:n].reshape(Q, top_n), wsc.astype(np.float32).view(np.uint32)), 'scores'
    if probs:
        assert np.all(pr[n:] == NAN32)
        got = pr[:n].view(np.float32).reshape(Q, top_n).astype(np.float64)
        assert not np.any(np.isnan(got))
        e = np.abs(got - wpr) / (PROB_BAR * wpr + 1e-30)
        worst = float(e.max())
        assert worst <= 1.0, worst
    return worst


def _tied_logits(rs, Q, N):
    lg = (rs.randn(Q, N) * 3).astype(np.float32)
    lg[0] = np.round(lg[0])                          # a handful of distinct values: ties everywhere
    if Q > 1:
        lg[1, ::3] = lg[1, 5]
    return lg


TOPN_SIZES = [(511, 1), (511, 2), (511, 3), (511, 511), (512, 1), (512, 512), (513, 511), (513, 512), (513, 513),
              (1025, 3), (1025, 513), (1025, 1025), (4095, 4095), (4096, 4095), (4096, 4096), (5000, 4096)]


@gpu
@pytest.mark.parametrize('N,top_n', TOPN_SIZES)
def test_topn_sizes(N, top_n):
    """top_n 1, 2, 3, 511, 512, 513, 4095 and 4096 over N = 511, 512, 513, 1025 and up, with and without a 6-click
    exclusion list: ids and scores bit for bit against topn_rule, probabilities within 1e-6 relative (worst on the
    H100 9.5e-8)."""
    rs = np.random.RandomState(N + top_n)
    Q, T = 4, 6
    lg = _tied_logits(rs, Q, N)
    cand = (rs.permutation(2 * N)[:N] + 1).astype(np.int64)
    ic = rs.randint(1, 2 * N + 10, (Q, T)).astype(np.int64)
    ic[:, 1] = cand[rs.randint(0, N, Q)]
    ic = ic.reshape(-1)
    q_pos = (np.arange(Q) * T + np.array([0, 5, 2, 5])).astype(np.int32)
    worst = 0.0
    for excl in (False, True):
        worst = max(worst, _topn_check(lg, cand, top_n, ic if excl else None, q_pos if excl else None, T))
    print('topn N=%d top_n=%d worst prob err / bar %.3g' % (N, top_n, worst))


@gpu
def test_topn_rejected_calls():
    """top_n 0, 4097 and > N are NAR_ERR_INVALID, T = 1025 with an exclusion list NAR_ERR_UNSUPPORTED, an exclusion list
    without q_pos NAR_ERR_INVALID; none writes an output."""
    rs = np.random.RandomState(4)
    lg = rs.randn(2, 5000).astype(np.float32)
    cand = np.arange(1, 5001, dtype=np.int64)
    ic = np.ones(2 * 1025, np.int64)
    qp = np.array([0, 1025], np.int32)
    for kw, want in ((dict(top_n=0), NAR_ERR_INVALID), (dict(top_n=4097), NAR_ERR_INVALID),
                     (dict(top_n=512, N=511), NAR_ERR_INVALID), (dict(top_n=5, T=1025, ic=ic, q_pos=qp), NAR_ERR_UNSUPPORTED),
                     (dict(top_n=5, T=6, ic=ic), NAR_ERR_INVALID)):
        N = kw.get('N', 5000)
        rc, ids, sc, pr = _topn(np.ascontiguousarray(lg[:, :N]), cand[:N], kw['top_n'], kw.get('ic'), kw.get('q_pos'),
                                kw.get('T', 0))
        assert rc == want, (kw, rc)
        assert np.all(ids == SENT64) and np.all(sc == NAN32) and np.all(pr == NAN32), kw


@gpu
def test_topn_longest_exclusion_list_and_bloom_collisions():
    """T = 1024 queried at t = 1023 (1024 excluded clicks, the last one a candidate no other click names), at 0 and at
    500; candidates that share a Bloom slot with an excluded id without being excluded must stay."""
    rs = np.random.RandomState(8)
    T, N, top_n = 1024, 6000, 2500
    cand = (rs.permutation(20000)[:N] + 1).astype(np.int64)
    lg = _tied_logits(rs, 3, N)
    ic = np.zeros((3, T), np.int64)
    for b in range(3):
        ic[b] = cand[rs.permutation(N)[:T]]
    q_pos = np.array([0 * T + 1023, 1 * T + 0, 2 * T + 500], np.int32)
    # the last click of query 0 scores high and appears nowhere else in its list
    last = ic[0, 1023]
    lg[0, np.flatnonzero(cand == last)] = 50.0
    excl = set(ic[0].tolist())
    slots = {bloom_slot(i) for i in excl}
    coll = [c for c in cand.tolist() if c not in excl and bloom_slot(c) in slots]
    assert len(coll) > 100                           # premise: many non-excluded candidates collide
    lg[0, np.isin(cand, coll[:50])] = 40.0           # and some of them rank at the top
    worst = _topn_check(lg, cand, top_n, ic.reshape(-1), q_pos, T)
    print('topn T=1024 worst prob err / bar %.3g' % worst)


@gpu
def test_topn_every_candidate_excluded_and_short_lists():
    """Every candidate excluded: every slot holds id 0, score -inf, probability 0.  7 of 10 excluded at top_n 5: three
    real slots, then the padding."""
    rs = np.random.RandomState(9)
    T = 12
    cand = np.arange(100, 110, dtype=np.int64)
    lg = rs.randn(2, 10).astype(np.float32)
    ic = np.zeros((2, T), np.int64)
    ic[0, :10] = cand
    ic[0, 10:] = 5
    ic[1, :7] = cand[[0, 2, 3, 5, 6, 8, 9]]
    ic[1, 7:] = 999
    q_pos = np.array([11, T + 11], np.int32)
    for top_n in (1, 5, 10):
        _topn_check(lg, cand, top_n, ic.reshape(-1), q_pos, T)
    rc, ids, sc, pr = _topn(lg, cand, 5, ic.reshape(-1), q_pos, T)
    assert np.all(ids[:5] == 0) and np.all(sc[:5].view(np.float32) == -np.inf) and np.all(pr[:5] == 0)
    assert np.count_nonzero(ids[5:10]) == 3


@gpu
def test_topn_signed_zeros_extremes_and_subnormals():
    """+0 / -0 ties (equal keys, order by index, each score returned with its own sign), +-3.4e38 and subnormals, and a
    row of nothing but signed zeros."""
    rs = np.random.RandomState(10)
    N = 1500
    base = np.array([0.0, -0.0, 3.4e38, -3.4e38, 1e-45, -1e-45, 1e-40, -1e-40, 1.17e-38, 0.0, -0.0, 2.0, -2.0],
                    np.float32)
    lg = np.zeros((3, N), np.float32)
    lg[0] = base[rs.randint(0, base.size, N)]
    lg[1] = base[rs.randint(0, base.size, N)]
    lg[1][lg[1] > 1e30] = 1.0                         # no 3.4e38: the zeros and subnormals carry probability
    lg[2] = np.where(rs.rand(N) < 0.5, np.float32(0.0), np.float32(-0.0))
    cand = np.arange(1, N + 1, dtype=np.int64)
    worst = 0.0
    for top_n in (1, 7, 200, 600, 1500):
        worst = max(worst, _topn_check(lg, cand, top_n))
    print('topn special values worst prob err / bar %.3g' % worst)


@gpu
def test_topn_pivot_tie_across_tiles():
    """100 scores above a value that 2500 candidates share, spread over every 512-wide tile: top_n 800 takes 700 of the
    ties, the lowest indices, so k_tie lands in the middle of a tile; top_n 101 takes one; 4096 of N = 8000 with 5000
    ties takes 3996."""
    rs = np.random.RandomState(12)
    for N, n_tie, top_n in ((4000, 2500, 800), (4000, 2500, 101), (8000, 5000, 4096)):
        lg = rs.uniform(-10, 0.5, (2, N)).astype(np.float32)
        for q in range(2):
            idx = rs.permutation(N)
            lg[q, idx[:100]] = rs.uniform(2, 5, 100).astype(np.float32)
            lg[q, idx[100:100 + n_tie]] = 1.0
        cand = (rs.permutation(3 * N)[:N] + 1).astype(np.int64)
        _topn_check(lg, cand, top_n)


@gpu
def test_topn_null_score_and_probability_outputs():
    """out_scores and / or out_probs null: the ids are the same, the other output unchanged."""
    rs = np.random.RandomState(13)
    lg = _tied_logits(rs, 3, 900)
    cand = np.arange(7, 907, dtype=np.int64)
    for scores, probs in ((False, True), (True, False), (False, False)):
        _topn_check(lg, cand, 50, scores=scores, probs=probs)


@gpu
def test_topn_many_queries():
    """Q = 70 000 (a grid above 65 535) over N = 5 candidates, top_n 3."""
    rs = np.random.RandomState(14)
    Q, N = 70000, 5
    lg = np.round(rs.randn(Q, N) * 2).astype(np.float32)
    cand = np.array([11, 3, 7, 5, 2], np.int64)
    _topn_check(lg, cand, 3)


# ================================================================================================ EvalMetrics limits
def test_eval_metrics_rejects_shared_memory_past_the_cap_up_front():
    """CPU: EvalMetrics raises ValueError when 8 top_n^2 + 4 top_n acr_dim exceeds 200 KB (top_n 64 with acr_dim 673,
    top_n 10 with acr_dim 5101), before it touches the device."""
    import torch
    from chameleon_recsys_b200.eval_metrics import EvalMetrics
    for top_n, dim in ((64, 673), (10, 5101)):
        with pytest.raises(ValueError, match='shared memory'):
            EvalMetrics(1, 10, torch.zeros(10, dim), dim, top_n, 0.1)


@gpu
def test_eval_metrics_accepts_the_cap():
    """EvalMetrics at exactly 200 KB (top_n 64, acr_dim 672) scores a batch and matches the oracle (bar 1e-12)."""
    import torch
    from chameleon_recsys_b200.eval_metrics import EvalMetrics
    from oracle.eval_metrics_ref import EvalMetricsRef
    rs = np.random.RandomState(15)
    V, dim, top_n, nq = 120, 672, 64, 3
    acr = rs.randn(V, dim).astype(np.float32)
    pop = rs.uniform(0.01, 1, V).astype(np.float32)
    ids = rs.randint(0, V, (nq, 70)).astype(np.int64)
    labels = np.array([ids[0, 3], 0, ids[2, 69]], np.int64)
    em = EvalMetrics(1, V, _dev(acr), dim, top_n, 0.1)
    em.begin(torch.zeros(4, dtype=torch.int64))
    em.add_lists(_dev(ids), _dev(labels), _dev(pop))
    got = em.results()[0]
    ref = EvalMetricsRef(1, top_n, acr.astype(np.float64), 0.1)
    ref.begin(np.zeros(4, np.int64))
    ref.add_lists(0, ids, labels, pop)
    want = ref.per_query_means(0)
    for i, k in enumerate(('ndcg_at_n', 'esi-r_at_n', 'esi-rr_at_n', 'content_eild-r_at_n', 'content_eild-rr_at_n')):
        w = want[('ndcg', 'esi-r', 'esi-rr', 'eild-r', 'eild-rr')[i]]
        assert abs(got[k] - w) <= 1e-12 * abs(w), (k, got[k], w)
