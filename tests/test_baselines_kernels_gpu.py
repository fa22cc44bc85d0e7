"""The evaluation baselines' kernels (csrc/baselines.cu, csrc/sknn.cu) bit for bit against their oracles
(oracle/baselines_ref.py, oracle/sknn_ref.py) at every table, ring and candidate limit.

Every output of these kernels is an integer or an exactly rounded fp64 value, so each case demands the oracle's bits.
The C entry points are driven directly (the wrappers cannot reach ``cap``, ``W``, ``S``, ``batch_seq`` or ``err`` at their
limits); ``BaselineTables`` / ``SessionKNN`` are driven for growth, snapshot / restore and load.  Outputs start from a
sentinel and carry guard space past their end that must keep it; output rows a call must not write (disabled baselines,
queries without a label) must keep the sentinel too.  ``metrics`` starts from a nonzero prefill and must grow by exactly
the oracle's sums.  A rejected call returns before any launch and leaves every output untouched.

Exactness premises (checked on the CPU): sequential-rules units divide lcm(1..20); integer ACR rows give exact norms,
dots and cosines; item_knn's ``pow`` is not correctly rounded on the GPU, so alpha 0.5 / 0.75 compare ranks only where
the oracle's score gaps exceed 8 ulp, and alpha 0 / 1 compare exactly.
"""
import ctypes as C
import itertools

import numpy as np
import pytest

from oracle.baselines_ref import SUFFIXES, BaselinesRef, lcm_upto
from oracle.sknn_ref import SknnRef

gpu = pytest.mark.gpu
NAR_ERR_INVALID, NAR_ERR_UNSUPPORTED = -1, -2
SENT64 = 0x5A5A5A5A5A5A5A5A
SENT32 = 0x5A5A5A5A
SENTF = -7.25
GUARD = 64
BIG = np.iinfo(np.int64).max
FIRST_NONE = 0x7F7F7F7F                     # buffer_hist's first index of an absent id
MAX_ID = (1 << 31) - 1                      # the largest num_items the entry points accept
WIDTH = 65                                  # SessionKNN's ring width
PRE5 = np.array([(i + 1) / 3.0 for i in range(15)])
PRE3 = np.array([1 / 7.0, 2 / 7.0, 3 / 7.0])


# ------------------------------------------------------------------------------------------------ plain models
M64 = (1 << 64) - 1


def mix64(x):
    """csrc/baselines.cu mix64"""
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33
    x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


def lane_norms(acr, dim):
    """row_norms_kernel's arithmetic: lane l sums x*x (exact in fp64) over k = l, l+32, ... with one rounding per add,
    then a butterfly over xor offsets 16..1, then sqrt."""
    x = np.asarray(acr, dtype=np.float64)[:, :dim]
    s = np.zeros((x.shape[0], 32))
    for k in range(dim):
        s[:, k % 32] = s[:, k % 32] + x[:, k] * x[:, k]
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, np.arange(32) ^ o]
    return np.sqrt(s[:, 0])


def hist_ref(buf, num_items):
    cnt = np.zeros(num_items, dtype=np.int32)
    first = np.full(num_items, FIRST_NONE, dtype=np.int32)
    for i, v in enumerate(np.asarray(buf).tolist()):
        if v != 0:
            cnt[v] += 1
            first[v] = min(first[v], i)
    return cnt, first


def knn_gap_ok(pop, lam, alpha, item, cands, co, ulps=8):
    """True when every two admissible item_knn candidates with different inputs (cooc, pop) have oracle scores more
    than ``ulps`` ulp apart: then pow errors of a few ulp cannot reorder them."""
    seen, xs = set(), []
    for c in cands:
        c = int(c)
        if c in seen or co.get((item, c), 0) <= 0:
            seen.add(c)
            continue
        seen.add(c)
        norm = np.power(pop[c] + lam, alpha) * np.power(pop[item] + lam, 1.0 - alpha)
        xs.append((float(co[(item, c)] / norm), (co[(item, c)], int(pop[c]))))
    for (a, ia), (b, ib) in itertools.combinations(xs, 2):
        if ia != ib and abs(a - b) <= ulps * np.spacing(max(abs(a), abs(b))):
            return False
    return True


# ------------------------------------------------------------------------------------------------ CPU premises
def test_sr_units_are_exact():
    """CPU: every 'div' decay 1/d of max_clicks_dist D is a whole number of units 1/lcm(1..D), and a table's weights stay
    far inside int64."""
    assert lcm_upto(20) == 232792560
    for D in range(1, 21):
        u = lcm_upto(D)
        assert all(u % d == 0 for d in range(1, D + 1))
        assert u * 1024 * 20 * (1 << 16) < 2 ** 62


def _int_acr(rs, n, dim, ld):
    a = np.zeros((n, ld), dtype=np.float32)
    a[:, :dim] = rs.randint(-3, 4, size=(n, dim))
    a[0] = 0.0
    return a


def test_integer_acr_cosines_are_exact():
    """CPU: for small-integer ACR rows the kernel's norms (lane order) equal numpy's, every dot is an integer below
    2^53, so the kernel's dot / (na * nc) is the oracle's cosine bit for bit."""
    rs = np.random.RandomState(1)
    for dim in (1, 24, 33, 250):
        acr = _int_acr(rs, 40, dim, dim + 5)
        x = acr[:, :dim].astype(np.float64)
        ln = lane_norms(acr, dim)
        np.testing.assert_array_equal(ln, np.array([np.linalg.norm(r) for r in x]))
        dots = x @ x.T
        assert np.all(dots == np.round(dots)) and np.abs(dots).max() < 2 ** 53
        ref = BaselinesRef(40, acr=x)
        for i in range(1, 40):
            sc = ref.candidate_scores('cb', i, list(range(40)), [], None)
            for c, v in sc.items():
                nn = ln[i] * ln[c]
                assert v == (dots[i, c] / nn if nn > 0 else 0.0)


def test_item_knn_gap_rule():
    """CPU: scores more than 8 ulp apart keep their order when each candidate's pow result moves by up to 2 ulp (the
    CUDA pow bound) and the product and quotient are rounded again; scores within 1 ulp can swap."""
    rs = np.random.RandomState(2)
    for alpha in (0.5, 0.75):
        co = rs.randint(1, 6, size=4000).astype(np.float64)
        pop = rs.randint(0, 60, size=4000).astype(np.float64)
        pa = np.power(31.0 + 20.0, 1.0 - alpha)
        pc = np.power(pop + 20.0, alpha)
        s = co / (pc * pa)
        i, j = rs.randint(0, 4000, size=(2, 20000))
        far = np.abs(s[i] - s[j]) > 8 * np.spacing(np.maximum(s[i], s[j]))
        assert far.mean() > 0.5
        for di, dj in itertools.product(range(-2, 3), repeat=2):
            pi, pj = pc[i].copy(), pc[j].copy()
            for _ in range(abs(di)):
                pi = np.nextafter(pi, np.inf if di > 0 else -np.inf)
            for _ in range(abs(dj)):
                pj = np.nextafter(pj, np.inf if dj > 0 else -np.inf)
            si, sj = co[i] / (pi * pa), co[j] / (pj * pa)
            assert np.array_equal(np.sign(si - sj)[far], np.sign(s[i] - s[j])[far])


RETURNING = [(5, [1]), (6, [1]), (5, [1]), (7, [1]), (8, [1]), (5, [1])]


def test_returning_id_oracle_export():
    """CPU: S = 4, one session per batch, ids 5, 6, 5, 7, 8, 5 each holding item 1.  The 5th batch evicts the first 5,
    which discards (1, 5): the surviving middle 5 is dead.  The 6th adds (1, 5) back before evicting 6: it is live."""
    ref = SknnRef(sessions_buffer_size=4)
    live = []
    for s, items in RETURNING:
        ref.update([s], np.array([items]))
        live.append(ref.export()['live'][:, 0].tolist())
    assert ref.export()['ids'].tolist() == [5, 7, 8, 5]
    assert live[4] == [True, False, True, True]            # [6, 5, 7, 8]
    assert live[5] == [True, True, True, True]             # [5, 7, 8, 5]


# ------------------------------------------------------------------------------------------------ GPU plumbing
def _torch():
    import torch
    return torch


def _lib():
    from chameleon_recsys_b200._lib import load
    return load()


def _s():
    return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _full(n, val, dtype):
    torch = _torch()
    dt = {'i64': torch.int64, 'i32': torch.int32, 'f64': torch.float64}[dtype]
    return torch.full((n + GUARD,), val, dtype=dt, device='cuda')


def _host(t):
    _torch().cuda.synchronize()
    return t.cpu().numpy()


def _prefilled(pre):
    t = _full(pre.size, SENTF, 'f64')
    t[:pre.size] = _dev(pre)
    return t


def _scalar(val, dtype):
    t = _full(1, SENT64 if dtype == 'i64' else SENT32, dtype)
    t[0] = val
    return t


def _guards(*pairs):
    for t, n, v in pairs:
        g = _host(t)[n:]
        assert (g == v).all(), 'guard overwritten'


# ------------------------------------------------------------------------------------------------ pair table
class Table:
    """A raw pair table of ``cap`` slots (+ guard), its occupancy counter and the error flag."""

    def __init__(self, cap, clear=True):
        self.cap = cap
        self.t = [_full(cap, SENT64, 'i64') for _ in range(4)]
        self.count = _scalar(0, 'i64')
        self.err = _scalar(0, 'i32')
        if clear:
            assert _lib().nar_baselines_clear(*self.ptrs(), cap, _s()) == 0

    def ptrs(self):
        return [_p(x) for x in self.t]

    def update(self, ai, num_items, D=10, seq=0, Bg=None, T1=None):
        ai = np.asarray(ai, dtype=np.int64)
        Bg = ai.shape[0] if Bg is None else Bg
        T1 = ai.shape[1] if T1 is None else T1
        d = _dev(ai) if ai.size else _full(0, 0, 'i64')
        return _lib().nar_baselines_update(*self.ptrs(), self.cap, _p(self.count), _p(d), Bg, T1, num_items, D, seq,
                                           _p(self.err), _s())

    def export(self):
        keys = _host(self.t[0])[:self.cap]
        occ = keys != -1
        order = np.argsort(keys[occ], kind='stable')
        out = {'keys': keys[occ][order]}
        for n, x in zip(('cooc', 'sr_w', 'sr_first'), self.t[1:]):
            out[n] = _host(x)[:self.cap][occ][order]
        return out

    def check(self, ref, err=0):
        got, want = self.export(), ref.export()
        for k in ('keys', 'cooc', 'sr_w', 'sr_first'):
            np.testing.assert_array_equal(got[k], want[k], err_msg=k)
        assert _host(self.count)[0] == want['keys'].size
        assert _host(self.err)[0] == err
        self.check_guards()

    def check_guards(self):
        _guards(*[(x, self.cap, SENT64) for x in self.t], (self.count, 1, SENT64), (self.err, 1, SENT32))

    def untouched(self, cleared=True):
        """the table as a fresh one: cleared (or sentinel everywhere), no count, no error"""
        if cleared:
            assert (_host(self.t[0])[:self.cap] == -1).all() and not _host(self.t[1])[:self.cap].any()
            assert not _host(self.t[2])[:self.cap].any() and (_host(self.t[3])[:self.cap] == BIG).all()
        else:
            for x in self.t:
                assert (_host(x)[:self.cap] == SENT64).all()
        assert _host(self.count)[0] == 0 and _host(self.err)[0] == 0
        self.check_guards()


def _cap_for(batches):
    """a power of two at least twice the keys the batches can create (pairs of the distinct ids of each row)"""
    bound = sum(len(set(r[r != 0].tolist())) ** 2 for ai in batches for r in np.asarray(ai))
    return max(16, 1 << (2 * max(bound, 1) - 1).bit_length())


def _rows(rs, B, T1, lo, V, min_len=1, gaps=0.0):
    ai = np.zeros((B, T1), dtype=np.int64)
    for b in range(B):
        n = int(rs.randint(min_len, T1 + 1))
        ai[b, :n] = rs.randint(lo, lo + V, size=n)
        if gaps:
            ai[b, :n][rs.rand(n) < gaps] = 0                  # padding between clicks
    return ai


def _update_case(name):
    """-> (batches, num_items, max_clicks_dist, first batch_seq)"""
    rs = np.random.RandomState(sum(map(ord, name)))
    if name == 't1_1':
        return [_rows(rs, 7, 1, 1, 9) for _ in range(3)], 10, 10, 0
    if name == 't1_2':
        return [_rows(rs, 40, 2, 1, 12) for _ in range(3)], 13, 10, 0
    if name == 't1_33':
        return [_rows(rs, 30, 33, 1, 50, gaps=0.1) for _ in range(3)], 51, 10, 0
    if name == 't1_1024':
        ai = np.zeros((4, 1024), dtype=np.int64)
        ai[0] = rs.randint(1, 40, size=1024)                  # every position, 39 ids
        ai[1] = 17                                             # one id 1024 times
        ai[2, :700] = rs.randint(100, 130, size=700)
        ai[2, rs.rand(1024) < 0.2] = 0                         # padding between clicks
        ai[3, 1023] = 5                                        # one click at the last position
        return [ai], 200, 20, 0
    if name == 'repeats':
        ai = np.zeros((7, 9), dtype=np.int64)
        ai[0, :6] = 3                                          # one distinct id
        ai[1, :7] = [4, 5, 4, 5, 4, 4, 5]                      # repeated ids: the s_next canonical pair
        ai[2, 0] = 7                                           # a single click
        ai[4, :5] = [9, 0, 9, 0, 2]                            # padding between clicks; row 3 all padding
        ai[5, :] = [2, 9, 2, 9, 2, 9, 2, 9, 2]
        ai[6, :4] = [1, 1, 2, 1]
        return [ai, ai[::-1].copy(), ai], 10, 10, 0
    if name.startswith('dist_'):
        return [_rows(rs, 20, 25, 1, 30) for _ in range(3)], 31, int(name[5:]), 0
    if name == 'seq_max':
        return [_rows(rs, 10, 8, 1, 20) for _ in range(2)], 21, 10, MAX_ID - 1
    if name == 'big_ids':
        batches = []
        for _ in range(3):
            ai = _rows(rs, 12, 10, 100, 300)                   # ids in the hundreds
            big = (ai % 3 == 0) & (ai != 0)
            ai[big] = MAX_ID - 1 - (ai[big] % 7)               # and ids near 2^31 - 1
            batches.append(ai)
        return batches, MAX_ID, 10, 0
    raise KeyError(name)


UPDATE_CASES = ['t1_1', 't1_2', 't1_33', 't1_1024', 'repeats', 'dist_1', 'dist_2', 'dist_7', 'dist_20', 'seq_max',
                'big_ids']


@gpu
@pytest.mark.parametrize('name', UPDATE_CASES)
def test_pair_table_update(name):
    """nar_baselines_update against BaselinesRef.update batch by batch: keys, cooc, sr_w and sr_first (whose high word is
    batch_seq), the occupancy counter, no error, guards."""
    batches, num_items, D, seq0 = _update_case(name)
    tab = Table(_cap_for(batches))
    ref = BaselinesRef(num_items, max_clicks_dist=D)
    ref.batch_seq = seq0
    for i, ai in enumerate(batches):
        assert tab.update(ai, num_items, D, seq0 + i) == 0
        ref.update(ai)
        tab.check(ref)
    if name != 't1_1':
        assert ref.sr_w and ref.cooc


def _wrap_pair(cap=16):
    """ids a != c whose keys (a, c) and (c, a) both hash to the last slot"""
    for a in range(1, 400):
        for c in range(a + 1, 400):
            if mix64((a << 32) | c) & (cap - 1) == cap - 1 and mix64((c << 32) | a) & (cap - 1) == cap - 1:
                return a, c
    raise AssertionError('no pair')


@gpu
def test_pair_table_probe_wraps():
    """Two keys hash to the last slot of a 16-slot table: the second one wraps to slot 0, and scoring finds both."""
    a, c = _wrap_pair()
    tab = Table(16)
    ref = BaselinesRef(400)
    ai = np.array([[a, c]], dtype=np.int64)
    assert tab.update(ai, 400) == 0
    ref.update(ai)
    tab.check(ref)
    keys = _host(tab.t[0])
    assert {int(keys[15]), int(keys[0])} == {(a << 32) | c, (c << 32) | a}
    ic = np.array([[a, c]], dtype=np.int64)
    ln = np.array([[c, a]], dtype=np.int64)
    neg = np.array([[[a, 3], [c, 3]]], dtype=np.int64)
    w = _world_from(tab, ref, 400, buf=np.zeros(1, np.int64), pop=None, acr=None)
    _score_and_check(w, ic, ln, neg, 2 | 16, 2)


@gpu
def test_pair_table_overflow():
    """A 16-slot table offered 56 cooc pairs: err = 2, exactly 16 keys of the session's pairs, nothing past cap; the
    wrapper, told the batch has no pairs, does not grow and raises."""
    ai = np.arange(1, 9, dtype=np.int64).reshape(1, 8)
    tab = Table(16)
    assert tab.update(ai, 20) == 0
    keys = _host(tab.t[0])[:16]
    pairs = {(a << 32) | c for a in range(1, 9) for c in range(1, 9) if a != c}
    assert (keys != -1).all() and set(keys.tolist()) <= pairs
    assert _host(tab.count)[0] == 16 and _host(tab.err)[0] == 2
    tab.check_guards()
    from chameleon_recsys_b200.baselines import BaselineTables
    bt = BaselineTables(['coocurrent'], 20, capacity=16)
    bt.update(_dev(ai), lens=[1])
    with pytest.raises(RuntimeError, match='overflow'):
        bt.check_errors()
    assert bt.cap == 16


REJECT_UPDATE = [
    ('t1_1025', dict(T1=1025), NAR_ERR_UNSUPPORTED),
    ('dist_21', dict(D=21), NAR_ERR_UNSUPPORTED),
    ('dist_0', dict(D=0), NAR_ERR_UNSUPPORTED),
    ('seq_2_31', dict(seq=1 << 31), NAR_ERR_INVALID),
    ('seq_neg', dict(seq=-1), NAR_ERR_INVALID),
    ('items_2_31', dict(num_items=1 << 31), NAR_ERR_INVALID),
    ('items_0', dict(num_items=0), NAR_ERR_INVALID),
    ('cap_24', dict(cap=24), NAR_ERR_INVALID),
    ('bg_neg', dict(Bg=-1), NAR_ERR_INVALID),
    ('t1_0', dict(T1=0), NAR_ERR_INVALID),
    ('bg_t1_t1', dict(Bg=4097, T1=1024), NAR_ERR_UNSUPPORTED),
    ('null_items', dict(null=True), NAR_ERR_INVALID),
]


@gpu
@pytest.mark.parametrize('name,kw,rc', REJECT_UPDATE, ids=[r[0] for r in REJECT_UPDATE])
def test_pair_table_update_rejects(name, kw, rc):
    T1, Bg = kw.get('T1', 4), kw.get('Bg', 2)
    ai = np.ones((max(Bg, 1), max(T1, 1)), dtype=np.int64)    # every row the call could read exists
    ai[:, ::2] = 2
    tab = Table(kw.get('cap', 16), clear='cap' not in kw)
    d = None if kw.get('null') else _dev(ai)
    got = _lib().nar_baselines_update(*tab.ptrs(), tab.cap, _p(tab.count), _p(d), Bg, T1, kw.get('num_items', 10),
                                      kw.get('D', 10), kw.get('seq', 0), _p(tab.err), _s())
    assert got == rc
    tab.untouched(cleared='cap' not in kw)


@gpu
def test_pair_table_empty_batch():
    tab = Table(16)
    assert tab.update(np.zeros((0, 5), np.int64), 10) == 0
    tab.untouched()


@gpu
def test_pair_table_growth_every_batch():
    """BaselineTables from capacity 16, every batch forcing a rehash: the export equals the oracle after each batch; a
    snapshot before two growths restores the old capacity and tables, and training continues from there."""
    from chameleon_recsys_b200.baselines import BaselineTables
    rs = np.random.RandomState(5)
    V = 400
    tab = BaselineTables(['coocurrent', 'sr'], V, capacity=16)
    ref = BaselinesRef(V)
    caps = [tab.cap]

    def batch(B, T1):
        return np.stack([rs.choice(np.arange(1, V), T1, replace=False) for _ in range(B)]).astype(np.int64)
    for i, (B, T1) in enumerate([(1, 5), (1, 7), (2, 7), (4, 7), (8, 7), (16, 7)]):
        ai = batch(B, T1)
        tab.update(_dev(ai))
        ref.update(ai)
        caps.append(tab.cap)
        got, want = tab.export(), ref.export()
        for k in ('keys', 'cooc', 'sr_w', 'sr_first'):
            np.testing.assert_array_equal(got[k], want[k], err_msg=k)
        if i == 2:
            tab.snapshot()
            ref.snapshot()
            snap = (tab.cap, want)
    assert all(b > a for a, b in zip(caps, caps[1:])), caps
    tab.restore()
    ref.restore()
    assert tab.cap == snap[0]
    got = tab.export()
    for k in ('keys', 'cooc', 'sr_w', 'sr_first'):
        np.testing.assert_array_equal(got[k], snap[1][k], err_msg=k)
    ai = batch(16, 7)
    tab.update(_dev(ai))
    ref.update(ai)
    got, want = tab.export(), ref.export()
    for k in ('keys', 'cooc', 'sr_w', 'sr_first'):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


@gpu
@pytest.mark.parametrize('factor', [1, 2, 8])
def test_pair_table_rehash(factor):
    """nar_baselines_rehash into 1x, 2x and 8x the capacity: the same entries, the source untouched, guards kept."""
    rs = np.random.RandomState(factor)
    ai = _rows(rs, 6, 6, 1, 30, min_len=3)
    tab = Table(_cap_for([ai]))
    ref = BaselinesRef(31)
    assert tab.update(ai, 31) == 0
    ref.update(ai)
    before = tab.export()
    new = Table(tab.cap * factor, clear=False)
    assert _lib().nar_baselines_rehash(*tab.ptrs(), tab.cap, *new.ptrs(), new.cap, _p(new.err), _s()) == 0
    got = new.export()
    for k in before:
        np.testing.assert_array_equal(got[k], before[k], err_msg=k)
    tab.check(ref)
    new.check_guards()
    assert _host(new.err)[0] == 0
    for bad_cap in (tab.cap // 2, tab.cap * factor + 16):
        other = Table(bad_cap, clear=False)
        assert _lib().nar_baselines_rehash(*tab.ptrs(), tab.cap, *other.ptrs(), bad_cap, _p(other.err),
                                           _s()) == NAR_ERR_INVALID
        other.untouched(cleared=False)


def _ref_from(arrays, V):
    ref = BaselinesRef(V)
    for k, c, w, f in zip(*(arrays[n].tolist() for n in ('keys', 'cooc', 'sr_w', 'sr_first'))):
        pr = (k >> 32, k & 0xffffffff)
        if c:
            ref.cooc[pr] = c
        if w:
            ref.sr_w[pr] = w
        if f != BIG:
            ref.sr_first[pr] = f
    ref.batch_seq = int(arrays['batch_seq'])
    return ref


@gpu
@pytest.mark.parametrize('n', [0, 1, 2, 3, 15, 16, 17])
def test_pair_table_load(n):
    """BaselineTables.load of n exported entries (a dense table of n slots rehashed into max(16, 2n) rounded up), then
    one more batch: both against the oracle holding the same entries."""
    from chameleon_recsys_b200.baselines import BaselineTables
    rs = np.random.RandomState(n)
    V = 40
    full = BaselinesRef(V)
    full.update(_rows(rs, 8, 6, 1, V - 1, min_len=3))
    ex = full.export()
    pick = np.sort(rs.choice(ex['keys'].size, n, replace=False))
    arrays = {k: ex[k][pick] for k in ('keys', 'cooc', 'sr_w', 'sr_first')}
    arrays['batch_seq'] = np.asarray(3, dtype=np.int64)
    tab = BaselineTables(['coocurrent', 'sr'], V)
    tab.load(arrays)
    assert tab.cap == max(16, 1 << (max(1, 2 * n) - 1).bit_length())
    got = tab.export()
    for k in ('keys', 'cooc', 'sr_w', 'sr_first'):
        np.testing.assert_array_equal(got[k], arrays[k], err_msg=k)
    assert int(_host(tab.count)[0]) == n
    ref = _ref_from(arrays, V)
    ai = _rows(rs, 2, 4, 1, V - 1, min_len=2)
    tab.update(_dev(ai))
    ref.update(ai)
    got, want = tab.export(), ref.export()
    for k in ('keys', 'cooc', 'sr_w', 'sr_first'):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


# ------------------------------------------------------------------------------------------------ buffer_hist, row_norms
def _hist_call(buf, num_items, n=None):
    cnt = _full(num_items, SENT32, 'i32')
    first = _full(num_items, SENT32, 'i32')
    err = _scalar(0, 'i32')
    d = _dev(buf) if buf.size else _full(0, 0, 'i64')
    rc = _lib().nar_baselines_buffer_hist(_p(d), buf.size if n is None else n, num_items, _p(cnt), _p(first), _p(err),
                                          _s())
    return rc, cnt, first, err


@gpu
@pytest.mark.parametrize('case', ['mixed', 'empty', 'long'])
def test_buffer_hist(case):
    """count and first index of every id against a plain loop: padding, repeats, an id only at the last index, n = 0,
    and a buffer long enough for the grid-stride loop."""
    rs = np.random.RandomState(len(case))
    V = {'mixed': 100, 'empty': 50, 'long': 1000}[case]
    if case == 'empty':
        buf = np.zeros(0, dtype=np.int64)
    else:
        n = 500 if case == 'mixed' else 300000
        buf = rs.randint(1, V - 1, size=n).astype(np.int64)
        buf[rs.rand(n) < 0.2] = 0
        buf[:7] = 4                                            # repeats
        buf[n - 1] = V - 1                                     # an id only at the last index
    rc, cnt, first, err = _hist_call(buf, V)
    assert rc == 0
    want_c, want_f = hist_ref(buf, V)
    np.testing.assert_array_equal(_host(cnt)[:V], want_c)
    np.testing.assert_array_equal(_host(first)[:V], want_f)
    assert _host(err)[0] == 0
    _guards((cnt, V, SENT32), (first, V, SENT32), (err, 1, SENT32))


@gpu
def test_buffer_hist_errors():
    rc, cnt, first, err = _hist_call(np.array([3, 10, 2], dtype=np.int64), 10)
    assert rc == 0 and _host(err)[0] == 1
    assert _host(cnt)[[2, 3]].tolist() == [1, 1]
    rc, cnt, first, err = _hist_call(np.array([3, -4], dtype=np.int64), 10)
    assert rc == 0 and _host(err)[0] == 1


@gpu
@pytest.mark.parametrize('n,V', [(-1, 10), (3, 0)])
def test_buffer_hist_rejects(n, V):
    """Rejected before the tables are reset: count, first and err untouched."""
    cnt, first, err = _full(10, SENT32, 'i32'), _full(10, SENT32, 'i32'), _scalar(0, 'i32')
    d = _dev(np.array([3, 4, 5], np.int64))
    assert _lib().nar_baselines_buffer_hist(_p(d), n, V, _p(cnt), _p(first), _p(err), _s()) == NAR_ERR_INVALID
    assert (_host(cnt) == SENT32).all() and (_host(first) == SENT32).all() and _host(err)[0] == 0


@gpu
@pytest.mark.parametrize('dim,ld,V', [(1, 4, 37), (31, 33, 37), (32, 40, 37), (33, 35, 9000), (250, 256, 37)])
def test_row_norms(dim, ld, V):
    """fp64 norms bit for bit against the kernel's lane order, and within (dim/32 + 7) ulp of a numpy fp64 norm; rows past
    dim and the guard untouched.  V = 9000 runs the grid-stride loop."""
    rs = np.random.RandomState(dim)
    acr = (rs.randn(V, ld) * 10.0 ** rs.uniform(-3, 3, size=(V, 1))).astype(np.float32)
    acr[0, :dim] = 0.0
    acr[1, :dim] = np.float32(1e-40)                          # subnormal float32
    norms = _full(V, SENTF, 'f64')
    assert _lib().nar_baselines_row_norms(_p(_dev(acr)), V, dim, ld, _p(norms), _s()) == 0
    got = _host(norms)
    np.testing.assert_array_equal(got[:V], lane_norms(acr, dim))
    assert (got[V:] == SENTF).all()
    ref = np.linalg.norm(acr[:, :dim].astype(np.float64), axis=1)
    assert np.all(np.abs(got[:V] - ref) <= (dim / 32 + 7) * np.spacing(ref))


@gpu
@pytest.mark.parametrize('V,dim,ld', [(0, 4, 4), (5, 0, 4), (5, 4, 3)])
def test_row_norms_rejects(V, dim, ld):
    acr = _dev(np.ones((5, 4), np.float32))
    norms = _full(5, SENTF, 'f64')
    assert _lib().nar_baselines_row_norms(_p(acr), V, dim, ld, _p(norms), _s()) == NAR_ERR_INVALID
    assert (_host(norms) == SENTF).all()


# ------------------------------------------------------------------------------------------------ baseline scoring
class World:
    pass


def _world_from(tab, ref, num_items, buf, pop, acr, dim=0):
    w = World()
    w.tab, w.ref, w.num_items, w.buf, w.pop, w.acr, w.dim = tab, ref, num_items, buf, pop, acr, dim
    return w


def _world(seed, V=48, absent=5, n_train=4, B=16, T1=8, acr='int', dim=24, ld=32, ties=False, D=10):
    """A pair table and oracle trained on ids [1, V - absent) (the last ``absent`` ids are never clicked), a recent-clicks
    buffer, popularity counts and ACR rows."""
    rs = np.random.RandomState(seed)
    lo_hi = V - absent - 1
    if ties:
        batches = [_rows(rs, 3 * B, 3, 1, lo_hi, min_len=2) for _ in range(n_train)]
        buf = rs.permutation(np.arange(1, V - absent)).astype(np.int64)        # every id once: all counts tie
        pop = rs.randint(0, 3, size=V).astype(np.int64)
    else:
        batches = [_rows(rs, B, T1, 1, lo_hi, min_len=2) for _ in range(n_train)]
        buf = np.where(rs.rand(4 * B) < 0.8, rs.randint(1, V - absent, size=4 * B), 0).astype(np.int64)
        pop = rs.randint(0, 50, size=V).astype(np.int64)
    tab = Table(_cap_for(batches))
    ref = BaselinesRef(V, max_clicks_dist=D)
    for i, ai in enumerate(batches):
        assert tab.update(ai, V, D, i) == 0
        ref.update(ai)
    if acr == 'int':
        a = _int_acr(rs, V, dim, ld)
    else:
        a = np.zeros((V, ld), dtype=np.float32)
        a[:, :dim] = rs.randn(V, dim)
    ref.acr = a[:, :dim].astype(np.float64)
    return _world_from(tab, ref, V, buf, pop, a, dim)


def _queries(seed, w, B, T, K, label_p=0.9, lo=1, hi=None):
    """item_clicked / label_next [B, T] and negatives [B, T, K]: labels partly partners of the item in the table, partly
    random (some never clicked), negatives with padding, repeats of the label and duplicates."""
    rs = np.random.RandomState(seed)
    hi = w.num_items if hi is None else hi
    ic = rs.randint(lo, hi - 5, size=(B, T)).astype(np.int64)
    ln = rs.randint(lo, hi, size=(B, T)).astype(np.int64)
    partners = {}
    for (a, c) in w.ref.cooc:
        partners.setdefault(a, []).append(c)
    for b in range(B):
        for t in range(T):
            p = partners.get(int(ic[b, t]))
            if p and rs.rand() < 0.5:
                ln[b, t] = p[rs.randint(len(p))]
    ln[rs.rand(B, T) > label_p] = 0
    neg = rs.randint(lo, hi - 5, size=(B, T, K)).astype(np.int64)
    if K:
        neg[rs.rand(B, T, K) < 0.1] = 0
        lab = rs.rand(B, T, K) < 0.05
        neg[lab] = np.broadcast_to(ln[:, :, None], neg.shape)[lab]
        neg[:, :, -1] = neg[:, :, 0]                           # a duplicate negative
    return ic, ln, neg


def _bl_call(w, ic, ln, neg, enabled, top_n, lam=20.0, alpha=0.75, with_out=True, K=None, B=None, T=None,
             cap=None, null=()):
    """-> rc, out [5, nq, top_n], rank_hist [5, top_n + 1], metrics [5, 3], err"""
    lib = _lib()
    Bq, Tq = ic.shape
    B = Bq if B is None else B
    T = Tq if T is None else T
    K = neg.shape[2] if K is None else K
    nq = Bq * Tq
    V = w.num_items
    per_item = V < (1 << 24)
    cnt = first = pop = acr = norms = None
    if per_item and w.buf is not None:
        cnt, first = _full(V, SENT32, 'i32'), _full(V, SENT32, 'i32')
        herr = _scalar(0, 'i32')
        bd = _dev(w.buf)
        assert lib.nar_baselines_buffer_hist(_p(bd), w.buf.size, V, _p(cnt), _p(first), _p(herr), _s()) == 0
    if per_item and w.pop is not None:
        pop = _dev(w.pop)
    if per_item and w.acr is not None:
        acr = _dev(w.acr)
        norms = _full(V, SENTF, 'f64')
        assert lib.nar_baselines_row_norms(_p(acr), V, w.dim, w.acr.shape[1], _p(norms), _s()) == 0
    hist = _full(5 * (top_n + 1), SENT64, 'i64')
    met = _prefilled(PRE5)
    out = _full(5 * nq * top_n, SENT64, 'i64') if with_out else None
    err = _scalar(0, 'i32')
    icd, lnd = _dev(ic), _dev(ln)
    ngd = _dev(neg) if neg.size else None
    tabs = [None] * 4 if 'table' in null else w.tab.t
    args = dict(cnt=cnt, first=first, pop=pop, acr=acr, norms=norms)
    for k in null:
        args[k] = None
    rc = lib.nar_baselines_score(*[_p(x) for x in tabs], w.tab.cap if cap is None else cap, _p(icd), _p(lnd), _p(ngd),
                                 B, T, K, _p(args['cnt']), _p(args['first']), _p(args['pop']), _p(args['acr']), w.dim,
                                 0 if w.acr is None else w.acr.shape[1], _p(args['norms']), V, lam, alpha, enabled,
                                 top_n, _p(hist), _p(met), _p(out), _p(err), _s())
    _guards((hist, 5 * (top_n + 1), SENT64), (met, 15, SENTF), (err, 1, SENT32))
    if with_out:
        _guards((out, 5 * nq * top_n, SENT64))
    h = _host(hist)[:5 * (top_n + 1)].reshape(5, top_n + 1)
    o = _host(out)[:5 * nq * top_n].reshape(5, nq, top_n) if with_out else None
    return rc, o, h, _host(met)[:15].reshape(5, 3), int(_host(err)[0])


def _oracle(w, ic, ln, neg, enabled, top_n, lam=20.0, alpha=0.75):
    w.ref.reg_lambda, w.ref.alpha = lam, alpha
    sfx = [s for i, s in enumerate(SUFFIXES) if enabled >> i & 1]
    return w.ref.score(ic, ln, neg, w.buf, w.pop, top_n, suffixes=sfx)


def _check_scores(got, want, ln, enabled, top_n, rows=None):
    rc, out, hist, met, err = got
    assert rc == 0 and err == 0
    act = ln.reshape(-1) != 0
    for i, sfx in enumerate(SUFFIXES):
        if not enabled >> i & 1:
            assert hist[i].tolist() == [0] * (top_n + 1), sfx
            assert met[i].tolist() == PRE5[3 * i:3 * i + 3].tolist(), sfx
            if out is not None:
                assert (out[i] == SENT64).all(), sfx
            continue
        wv = want[sfx]
        if rows is None or i not in rows:
            np.testing.assert_array_equal(hist[i], wv['hist'], err_msg=sfx)
            assert met[i].tolist() == [PRE5[3 * i] + wv['hits'], PRE5[3 * i + 1] + wv['rr'],
                                       PRE5[3 * i + 2] + wv['count']], sfx
            if out is not None:
                np.testing.assert_array_equal(out[i][act], wv['ids'][act], err_msg=sfx)
        else:
            assert hist[i][top_n] == wv['hist'][top_n] and met[i][2] == PRE5[3 * i + 2] + wv['count'], sfx
            if out is not None:
                np.testing.assert_array_equal(out[i][rows[i]], wv['ids'][rows[i]], err_msg=sfx)
        if out is not None:
            assert (out[i][~act] == SENT64).all(), sfx


def _score_and_check(w, ic, ln, neg, enabled, top_n, lam=20.0, alpha=1.0, with_out=True):
    got = _bl_call(w, ic, ln, neg, enabled, top_n, lam, alpha, with_out)
    want = _oracle(w, ic, ln, neg, enabled, top_n, lam, alpha)
    _check_scores(got, want, ln, enabled, top_n)
    return got, want


@gpu
@pytest.mark.parametrize('enabled', range(32))
def test_score_enabled_masks(enabled):
    """Every subset of the five baselines at a small shape: enabled rows equal the oracle (ids, rank histogram, metrics
    grown by exactly its sums), disabled rows untouched.  Integer ACR rows and alpha 1: every score is exact."""
    w = _world(enabled)
    ic, ln, neg = _queries(enabled, w, 5, 6, 9)
    _score_and_check(w, ic, ln, neg, enabled, 5)


@gpu
def test_score_ties():
    """Sessions of two or three clicks and a buffer holding every id once: pop_recent counts all tie (first buffer index
    decides), cooc / item_knn scores tie (the higher id first), sr weights tie (sr_first decides)."""
    w = _world(11, V=40, ties=True)
    ic, ln, neg = _queries(11, w, 12, 6, 20)
    got, want = _score_and_check(w, ic, ln, neg, 31, 10)
    ids = want['pop_recent']['ids']
    assert (ids[:, 1:] != 0).any()
    for sfx in ('coocurrent', 'sr'):
        tie = 0
        for q in np.flatnonzero(ln.reshape(-1)):
            item = int(ic.reshape(-1)[q])
            sc = w.ref.candidate_scores(sfx, item, [ln.reshape(-1)[q]] + neg.reshape(-1, 20)[q].tolist(), w.buf, w.pop)
            v = sorted(sc.values())
            tie += any(a == b for a, b in zip(v, v[1:]))
        assert tie > 10, sfx


SHAPES = [  # (K, top_n, B, T)
    (0, 1, 6, 5), (1, 3, 6, 5), (31, 32, 4, 5), (32, 33, 4, 5), (40, 64, 3, 4), (50, 33, 3, 3), (1023, 10, 2, 2),
]


@gpu
@pytest.mark.parametrize('K,top_n,B,T', SHAPES)
def test_score_shapes(K, top_n, B, T):
    """K = 0 .. 1023 and top_n 1, 32, 33, 64 (larger than the admissible count: 0-padded), all five baselines."""
    w = _world(K + top_n, V=1100 if K == 1023 else 80, T1=12, B=40)
    ic, ln, neg = _queries(K, w, B, T, K)
    got, want = _score_and_check(w, ic, ln, neg, 31, top_n)
    if K >= 40 and top_n > 32:
        assert (want['cb']['ids'][:, 32:] != 0).any()              # ranks past the first 32 lanes
    if top_n > K + 1:
        assert (want['cb']['ids'][:, K + 1:] == 0).all()            # more slots than candidates: 0-padded


@gpu
@pytest.mark.parametrize('K,B,T,enabled', [(3, 850, 20, 2 | 16), (1023, 2200, 1, 2)], ids=['8warps', '1warp'])
def test_score_grid_stride(K, B, T, enabled):
    """More queries than the capped grid holds warps (16 x 132 CTAs of 8 warps at K = 3, of 1 warp at K = 1023): the
    queries past the first stride carry labels, as do a sparse set before it."""
    w = _world(K, V=1100 if K == 1023 else 60, B=40, T1=10)
    ic, ln, neg = _queries(K, w, B, T, K, label_p=1.0)
    nq = B * T
    warps = 8 if K == 3 else 1
    first_stride = 16 * 132 * warps
    assert nq > first_stride
    q = np.arange(nq)
    ln.reshape(-1)[(q % 53 != 0) & (q < first_stride - 20)] = 0
    assert (ln.reshape(-1)[first_stride:] != 0).all()
    _score_and_check(w, ic, ln, neg, enabled, 5)


@gpu
@pytest.mark.parametrize('alpha,lam', [(0.0, 20.0), (1.0, 20.0), (0.0, 0.5), (1.0, 3.0)])
def test_score_item_knn_exact(alpha, lam):
    """item_knn at alpha 0 and 1 (pow(x, 0) = 1 and pow(x, 1) = x on both sides) and reg_lambda other than 20."""
    w = _world(int(alpha * 10 + lam), V=60)
    ic, ln, neg = _queries(3, w, 8, 6, 24)
    _score_and_check(w, ic, ln, neg, 4, 10, lam, alpha)


@gpu
@pytest.mark.parametrize('alpha', [0.5, 0.75])
def test_score_item_knn_gap(alpha):
    """item_knn at alpha 0.5 and 0.75: ids compared on the queries whose oracle score gaps all exceed 8 ulp (most of
    them); the query count exactly."""
    w = _world(int(alpha * 100), V=60)
    ic, ln, neg = _queries(4, w, 10, 8, 24)
    rows = []
    for q in np.flatnonzero(ln.reshape(-1)):
        item = int(ic.reshape(-1)[q])
        cands = [ln.reshape(-1)[q]] + neg.reshape(-1, 24)[q].tolist()
        if knn_gap_ok(w.pop, 20.0, alpha, item, cands, w.ref.cooc):
            rows.append(q)
    assert len(rows) >= 0.8 * np.count_nonzero(ln)
    got = _bl_call(w, ic, ln, neg, 4, 10, 20.0, alpha)
    want = _oracle(w, ic, ln, neg, 4, 10, 20.0, alpha)
    _check_scores(got, want, ln, 4, 10, rows={2: np.array(rows)})


@gpu
def test_score_cb_random_floats():
    """cb on random float ACR rows: ids equal except on queries where two candidates' cosines lie within 1e-12
    relative; the query count exactly."""
    w = _world(21, V=200, acr='float', dim=40, ld=48)
    ic, ln, neg = _queries(21, w, 12, 8, 30)
    rows = []
    for q in np.flatnonzero(ln.reshape(-1)):
        sc = w.ref.candidate_scores('cb', ic.reshape(-1)[q], [ln.reshape(-1)[q]] + neg.reshape(-1, 30)[q].tolist(),
                                    w.buf, w.pop)
        v = np.sort(np.array(list(sc.values())))
        if not np.any(np.diff(v) <= 1e-12 * np.maximum(np.abs(v[1:]), np.abs(v[:-1]))):
            rows.append(q)
    assert len(rows) >= 0.9 * np.count_nonzero(ln)
    got = _bl_call(w, ic, ln, neg, 8, 10)
    want = _oracle(w, ic, ln, neg, 8, 10)
    _check_scores(got, want, ln, 8, 10, rows={3: np.array(rows)})


@gpu
def test_score_big_ids():
    """Ids in the hundreds and near 2^31 - 1 with num_items = 2^31 - 1: coocurrent and sr (the per-item tables of the
    other baselines are not allocated)."""
    batches, V, D, _ = _update_case('big_ids')
    tab = Table(_cap_for(batches))
    ref = BaselinesRef(V, max_clicks_dist=D)
    for i, ai in enumerate(batches):
        assert tab.update(ai, V, D, i) == 0
        ref.update(ai)
    w = _world_from(tab, ref, V, np.zeros(0, np.int64), None, None)
    rs = np.random.RandomState(9)
    ids = np.unique(np.concatenate(batches))
    ids = ids[ids != 0]
    ic = rs.choice(ids, size=(6, 5)).astype(np.int64)
    ln = rs.choice(ids, size=(6, 5)).astype(np.int64)
    neg = rs.choice(ids, size=(6, 5, 20)).astype(np.int64)
    _score_and_check(w, ic, ln, neg, 2 | 16, 8)
    assert (ic >= MAX_ID - 7).any() and (neg >= MAX_ID - 7).any()


@gpu
def test_score_without_out_ids():
    w = _world(31)
    ic, ln, neg = _queries(31, w, 6, 5, 9)
    _score_and_check(w, ic, ln, neg, 31, 5, with_out=False)


@gpu
@pytest.mark.parametrize('where', ['negative', 'label', 'item', 'item_zero'])
def test_score_bad_ids_set_err(where):
    """An id outside [0, num_items) among the negatives, as a label or as the current click (and a click 0 under a label)
    sets err = 1."""
    w = _world(41)
    ic, ln, neg = _queries(41, w, 4, 5, 9, label_p=1.0)
    if where == 'negative':
        neg[1, 2, 3] = w.num_items
        neg[2, 1, 0] = -3
    elif where == 'label':
        ln[0, 0] = w.num_items + 7
    elif where == 'item':
        ic[3, 4] = w.num_items
    else:
        ic[3, 4] = 0
    rc, out, hist, met, err = _bl_call(w, ic, ln, neg, 31, 5)
    assert rc == 0 and err == 1


REJECT_SCORE = [
    ('k_1024', dict(K=1024), NAR_ERR_UNSUPPORTED),
    ('top_n_0', dict(top_n=0), NAR_ERR_INVALID),
    ('enabled_32', dict(enabled=32), NAR_ERR_INVALID),
    ('t_0', dict(T=0), NAR_ERR_INVALID),
    ('b_neg', dict(B=-1), NAR_ERR_INVALID),
    ('k_neg', dict(K=-1), NAR_ERR_INVALID),
    ('cap_24', dict(cap=24), NAR_ERR_INVALID),
    ('null_table', dict(null=('table',)), NAR_ERR_INVALID),
    ('null_hist', dict(null=('cnt',)), NAR_ERR_INVALID),
    ('null_pop', dict(null=('pop',)), NAR_ERR_INVALID),
    ('null_norms', dict(null=('norms',)), NAR_ERR_INVALID),
    ('null_negatives', dict(null_neg=True), NAR_ERR_INVALID),
]


@gpu
@pytest.mark.parametrize('name,kw,rc', REJECT_SCORE, ids=[r[0] for r in REJECT_SCORE])
def test_score_rejects(name, kw, rc):
    """Rejected before any launch: rank_hist, metrics, out_ids and err untouched."""
    w = _world(51)
    ic, ln, neg = _queries(51, w, 2, 3, 1024 if name == 'k_1024' else 5)
    if kw.get('null_neg'):
        neg = np.zeros((2, 3, 0), dtype=np.int64)
        kw = dict(K=5)
    got_rc, out, hist, met, err = _bl_call(w, ic, ln, neg, kw.get('enabled', 31), kw.get('top_n', 5), K=kw.get('K'),
                                           B=kw.get('B'), T=kw.get('T'), cap=kw.get('cap'), null=kw.get('null', ()))
    assert got_rc == rc
    assert (hist == SENT64).all() and met.reshape(-1).tolist() == PRE5.tolist() and err == 0
    assert (out == SENT64).all()


@gpu
def test_score_enabled_zero():
    """enabled = 0: rank_hist zeroed, nothing else written."""
    w = _world(61)
    ic, ln, neg = _queries(61, w, 3, 4, 6)
    got = _bl_call(w, ic, ln, neg, 0, 4)
    _check_scores(got, {}, ln, 0, 4)


# ------------------------------------------------------------------------------------------------ session-kNN ring
class Ring:
    """A raw V-SkNN / SkNN ring of S slots of width W and its staging scratch, each with guard space; head and count
    kept here as SessionKNN keeps them."""

    def __init__(self, S, num_items, W=WIDTH):
        self.S, self.W, self.num_items = S, W, num_items
        self.ids, self.st_ids = _full(S, SENT64, 'i64'), _full(S, SENT64, 'i64')
        self.lens, self.st_lens = _full(S, SENT32, 'i32'), _full(S, SENT32, 'i32')
        self.items, self.st_items = _full(S * W, SENT32, 'i32'), _full(S * W, SENT32, 'i32')
        self.err = _scalar(0, 'i32')
        self.head = self.count = 0

    def tensors(self):
        return [self.ids, self.lens, self.items, self.st_ids, self.st_lens, self.st_items]

    def update(self, sids, ai, B=None, T1=None, W=None, head=None, count=None, num_items=None):
        ai = np.asarray(ai, dtype=np.int64)
        sids = np.asarray(sids, dtype=np.int64)
        B = ai.shape[0] if B is None else B
        T1 = ai.shape[1] if T1 is None else T1
        t = self.tensors()
        ad = _dev(ai) if ai.size else None
        sd = _dev(sids) if sids.size else None
        rc = _lib().nar_sknn_update(*[_p(x) for x in t[:3]], self.S, self.W if W is None else W,
                                    self.head if head is None else head, self.count if count is None else count,
                                    *[_p(x) for x in t[3:]], _p(ad), _p(sd), B, T1,
                                    self.num_items if num_items is None else num_items, _p(self.err), _s())
        if rc == 0:
            ev = max(0, self.count + B - self.S)
            self.head = (self.head + ev) % self.S
            self.count += B - ev
        return rc

    def export(self):
        idx = (self.head + np.arange(self.count)) % self.S
        items = _host(self.items)[:self.S * self.W].reshape(self.S, self.W)[idx].astype(np.int64)
        return {'ids': _host(self.ids)[idx], 'lens': _host(self.lens)[idx].astype(np.int64), 'items': np.abs(items),
                'live': items > 0}

    def check(self, ref, err=0):
        got, want = self.export(), ref.export()
        np.testing.assert_array_equal(got['ids'], want['ids'])
        np.testing.assert_array_equal(got['lens'], want['lens'])
        W = want['items'].shape[1]
        np.testing.assert_array_equal(got['items'][:, :W], want['items'])
        assert not got['items'][:, W:].any()
        np.testing.assert_array_equal(got['live'][:, :W], want['live'])
        assert _host(self.err)[0] == err
        self.check_guards()

    def check_guards(self):
        S, W = self.S, self.W
        _guards((self.ids, S, SENT64), (self.st_ids, S, SENT64), (self.lens, S, SENT32), (self.st_lens, S, SENT32),
                (self.items, S * W, SENT32), (self.st_items, S * W, SENT32), (self.err, 1, SENT32))

    def untouched(self):
        for x, v in zip(self.tensors(), (SENT64, SENT32, SENT32) * 2):
            assert (_host(x) == v).all()
        assert _host(self.err)[0] == 0

    def score(self, ic, ln, neg, sample, nn, decay_div, jaccard, top_n, with_out=True, **over):
        """``over``: arguments passed in place of the ring's and the inputs' own (``top_n_arg``: the top_n passed, the
        outputs sized for ``top_n``)"""
        B, T = ic.shape
        K = neg.shape[2]
        nq = B * T
        hist = _full(top_n + 1, SENT64, 'i64')
        met = _prefilled(PRE3)
        out = _full(nq * top_n, SENT64, 'i64') if with_out else None
        err = _scalar(0, 'i32')
        o = dict(S=self.S, W=self.W, head=self.head, count=self.count, B=B, T=T, K=K, num_items=self.num_items,
                 sample=sample, nn=nn, top_n_arg=top_n)
        o.update(over)
        icd, lnd = _dev(ic), _dev(ln)
        ngd = _dev(neg) if neg.size else None
        rc = _lib().nar_sknn_score(_p(self.ids), _p(self.lens), _p(self.items), o['S'], o['W'], o['head'], o['count'],
                                   _p(icd), _p(lnd), _p(ngd), o['B'], o['T'], o['K'], o['num_items'], o['sample'],
                                   o['nn'], decay_div, jaccard, o['top_n_arg'], _p(hist), _p(met), _p(out), _p(err),
                                   _s())
        _guards((hist, top_n + 1, SENT64), (met, 3, SENTF), (err, 1, SENT32))
        if with_out:
            _guards((out, nq * top_n, SENT64))
        return (rc, _host(out)[:nq * top_n].reshape(nq, top_n) if with_out else None, _host(hist)[:top_n + 1],
                _host(met)[:3], int(_host(err)[0]))


def _revived(before, after, B):
    """(session id, item) pairs dead in some entry before a batch and live in an entry that was already there after it"""
    dead = {(int(s), int(x)) for s, it, lv in zip(before['ids'], before['items'], before['live'])
            for x, l in zip(it, lv) if x and not l}
    n_old = len(after['ids']) - B
    live = {(int(s), int(x)) for s, it, lv in zip(after['ids'][:n_old], after['items'][:n_old], after['live'][:n_old])
            for x, l in zip(it, lv) if x and l}
    return dead & live


def _ring_batches(name):
    """-> (S, T1, num_items, [(session ids, all_items)], must revive)"""
    rs = np.random.RandomState(sum(map(ord, name)))

    def one(seq, T1=1):
        out = []
        for batch in seq:
            ai = np.zeros((len(batch), T1), dtype=np.int64)
            for b, (_, items) in enumerate(batch):
                ai[b, :len(items)] = items
            out.append((np.array([s for s, _ in batch], dtype=np.int64), ai))
        return out
    if name == 'returning':
        return 4, 1, 10, one([[r] for r in RETURNING] + [[(9, [2])], [(5, [1])], [(10, [1])]]), True
    if name == 'returning_partial':
        seq = [(5, [1, 3]), (6, [1]), (5, [1, 3]), (7, [3]), (8, [1]), (5, [1, 2]), (11, [4]), (5, [3])]
        return 4, 2, 10, one([[r] for r in seq], 2), True
    if name == 'returning_batches':
        seq = [[(5, [1]), (6, [2])], [(7, [3]), (5, [1])], [(8, [4]), (9, [5])], [(5, [1])], [(5, [1]), (5, [2])],
               [(12, [1])]]
        return 4, 1, 10, one(seq), True
    if name == 'twins_random':
        out = []
        for step in range(40):
            B = int(rs.randint(1, 4))
            sids = rs.randint(1, 4, size=B).astype(np.int64)   # three ids: twins within and across batches
            out.append((sids, _rows(rs, B, 3, 1, 4)))
        return 5, 3, 6, out, True
    if name in ('s1', 's2', 's17', 's17_full', 's4096'):
        S = {'s1': 1, 's2': 2, 's17': 17, 's17_full': 17, 's4096': 4096}[name]
        Bs = {'s1': [1] * 6, 's2': [1, 2, 1, 2, 2, 1], 's17': [5] * 9, 's17_full': [17, 17, 3, 17],
              's4096': [1000, 1500, 1200, 1700, 4096, 50]}[name]
        V = 3000 if S == 4096 else 12
        out = []
        for step, B in enumerate(Bs):
            sids = 1000 * (step * 5000 + np.arange(B, dtype=np.int64)) + rs.randint(0, 2500, size=B)
            sids[rs.rand(B) < 0.2] = 7                         # twins within and across batches
            out.append((sids, _rows(rs, B, 9, 1, V - 1)))
        return S, 9, V, out, False
    if name in ('t1_1', 't1_65'):
        T1 = int(name[3:])
        out = []
        for step in range(8):
            sids = rs.randint(1, 9, size=3).astype(np.int64)
            ai = _rows(rs, 3, T1, 1, 200)
            if T1 == 65:
                ai[0] = rs.permutation(np.arange(1, 66))[::-1]      # 65 distinct items, unsorted
                ai[1, :40] = 7                                     # repeats
            out.append((sids, ai))
        return 6, T1, 201, out, False
    if name == 'big_ids':
        out = []
        for step in range(6):
            sids = rs.randint(1, 6, size=2).astype(np.int64)
            out.append((sids, _rows(rs, 2, 5, MAX_ID - 30, 30)))
        return 3, 5, MAX_ID, out, False
    raise KeyError(name)


RING_CASES = ['returning', 'returning_partial', 'returning_batches', 'twins_random', 's1', 's2', 's17', 's17_full',
              's4096', 't1_1', 't1_65', 'big_ids']


@gpu
@pytest.mark.parametrize('name', RING_CASES)
def test_ring_update(name):
    """nar_sknn_update against SknnRef.update batch by batch: ids, lens, sorted sets, live bits (including ids that come
    back after an eviction discarded their pairs), the zero tail of every slot, guards."""
    S, T1, V, batches, must_revive = _ring_batches(name)
    ring = Ring(S, V)
    ref = SknnRef(sessions_buffer_size=S)
    revived = set()
    for sids, ai in batches:
        before = ref.export()
        assert ring.update(sids, ai) == 0
        ref.update(sids, ai)
        revived |= _revived(before, ref.export(), len(sids))
        ring.check(ref)
    assert bool(revived) or not must_revive


@gpu
@pytest.mark.parametrize('B', [1, 2, 3, 4, 5])
def test_ring_every_head(B):
    """A ring of 5 slots fed batches of B: updates start at every head residue."""
    rs = np.random.RandomState(B)
    ring = Ring(5, 20)
    ref = SknnRef(sessions_buffer_size=5)
    heads = set()
    for step in range(12):
        heads.add(ring.head)
        sids = rs.randint(1, 5, size=B).astype(np.int64)
        ai = _rows(rs, B, 4, 1, 6)
        assert ring.update(sids, ai) == 0
        ref.update(sids, ai)
        ring.check(ref)
    assert heads == set(range(5)) or B == 5


REJECT_RING = [
    ('b_gt_s', dict(B=5), NAR_ERR_INVALID),
    ('t1_66', dict(T1=66), NAR_ERR_INVALID),
    ('w_129', dict(W=129), NAR_ERR_INVALID),
    ('head_s', dict(head=4), NAR_ERR_INVALID),
    ('count_gt_s', dict(count=5), NAR_ERR_INVALID),
    ('items_2_31', dict(num_items=1 << 31), NAR_ERR_INVALID),
    ('items_0', dict(num_items=0), NAR_ERR_INVALID),
    ('b_neg', dict(B=-1), NAR_ERR_INVALID),
]


@gpu
@pytest.mark.parametrize('name,kw,rc', REJECT_RING, ids=[r[0] for r in REJECT_RING])
def test_ring_update_rejects(name, kw, rc):
    ring = Ring(4, 20, W=129 if 'W' in kw else WIDTH)
    B, T1 = max(kw.get('B', 2), 1), kw.get('T1', 3)
    ai = np.ones((B, T1), dtype=np.int64)
    assert ring.update(np.arange(B), ai, **kw) == rc
    ring.untouched()


@gpu
def test_ring_empty_batch_and_bad_ids():
    """B = 0 changes nothing; an id outside [0, num_items) sets err = 1 and is dropped like padding."""
    ring = Ring(4, 20)
    assert ring.update(np.zeros(0, np.int64), np.zeros((0, 3), np.int64)) == 0
    ring.untouched()
    ai = np.array([[3, 20, 4], [-2, 5, 0]], dtype=np.int64)
    assert ring.update([1, 2], ai) == 0
    ref = SknnRef(sessions_buffer_size=4)
    ref.update([1, 2], np.where((ai < 0) | (ai >= 20), 0, ai))
    ring.check(ref, err=1)


@gpu
def test_ring_load_and_continue():
    """SessionKNN.load of an oracle export narrower than the ring (dead pairs included, as a checkpoint written before
    returning ids revived them would hold), then the returning-id batches: the ring follows the oracle."""
    from chameleon_recsys_b200.baselines import BaselineTables
    ref = SknnRef(sessions_buffer_size=4)
    for s, items in RETURNING[:5]:
        ref.update([s], np.array([items]))
    ex = ref.export()
    assert not ex['live'].all()
    tab = BaselineTables([{'recommender': 'v-sknn', 'params': {'sessions_buffer_size': 4}}], 10)
    tab.load({'sknn_v-sknn_%s' % k: v for k, v in ex.items()})
    got = tab.export_knn('v-sknn')
    for k in ex:
        np.testing.assert_array_equal(got[k][:, :ex['items'].shape[1]] if got[k].ndim == 2 else got[k], ex[k])
    for s, items in RETURNING[5:] + [(9, [2]), (5, [1])]:
        tab.update(_dev(np.array([items])), session_ids=[s])
        ref.update([s], np.array([items]))
        got, want = tab.export_knn('v-sknn'), ref.export()
        for k in want:
            np.testing.assert_array_equal(got[k][:, :want['items'].shape[1]] if got[k].ndim == 2 else got[k], want[k])


# ------------------------------------------------------------------------------------------------ session-kNN scoring
def _knn_ref(S, sample, nn, decay_div, jaccard):
    return SknnRef(S, sample, nn, 'jaccard' if jaccard else 'cosine', 'div' if decay_div else 'same')


def _fill(ring, ref, rs, n_batches, B, T1, lo, V, hub=None, hub_p=0.0):
    for step in range(n_batches):
        sids = 1000 * (step * B + np.arange(B, dtype=np.int64)) + rs.randint(0, 2500, size=B)   # not ascending
        ai = _rows(rs, B, T1, lo, V)
        if hub is not None:
            ai[rs.rand(B) < hub_p, 0] = hub
        assert ring.update(sids, ai) == 0
        ref.update(sids, ai)


def _knn_queries(rs, B, T, K, lo, V, hub=None):
    ic = _rows(rs, B, T, lo, V, min_len=max(1, T // 2))
    if hub is not None:
        ic[:, 0] = hub
    ln = np.zeros((B, T), dtype=np.int64)
    ln[:, :-1] = ic[:, 1:]
    ln[:, -1] = rs.randint(lo, lo + V, size=B)
    ln[ic == 0] = 0
    neg = rs.randint(lo, lo + V, size=(B, T, K)).astype(np.int64)
    if K > 2:
        neg[rs.rand(B, T, K) < 0.1] = 0
        neg[:, :, 1] = ic                                      # the session's own items are candidates too
        neg[:, :, 2] = neg[:, :, 3 % K]                        # a duplicate
    return ic, ln, neg


def _knn_check(got, want, ln, top_n):
    rc, out, hist, met, err = got
    assert rc == 0 and err == 0
    act = ln.reshape(-1) != 0
    if out is not None:
        np.testing.assert_array_equal(out[act], want['ids'][act])
        assert (out[~act] == SENT64).all()
    np.testing.assert_array_equal(hist, want['hist'])
    assert met.tolist() == [PRE3[0] + want['hits'], PRE3[1] + want['rr'], PRE3[2] + want['count']]


def _knn_case(ring, ref, ic, ln, neg, sample, nn, decay_div, jaccard, top_n, with_out=True):
    got = ring.score(ic, ln, neg, sample, nn, decay_div, jaccard, top_n, with_out)
    want = ref.score(ic, ln, neg, top_n)
    _knn_check(got, want, ln, top_n)
    return want


@gpu
@pytest.mark.parametrize('decay_div,jaccard', [(1, 0), (1, 1), (0, 0), (0, 1)])
def test_knn_score_variants(decay_div, jaccard):
    """Both decays x both similarities on a ring with twins and ids that are not ascending, with and without out_ids."""
    rs = np.random.RandomState(10 * decay_div + jaccard)
    ring, ref = Ring(60, 40), _knn_ref(60, 40, 15, decay_div, jaccard)
    _fill(ring, ref, rs, 8, 10, 8, 1, 39)
    ic, ln, neg = _knn_queries(rs, 4, 8, 30, 1, 39)
    want = _knn_case(ring, ref, ic, ln, neg, 40, 15, decay_div, jaccard, 10)
    assert want['hits'] > 0
    _knn_case(ring, ref, ic, ln, neg, 40, 15, decay_div, jaccard, 10, with_out=False)


@gpu
def test_knn_score_empty_ring():
    ring, ref = Ring(8, 30), _knn_ref(8, 5, 5, 1, 0)
    rs = np.random.RandomState(0)
    ic, ln, neg = _knn_queries(rs, 3, 4, 6, 1, 29)
    want = _knn_case(ring, ref, ic, ln, neg, 5, 5, 1, 0, 5)
    assert want['count'] > 0 and want['hits'] == 0


@gpu
@pytest.mark.parametrize('T', [1, 63, 64])
def test_knn_score_positions(T):
    """Active sessions of 1, 63 and 64 positions (the 64-bit position masks, bit 63) with repeated items."""
    rs = np.random.RandomState(T)
    ring, ref = Ring(80, 40), _knn_ref(80, 0, 50, 1, 0)
    _fill(ring, ref, rs, 8, 10, 20, 1, 39)
    ic, ln, neg = _knn_queries(rs, 2, T, 12, 1, 39)
    if T > 1:
        ic[0, :] = rs.randint(1, 40, size=T)                   # every position, repeats
        ic[0, 40:45] = ic[0, 0]
        ln[0, :-1] = ic[0, 1:]
    want = _knn_case(ring, ref, ic, ln, neg, 0, 50, 1, 0, 10)
    assert want['hits'] > 0 or T == 1


@gpu
@pytest.mark.parametrize('n', [63, 64, 65, 129, 1023])
def test_knn_score_candidate_chunks(n):
    """Exactly n distinct nonzero candidates per query: scored 64 at a time, so 63, 64, 65, 129 and 1023 end the last
    chunk at every kind of boundary."""
    rs = np.random.RandomState(n)
    V = 1200
    ring, ref = Ring(300, V + 1), _knn_ref(300, 0, 300, 1, 0)
    _fill(ring, ref, rs, 6, 50, 60, 1, V, hub=7, hub_p=0.5)
    B, T = 2, 3
    ic, ln, _ = _knn_queries(rs, B, T, 1, 1, V, hub=7)
    held = np.array(sorted({x for _, it in ref.buffer if 7 in it for x in it} - {7}), dtype=np.int64)
    K = 1023 if n == 1023 else n + 6                       # duplicates and padding past the distinct ones
    neg = np.zeros((B, T, K), dtype=np.int64)
    for b in range(B):
        for t in range(T):
            if ln[b, t] == 0:
                continue
            pool = np.setdiff1d(held, [ln[b, t]])
            rest = np.setdiff1d(np.arange(1, V + 1), np.append(pool, ln[b, t]))
            others = np.concatenate([rs.permutation(pool), rs.permutation(rest)])[:n - 1]
            row = np.concatenate([others, others[rs.randint(0, n - 1, size=K - (n - 1))]])
            row[-1] = 0
            neg[b, t] = row
            assert len(set(row[row != 0].tolist()) | {int(ln[b, t])}) == n
    top_n = min(100, n)
    want = _knn_case(ring, ref, ic, ln, neg, 0, 300, 1, 0, top_n)
    assert (want['ids'] != 0).sum(axis=1).max() >= top_n - 4          # nearly every candidate is scored


@gpu
@pytest.mark.parametrize('mode', ['zero', 'total', 'total-1', 'small'])
def test_knn_score_sample_size(mode):
    """candidate_sessions_sample_size 0 (no cut), exactly the query's copy total, one less, and far less."""
    rs = np.random.RandomState(len(mode))
    ring, ref0 = Ring(120, 30), _knn_ref(120, 0, 60, 1, 0)
    _fill(ring, ref0, rs, 6, 20, 8, 1, 29)
    ic, ln, neg = _knn_queries(rs, 1, 5, 25, 1, 29)
    ic[0] = rs.randint(1, 30, size=5)
    ln[0, :-1] = 0                                             # one query: the whole session
    ln[0, -1] = rs.randint(1, 30)
    total = sum(ref0.candidates(ic[0].tolist()).values())
    assert total > 10
    sample = {'zero': 0, 'total': total, 'total-1': total - 1, 'small': 7}[mode]
    ref = _knn_ref(120, sample, 60, 1, 0)
    ref.buffer, ref.map = ref0.buffer, ref0.map
    _knn_case(ring, ref, ic, ln, neg, sample, 60, 1, 0, 10)


@gpu
@pytest.mark.parametrize('nn', [0, 1, 3, 10000])
def test_knn_score_neighbours(nn):
    """nearest_neighbor_session_for_scoring 0 (no item scored), 1, 3 and more than every copy."""
    rs = np.random.RandomState(nn % 97)
    ring, ref = Ring(50, 25), _knn_ref(50, 0, nn, 0, 0)
    _fill(ring, ref, rs, 5, 10, 8, 1, 24)
    ic, ln, neg = _knn_queries(rs, 3, 6, 20, 1, 24)
    want = _knn_case(ring, ref, ic, ln, neg, 0, nn, 0, 0, 10)
    if nn == 0:
        assert not want['ids'].any()
    else:
        assert want['ids'].any()


@gpu
@pytest.mark.parametrize('decay_div,jaccard', [(1, 0), (0, 1), (0, 0)])
def test_knn_score_similarity_one_excluded(decay_div, jaccard):
    """A stored session equal to the query's item set: a similarity of exactly 1 is no neighbour (V-SkNN cosine and
    SkNN jaccard of a one-item session, SkNN jaccard of a repeated pair); the other neighbours decide."""
    ring, ref = Ring(16, 20), _knn_ref(16, 0, 3, decay_div, jaccard)
    batches = [([101, 102, 103, 104], [[3, 0, 0], [3, 7, 0], [3, 9, 11], [7, 12, 0]]),
               ([105, 106, 107, 108], [[7, 3, 0], [3, 5, 0], [7, 13, 3], [5, 14, 0]])]
    for sids, ai in batches:
        assert ring.update(sids, np.array(ai)) == 0
        ref.update(sids, np.array(ai))
    ic = np.array([[3, 7, 7]], dtype=np.int64)
    ln = np.array([[7, 7, 5]], dtype=np.int64)
    neg = np.array([[[3, 9, 11, 12, 13, 14, 5]] * 3], dtype=np.int64)
    want = _knn_case(ring, ref, ic, ln, neg, 0, 3, decay_div, jaccard, 5)
    assert ref._sim([3], frozenset([3])) == 1.0
    assert want['count'] == 3 and want['ids'].any()


@gpu
@pytest.mark.parametrize('sample,nn', [(700, 600), (0, 1000)])
def test_knn_score_many_candidates(sample, nn):
    """More than 512 candidate sessions (each score-kernel thread handles several in the prefix cuts) in a ring of 1600
    slots, with the 'recent' cut and the neighbour cut both active, or the neighbour cut alone."""
    rs = np.random.RandomState(sample + nn)
    ring, ref = Ring(1600, 400), _knn_ref(1600, sample, nn, 1, 0)
    _fill(ring, ref, rs, 4, 400, 8, 1, 399, hub=5, hub_p=0.9)
    ic, ln, neg = _knn_queries(rs, 1, 3, 60, 1, 399, hub=5)
    ic[0, 1:] = rs.randint(6, 399, size=2)
    ln[0] = [ic[0, 1], ic[0, 2], rs.randint(6, 399)]
    ref.C = 0
    assert len(ref.candidates(ic[0].tolist())) > 1000     # sessions the binary search finds, before the cuts
    ref.C = sample
    kept = len(ref.neighbors(ic[0].tolist(), cut=False))
    assert kept > 512
    _knn_case(ring, ref, ic, ln, neg, sample, nn, 1, 0, 20)


@gpu
def test_knn_score_full_ring_and_big_ids():
    """S = 4096 slots (the shared-memory limit), T1 = 65, item ids near 2^31 - 1."""
    rs = np.random.RandomState(4096)
    lo, V = MAX_ID - 500, 499
    ring, ref = Ring(4096, MAX_ID), _knn_ref(4096, 1000, 500, 1, 0)
    _fill(ring, ref, rs, 5, 1000, 65, lo, V, hub=lo + 3, hub_p=0.3)
    ring.check(ref)
    ic, ln, neg = _knn_queries(rs, 2, 4, 40, lo, V, hub=lo + 3)
    want = _knn_case(ring, ref, ic, ln, neg, 1000, 500, 1, 0, 10)
    assert want['ids'].any()


REJECT_KNN = [
    ('s_4097', dict(S=4097), NAR_ERR_UNSUPPORTED),
    ('t_65', dict(T=65), NAR_ERR_UNSUPPORTED),
    ('k_1024', dict(K=1024), NAR_ERR_UNSUPPORTED),
    ('top_n_0', dict(top_n=0), NAR_ERR_INVALID),
    ('head_s', dict(head=8), NAR_ERR_INVALID),
    ('count_gt_s', dict(count=9), NAR_ERR_INVALID),
    ('sample_neg', dict(sample=-1), NAR_ERR_INVALID),
    ('nn_neg', dict(nn=-1), NAR_ERR_INVALID),
    ('items_2_31', dict(num_items=1 << 31), NAR_ERR_INVALID),
    ('t_0', dict(T=0), NAR_ERR_INVALID),
]


@gpu
@pytest.mark.parametrize('name,kw,rc', REJECT_KNN, ids=[r[0] for r in REJECT_KNN])
def test_knn_score_rejects(name, kw, rc):
    """Rejected before any launch: rank_hist, metrics, out_ids and err untouched (S = 4097 on a ring that large)."""
    S = kw.get('S', 8)
    ring = Ring(S, 20)
    T = max(kw.get('T', 3), 1)
    rs = np.random.RandomState(1)
    ic = rs.randint(1, 20, size=(2, T)).astype(np.int64)
    ln = rs.randint(1, 20, size=(2, T)).astype(np.int64)
    neg = rs.randint(1, 20, size=(2, T, kw.get('K', 4))).astype(np.int64)
    over = {k: v for k, v in kw.items() if k not in ('S', 'top_n')}
    if 'top_n' in kw:
        over['top_n_arg'] = kw['top_n']
    got = ring.score(ic, ln, neg, over.pop('sample', 0), over.pop('nn', 5), 1, 0, 5, **over)
    rc_, out, hist, met, err = got
    assert rc_ == rc
    assert (hist == SENT64).all() and met.tolist() == PRE3.tolist() and err == 0 and (out == SENT64).all()


@gpu
def test_knn_score_bad_ids_set_err():
    ring, ref = Ring(8, 20), _knn_ref(8, 0, 5, 1, 0)
    rs = np.random.RandomState(3)
    _fill(ring, ref, rs, 2, 4, 4, 1, 19)
    ic, ln, neg = _knn_queries(rs, 2, 3, 5, 1, 19)
    ln[:] = np.where(ic != 0, 3, 0)
    neg[1, 0, 0] = 20
    rc, out, hist, met, err = ring.score(ic, ln, neg, 0, 5, 1, 0, 5)
    assert rc == 0 and err == 1
