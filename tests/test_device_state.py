"""Device-resident ClickedItemsState (SURVEY.md section 8f #1) against the host class, batch by batch."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu


def test_device_state_tracks_host_state():
    from chameleon_recsys_b200.clicked_items_state import ClickedItemsState
    from chameleon_recsys_b200.device_state import DeviceClickedItemsState
    from chameleon_recsys_b200.harness import make_problem
    pb = make_problem('tiny', profile='B')
    V = pb.plan.num_items
    host = ClickedItemsState(0.01, 300, 50, V)                      # 36 s window, 300 rows: cut-off and clip both bite
    dev = DeviceClickedItemsState(host)
    it = pb.input_fn()
    for step in range(25):
        f, l = it.get_next()
        all_items = np.concatenate([f['item_clicked'], l['label_last_item']], axis=1)
        host.update_from_batch(f['item_clicked'], f['event_timestamp'], l['label_last_item'])
        dev.update(torch.from_numpy(all_items).cuda(), torch.from_numpy(np.ascontiguousarray(f['event_timestamp'])).cuda(),
                   has_clicks=bool(all_items.any()))
        assert np.array_equal(dev.buffer_ids().cpu().numpy(), host.get_recent_clicks_buffer()), step
        assert np.array_equal(dev.articles_recent_pop_norm().cpu().numpy(),
                              host.get_articles_recent_pop_norm().astype(np.float32)), step
    back = dev.to_host(ClickedItemsState(0.01, 300, 50, V))
    assert np.array_equal(back.pop_recent_clicks_buffer, host.pop_recent_clicks_buffer)
    assert np.array_equal(back.get_articles_recent_pop_norm(), host.get_articles_recent_pop_norm())   # float64, bit-exact
    assert np.array_equal(back.get_articles_pop(), host.get_articles_pop())
    assert np.array_equal(back.get_articles_recent_pop(), host.get_articles_recent_pop())


# ------------------------------------------------------------------------------------------------ nar_state_update, bit-exact
# nar_state_update against oracle/clicked_items_state_ref.py (ClickedItemsStateRef.update_from_batch): the new buffer's ids
# and timestamps, recent_pop, pop_norm as float32 and float64, and articles_pop, all bit for bit.  Outputs start from a
# sentinel (the new buffer slot too, so every one of its cap entries must be written) and carry guard entries past their
# end that must keep it.
NAR_ERR_INVALID = -1
SENT = 0x5A5A5A5A5A5A5A5A
GUARD = 16
T0 = 1_500_000_000_000                                             # a 2017 timestamp in ms, like the datasets'


def _p(t):
    import ctypes as C
    return C.c_void_p(0 if t is None else t.data_ptr())


class _DeviceState:
    """two ping-pong buffer slots and the per-item vectors of nar_state_update, each with a guard past its end"""

    def __init__(self, cap, V, old_items, old_ts, articles_pop, pop64=True):
        d = 'cuda'
        self.cap, self.V = cap, V
        self.items = [torch.full((cap + GUARD,), SENT, dtype=torch.int64, device=d) for _ in range(2)]
        self.ts = [torch.full((cap + GUARD,), SENT, dtype=torch.int64, device=d) for _ in range(2)]
        self.items[0][:cap] = torch.from_numpy(old_items)
        self.ts[0][:cap] = torch.from_numpy(old_ts)
        self.recent_pop = torch.full((V + GUARD,), SENT, dtype=torch.int64, device=d)
        self.pop_norm = torch.full((V + GUARD,), SENT & 0xFFFFFFFF, dtype=torch.int32, device=d).view(torch.float32)
        self.pop_norm64 = torch.full((V + GUARD,), SENT, dtype=torch.int64, device=d).view(torch.float64) if pop64 else None
        self.articles_pop = torch.full((V + GUARD,), SENT, dtype=torch.int64, device=d)
        self.articles_pop[:V] = torch.from_numpy(articles_pop)
        self.err = torch.zeros(1 + GUARD, dtype=torch.int32, device=d)
        self.cur = 0

    def update(self, allc, ts, hours_ms, min_norm, **over):
        from chameleon_recsys_b200._lib import load
        from chameleon_recsys_b200 import ops
        o, n = self.cur, self.cur ^ 1
        self.items[n][:self.cap] = SENT
        self.ts[n][:self.cap] = SENT
        Bg, T1 = allc.shape
        a = dict(old_items=self.items[o], old_ts=self.ts[o], cap=self.cap, Bg=Bg, T=T1 - 1, new_items=self.items[n],
                 new_ts=self.ts[n], V=self.V)
        a.update(over)
        # an empty batch still passes real (non-null) pointers
        allc_d = torch.from_numpy(np.ascontiguousarray(allc).reshape(-1) if allc.size else np.zeros(1, np.int64)).cuda()
        ts_d = torch.from_numpy(np.ascontiguousarray(ts).reshape(-1) if ts.size else np.zeros(1, np.int64)).cuda()
        rc = load().nar_state_update(_p(a['old_items']), _p(a['old_ts']), a['cap'], _p(allc_d), _p(ts_d), a['Bg'], a['T'],
                                     hours_ms, _p(a['new_items']), _p(a['new_ts']), _p(self.recent_pop), _p(self.pop_norm),
                                     _p(self.pop_norm64), _p(self.articles_pop), a['V'], min_norm, _p(self.err),
                                     ops._stream())
        torch.cuda.synchronize()
        return rc

    def check(self, ref, slot):
        cap, V = self.cap, self.V
        buf = ref.pop_recent_clicks_buffer
        assert np.array_equal(self.items[slot][:cap].cpu().numpy(), buf[:, 0])
        assert np.array_equal(self.ts[slot][:cap].cpu().numpy(), buf[:, 1])
        assert np.array_equal(self.recent_pop[:V].cpu().numpy(), ref.articles_recent_pop)
        norm = np.asarray(ref.articles_recent_pop_norm, dtype=np.float64)
        assert np.array_equal(self.pop_norm[:V].cpu().numpy().view(np.int32), norm.astype(np.float32).view(np.int32))
        if self.pop_norm64 is not None:
            assert np.array_equal(self.pop_norm64[:V].cpu().numpy().view(np.int64), norm.view(np.int64))
        assert np.array_equal(self.articles_pop[:V].cpu().numpy(), ref.articles_pop)
        self.check_guards()
        assert int(self.err[0].item()) == 0

    def check_guards(self):
        for t in self.items + self.ts + [self.recent_pop, self.articles_pop]:
            assert bool((t[-GUARD:] == SENT).all()), 'write past the end of a buffer'
        assert bool((self.pop_norm.view(torch.int32)[-GUARD:] == (SENT & 0xFFFFFFFF)).all())
        if self.pop_norm64 is not None:
            assert bool((self.pop_norm64.view(torch.int64)[-GUARD:] == SENT).all())
        assert bool((self.err[1:] == 0).all())


def _ref(hours, cap, n_norm, V, old_items, old_ts, articles_pop):
    from oracle.clicked_items_state_ref import ClickedItemsStateRef
    ref = ClickedItemsStateRef(hours, cap, n_norm, V)
    ref.pop_recent_clicks_buffer = np.stack([old_items, old_ts], axis=1).astype(np.int64)
    ref.articles_pop = articles_pop.copy()
    return ref


def _batch(rs, Bg, T, V, zero_frac, t0, span):
    """[Bg, T+1] ids with padding anywhere in a session, [Bg, T] timestamps in no particular order within a session"""
    allc = rs.randint(1, V, size=(Bg, T + 1)).astype(np.int64)
    allc[rs.random_sample(allc.shape) < zero_frac] = 0
    ts = (t0 + rs.randint(0, span, size=(Bg, T))).astype(np.int64)
    return allc, ts


def _batch_min_ts(allc, ts):
    from oracle.clicked_items_state_ref import batch_clicks_for_state_update
    T = ts.shape[1]
    return int(batch_clicks_for_state_update(allc[:, :T], ts, allc[:, T:])[1].min())


def _with_nonzero(rs, allc, n):
    """zero entries of allc (anywhere) until exactly n are nonzero"""
    flat = allc.reshape(-1)
    nz = np.flatnonzero(flat)
    flat[rs.choice(nz, nz.size - n, replace=False)] = 0
    return allc


def _run_update(ref, dev, allc, ts, hours_ms, min_norm):
    T = ts.shape[1]
    ref.update_from_batch(allc[:, :T], ts, allc[:, T:])
    assert dev.update(allc, ts, hours_ms, min_norm) == 0
    dev.check(ref, dev.cur ^ 1)
    dev.cur ^= 1


# id, cap, V, Bg, T, zero fraction, nonzero old entries, hours, n_norm
UPDATE_CASES = [
    ('g1_batch_over_cap', 300, 1000, 256, 20, 0.2, 300, 0.01, 50),
    ('batch_equals_cap', 1025, 1025, 64, 20, 0.0, 500, 0.01, 50),
    ('batch_plus_kept_equals_cap', 1025, 46034, 40, 20, 0.1, 0, 1.0, 500),
    ('cap20000_window_keeps_all', 20000, 46034, 256, 20, 0.3, 15000, 1e6, 1000),
    ('window_keeps_nothing', 1025, 1000, 60, 20, 0.25, 1025, 0.0, 50),
    ('cutoff_exact', 20000, 1025, 256, 20, 0.1, 3000, 1.0, 50),
    ('label_ts_unsorted_padding', 300, 1000, 5, 7, 0.3, 100, 0.5, 50),
    ('norm_floor_exact', 300, 1000, 11, 9, 0.0, 200, 0.0, 100),
    ('single_click_sessions', 1025, 1025, 700, 1, 0.3, 400, 2.0, 50),
]


@pytest.mark.parametrize('pop64', [True, False], ids=['pop64', 'pop64_null'])
@pytest.mark.parametrize('case', UPDATE_CASES, ids=[c[0] for c in UPDATE_CASES])
def test_state_update_bit_exact(case, pop64):
    name, cap, V, Bg, T, zf, n_old, hours, n_norm = case
    rs = np.random.RandomState(cap + V + Bg)
    hours_ms = int(hours * 1000 * 60 * 60)                         # as ClickedItemsStateRef and DeviceClickedItemsState
    min_norm = 1.0 / n_norm
    span = 600_000
    allc, ts = _batch(rs, Bg, T, V, zf, T0, span)
    old_items = np.zeros(cap, np.int64)
    old_ts = np.zeros(cap, np.int64)
    old_items[:n_old] = rs.randint(1, V, size=n_old)
    old_ts[:n_old] = T0 - rs.randint(0, 2 * max(hours_ms, 1) + span, size=n_old)
    if name == 'batch_equals_cap':
        allc = _with_nonzero(rs, allc, cap)
    elif name == 'batch_plus_kept_equals_cap':
        allc = _with_nonzero(rs, allc, 600)
        thr = _batch_min_ts(allc, ts) - hours_ms
        n = 700                                                   # 425 inside the window, 275 before it, interleaved
        inside = rs.permutation(n) < 425
        old_items[:n] = rs.randint(1, V, size=n)
        old_ts[:n] = np.where(inside, thr + rs.randint(0, 1000, size=n), thr - 1 - rs.randint(0, 1000, size=n))
    elif name == 'cap20000_window_keeps_all':
        old_ts[:n_old] = T0 - rs.randint(0, 10 ** 9, size=n_old)  # and the zero rows (ts 0) are inside the window too
    elif name == 'window_keeps_nothing':
        old_ts[:n_old] = _batch_min_ts(allc, ts) - 1 - rs.randint(0, 10_000, size=n_old)
    elif name == 'cutoff_exact':
        thr = _batch_min_ts(allc, ts) - hours_ms
        old_ts[:n_old:3] = thr                                    # kept
        old_ts[1:n_old:3] = thr - 1                               # dropped
    elif name == 'label_ts_unsorted_padding':
        allc[:, 2] = 0                                            # padding inside every session ...
        ts[:, 2] = T0 + span + 5                                  # ... whose timestamp is the row maximum: the label's
        ts[0] = T0 + np.array([50, 10, 40, 20, 30, 5, 60])        # maximum at the last click
        allc[1, T] = 0                                            # a session without a label
    elif name == 'norm_floor_exact':
        # 99 distinct clicks, nothing kept: pop / (99 + 1) = 1/100 = min_norm exactly for every clicked id
        allc[:] = 0
        allc.reshape(-1)[rs.choice(allc.size, 99, replace=False)] = rs.choice(np.arange(1, V), 99, replace=False)
        old_ts[:n_old] = 0
    articles_pop = rs.randint(0, 50, size=V).astype(np.int64)
    ref = _ref(hours, cap, n_norm, V, old_items, old_ts, articles_pop)
    dev = _DeviceState(cap, V, old_items, old_ts, articles_pop, pop64=pop64)
    _run_update(ref, dev, allc, ts, hours_ms, min_norm)
    if name == 'batch_plus_kept_equals_cap':
        assert (ref.pop_recent_clicks_buffer[:, 0] != 0).all()
    if name == 'norm_floor_exact':
        clicked = np.unique(allc[allc != 0])
        assert (ref.articles_recent_pop_norm[clicked] == min_norm).all()
    if name == 'cutoff_exact':
        assert (ref.pop_recent_clicks_buffer[:, 1] == thr).sum() == len(range(0, n_old, 3))


def test_state_update_g1_ping_pong():
    """30 G1-shaped steps (256 x 21) through the two buffer slots: the 36 s window and the 20000-row cap both bite"""
    cap, V, Bg, T, hours, n_norm = 20000, 46034, 256, 20, 0.01, 1000
    hours_ms = int(hours * 1000 * 60 * 60)
    rs = np.random.RandomState(30)
    zeros = np.zeros(cap, np.int64)
    articles_pop = np.zeros(V, np.int64)
    ref = _ref(hours, cap, n_norm, V, zeros, zeros, articles_pop)
    dev = _DeviceState(cap, V, zeros, zeros, articles_pop)
    for step in range(30):
        allc, ts = _batch(rs, Bg, T, V, 0.15, T0 + step * 15_000, 20_000)
        _run_update(ref, dev, allc, ts, hours_ms, 1.0 / n_norm)


def test_state_update_trivial_batches():
    """Bg = 0 and a batch of padding only: NAR_OK, nothing written (the caller keeps the old slot)"""
    cap, V = 300, 1000
    rs = np.random.RandomState(2)
    old_items = rs.randint(0, V, size=cap).astype(np.int64)
    old_ts = rs.randint(0, 1000, size=cap).astype(np.int64)
    articles_pop = rs.randint(0, 9, size=V).astype(np.int64)
    dev = _DeviceState(cap, V, old_items, old_ts, articles_pop)
    for allc, ts in ((np.zeros((0, 6), np.int64), np.zeros((0, 5), np.int64)),
                     (np.zeros((40, 6), np.int64), np.full((40, 5), T0, np.int64))):
        assert dev.update(allc, ts, 36_000, 0.02) == 0
        assert bool((dev.items[1][:cap] == SENT).all()) and bool((dev.ts[1][:cap] == SENT).all())
        assert bool((dev.recent_pop == SENT).all()) and bool((dev.pop_norm.view(torch.int32) == (SENT & 0xFFFFFFFF)).all())
        assert np.array_equal(dev.articles_pop[:V].cpu().numpy(), articles_pop)
        assert np.array_equal(dev.items[0][:cap].cpu().numpy(), old_items)
        dev.check_guards()


@pytest.mark.parametrize('bad', [-1, 1000, 1 << 40], ids=['negative', 'V', 'far'])
def test_state_update_flags_bad_ids(bad):
    """an id outside [0, V) sets err[0] to 1 (the state is unspecified afterwards)"""
    cap, V = 300, 1000
    rs = np.random.RandomState(3)
    allc, ts = _batch(rs, 20, 6, V, 0.1, T0, 1000)
    allc[7, 3] = bad
    dev = _DeviceState(cap, V, np.zeros(cap, np.int64), np.zeros(cap, np.int64), np.zeros(V, np.int64))
    assert dev.update(allc, ts, 36_000, 0.02) == 0
    assert int(dev.err[0].item()) == 1


@pytest.mark.parametrize('over', ['cap_0', 'cap_neg', 'V_0', 'T_0', 'alias_items', 'alias_ts'])
def test_state_update_rejects(over):
    cap, V = 300, 1000
    rs = np.random.RandomState(4)
    allc, ts = _batch(rs, 20, 6, V, 0.1, T0, 1000)
    dev = _DeviceState(cap, V, np.zeros(cap, np.int64), np.zeros(cap, np.int64), np.zeros(V, np.int64))
    kw = {'cap_0': dict(cap=0), 'cap_neg': dict(cap=-5), 'V_0': dict(V=0), 'T_0': dict(T=0),
          'alias_items': dict(new_items=dev.items[0]), 'alias_ts': dict(new_ts=dev.ts[0])}[over]
    assert dev.update(allc, ts, 36_000, 0.02, **kw) == NAR_ERR_INVALID
    assert bool((dev.items[1][:cap] == SENT).all()) and bool((dev.recent_pop == SENT).all())
    assert bool((dev.items[0][:cap] == 0).all()) and bool((dev.articles_pop[:V] == 0).all())
    dev.check_guards()
