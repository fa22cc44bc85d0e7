"""The feature-row kernels of csrc/features.cu against a plain fp64 reference written here (pytest -m gpu).

Every entry point is called directly: nar_gather_features (ops.gather_features), its backward, nar_feature_stats and the
two row builders.  Plans are built with plan.FeaturePlan from synthetic configs (so the column order and ctx_col0 are the
real ones) and completed the way the engine completes them (engine.set_plan_columns); every embedding table and gamma /
beta is carved out of one flat fp32 buffer, as the engine's ParamLayout does.

Inputs are chosen where the kernels can go wrong: context and metadata ids of -5, card and >= 2^31 (one-hot all zero,
embeddings clamped to [0, card-1]), int64 numeric metadata above 2^24, rows of item 0, input rows whose event_timestamp
differs from max_ts, articles created after the reference time (the elapsed-days clamp), row counts that are not a
multiple of the gather's 8-row chunks, and three row groups with statistics of their own.  Item ids stay in [0, V): the
wide path does not clamp them.

The bars, and the agreement measured on one H100 SXM (80 GB, 700 W), are in each test's docstring.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

MS_PER_DAY = 1000.0 * 60.0 * 60.0 * 24.0
DAY = 86400000
T0 = 1_520_000_000_000                      # ms, the synthetic "now"
LB_REC, LB_NOV = 1.3, 2.0                   # elapsed_days_smooth_log_base, popularity_smooth_log_base
MAX_OHE = 10
N_POS = 96                                  # positions (B*T) of the synthetic batch
L, K, U, N_CAND = 37, 5, 23, 29             # L is not a multiple of the gather's 8-row chunk
SLACK = 1 << 16                             # floats after the last table of a flat buffer
ONE_ROUNDING = 2.0 ** -24                   # |RN32(x) - x| <= 2^-24 |x|
NORM_BAR = 4e-6
GRAD_BAR = 1e-5


def _seq(**feats):
    cfg = {'event_timestamp': {'type': 'numerical', 'dtype': 'int'}}
    cfg.update(feats)
    return {'single_features': {}, 'sequence_features': cfg}


def _cat(card):
    return {'type': 'categorical', 'dtype': 'int', 'cardinality': int(card)}


_NUM = {'type': 'numerical', 'dtype': 'float'}
_ALL_INTERNAL = {'recency': True, 'novelty': True, 'article_content_embeddings': True, 'item_clicked_embeddings': True}


def _articles(V, **feats):
    cfg = {'article_id': _cat(V), 'created_at_ts': {'type': 'numerical', 'dtype': 'int'}}
    cfg.update(feats)
    return cfg


def _cfg_g1():
    """The G1 feature set at g1 dimensions: ACR 250 and item embedding 117 give 2 + 1 tail columns."""
    from chameleon_recsys_b200.hparams import get_articles_features_config, get_session_features_config
    V = 46034
    return get_session_features_config(V), get_articles_features_config(V), dict(_ALL_INTERNAL), 250, V


def _cfg_adressa(V=72933, city=1022):
    """nar_trainer_adressa.py:106-224 with the cardinalities of its comments: three metadata embeddings and a 1022-value
    city embedding."""
    scfg = _seq(item_clicked=_cat(V), city=_cat(city), region=_cat(237), country=_cat(70), device=_cat(5), os=_cat(10),
                local_hour_sin=_NUM, local_hour_cos=_NUM, weekday=_NUM, referrer_class=_cat(7))
    acfg = _articles(V, category0=_cat(41), category1=_cat(128), author=_cat(112))
    return scfg, acfg, dict(_ALL_INTERNAL), 250, V


def _cfg_meta():
    """Metadata one-hot (cardinality 7 and 10), metadata numeric (int64, above 2^24) and a metadata embedding; ACR 98
    and item embedding 59 give 2 + 3 tail columns."""
    V = 3000
    scfg = _seq(item_clicked=_cat(V), device=_cat(4), city=_cat(1022), hour=_NUM)
    acfg = _articles(V, kind=_cat(7), words={'type': 'numerical', 'dtype': 'int'}, section=_cat(10),
                     delay={'type': 'numerical', 'dtype': 'int'}, author=_cat(300))
    return scfg, acfg, dict(_ALL_INTERNAL), 98, V


def _cfg_no_acr():
    """Item embedding as the only wide segment (at column 0), with context and metadata."""
    V = 5000
    scfg = _seq(item_clicked=_cat(V), os=_cat(23), region=_cat(29), hour=_NUM)
    acfg = _articles(V, category_id=_cat(461))
    return scfg, acfg, dict(_ALL_INTERNAL, article_content_embeddings=False), 250, V


def _cfg_profile_a():
    """Profile A: no context (CTX_ZERO), no metadata, ACR + item embedding only."""
    V = 5000
    icfg = dict(_ALL_INTERNAL, recency=False, novelty=False)
    return _seq(item_clicked=_cat(V)), _articles(V), icfg, 250, V


def _cfg_budget(n_ci=0, n_cf=0, n_me=0):
    """n_ci context ids, n_cf context floats, n_me metadata arrays (one-hot, embedding and numeric mixed)."""
    V = 1000
    feats = {'item_clicked': _cat(V)}
    for i in range(n_ci):
        feats['c%d' % i] = _cat((5, 40, 9, 300)[i % 4])
    for i in range(n_cf):
        feats['f%d' % i] = _NUM
    meta = {}
    for i in range(n_me):
        meta['m%d' % i] = {'type': 'numerical', 'dtype': 'int'} if i % 3 == 2 else _cat((7, 60)[i % 2])
    icfg = dict(_ALL_INTERNAL, article_content_embeddings=False)
    return _seq(**feats), _articles(V, **meta), icfg, 64, V


PLANS = {'g1': _cfg_g1, 'adressa': _cfg_adressa, 'meta': _cfg_meta, 'no_acr': _cfg_no_acr, 'profile_a': _cfg_profile_a}


def _feature_plan(cfgs):
    from chameleon_recsys_b200.plan import FeaturePlan
    scfg, acfg, icfg, E, V = cfgs
    return FeaturePlan(scfg, acfg, icfg, MAX_OHE, E, V)


# ---------------------------------------------------------------------------------------------------------------- data
class Case:
    """One plan with its tables and one synthetic batch, on the host (numpy) and on the device.  ``order`` permutes the
    small embedding tables inside the flat buffer; ``flat`` = (host array, device tensor) shares a flat buffer between
    cases."""

    def __init__(self, fp, seed=0, order=None, flat=None):
        import torch
        from chameleon_recsys_b200.plan import SEG_META_NUM
        rs = np.random.RandomState(seed)
        self.fp, V = fp, fp.num_items
        self.V = V
        self.tab, self.gamma_off, self.beta_off, self.total = self.carve(fp, order)
        if flat is None:
            h = rs.standard_normal(self.total).astype(np.float32)
            if fp.use_item_emb:              # never read: NaN shows a read past the embedding width
                o, _, ld = self.tab['items_embedding']
                h[o:o + V * ld].reshape(V, ld)[:, fp.item_emb_dim:] = np.nan
            flat = (h, torch.from_numpy(h).cuda())
        self.flat, self.flat_dev = flat
        assert self.flat.size >= self.total
        self.acr = np.full((V, fp.acr_ld), np.nan, dtype=np.float32)
        self.acr[:, :fp.acr_dim] = rs.standard_normal((V, fp.acr_dim))
        self.acr_dev = torch.from_numpy(self.acr).cuda()
        # batch: positions, their context, and a pool of items the rows draw from
        self.pool = np.unique(np.concatenate([[0, 1, V - 1], rs.choice(V, 150, replace=False)]))
        self.event_ts = (T0 - rs.randint(0, 3 * DAY, size=N_POS)).astype(np.int64)
        self.max_ts = int(self.event_ts.max())
        self.ctx_int = []
        for n in fp.ctx_int_names:
            card = next(s.card for s in fp.segments if s.name == n)
            ids = rs.randint(0, card, size=N_POS).astype(np.int64)
            sp = rs.rand(N_POS) < 0.25
            ids[sp] = rs.choice([-5, -1, card, card + 3, 2 ** 31, 2 ** 31 + 5, 2 ** 40], size=int(sp.sum()))
            self.ctx_int.append(ids)
        self.ctx_float = [rs.uniform(-2, 2, size=N_POS).astype(np.float32) for _ in fp.ctx_float_names]
        self.meta = []
        for n in fp.meta_names:
            s = next(s for s in fp.segments if s.name == n)
            if s.kind == SEG_META_NUM:
                m = rs.randint(-10 ** 6, 10 ** 6, size=V).astype(np.int64)
                big = [2 ** 24 + 1, 2 ** 24 + 3, 123456789, -(2 ** 31) - 1, 2 ** 40 + 12345, 2 ** 53 + 1, -(2 ** 45) - 7]
                sp = self.pool[rs.rand(self.pool.size) < 0.5]
                m[sp] = rs.choice(big, size=sp.size)
            else:
                m = rs.randint(0, s.card, size=V).astype(np.int64)
                sp = self.pool[rs.rand(self.pool.size) < 0.25]
                m[sp] = rs.choice([-5, -1, s.card, s.card + 3, 2 ** 31, 2 ** 40], size=sp.size)
            self.meta.append(m)
        self.created = (T0 - rs.randint(0, 16 * DAY, size=V)).astype(np.int64)
        late = self.pool[rs.rand(self.pool.size) < 0.15]
        self.created[late] = T0 + rs.randint(1, 2 * DAY, size=late.size)        # after every reference time: days clamp to 0
        self.pop = rs.uniform(1e-4, 1.0, size=V).astype(np.float32)
        self.item_clicked = rs.choice(self.pool, size=N_POS).astype(np.int64)
        self.label_next = rs.choice(self.pool, size=N_POS).astype(np.int64)
        self.negatives = rs.choice(self.pool, size=(N_POS, K)).astype(np.int64)
        self.item_clicked[::7] = 0
        self.negatives[::5, 1] = 0
        # per-group statistics for the forward / backward tests: each group its own item set and reference time
        st = [_ref_stats(_rec_raw(self.max_ts - 2 * g * DAY, self.created[S]), _nov_raw(self.pop[S]))
              for g, S in enumerate(rs.choice(self.pool, size=(3, 60)))]
        self.group_stats = np.asarray(st, dtype=np.float32)
        self.dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda()
                    for k, v in dict(event_ts=self.event_ts, max_ts=np.array([self.max_ts], np.int64), created=self.created,
                                     pop=self.pop, item_clicked=self.item_clicked, label_next=self.label_next,
                                     negatives=self.negatives).items()}
        self.ctx_int_dev = [torch.from_numpy(a).cuda() for a in self.ctx_int]
        self.ctx_float_dev = [torch.from_numpy(a).cuda() for a in self.ctx_float]
        self.meta_dev = [torch.from_numpy(a).cuda() for a in self.meta]

    @staticmethod
    def carve(fp, order=None):
        """Offsets in the flat buffer: the small embedding tables (permuted by ``order``), the item embedding, gamma,
        beta, then SLACK floats.  Returns ({key: (offset, rows, ld)}, gamma offset, beta offset, total floats)."""
        from chameleon_recsys_b200.plan import SEG_CTX_EMBED, SEG_META_EMBED, round_up
        tabs = [(s.param, s.card, s.width) for s in fp.segments if s.kind in (SEG_CTX_EMBED, SEG_META_EMBED)]
        if order is not None:
            tabs = [tabs[i] for i in order]
        if fp.use_item_emb:
            tabs.append(('items_embedding', fp.num_items, fp.item_emb_ld))
        off, tab = 0, {}
        for key, rows, ld in tabs:
            tab[key] = (off, rows, ld)
            off += round_up(rows * ld, 4)
        return tab, off, off + fp.Fp, off + 2 * fp.Fp + SLACK

    def table(self, key):
        off, rows, ld = self.tab[key]
        return self.flat[off:off + rows * ld].reshape(rows, ld)

    def gamma(self):
        return self.flat[self.gamma_off:self.gamma_off + self.fp.Fp]

    def beta(self):
        return self.flat[self.beta_off:self.beta_off + self.fp.Fp]

    def plan_c(self, stats_dev, grad_dev=None):
        """The C plan, completed the way NarEngine._plan_c_static completes it; gradients (backward) go to ``grad_dev``, a
        flat buffer with this case's offsets."""
        from chameleon_recsys_b200._lib import FeaturePlanC
        from chameleon_recsys_b200.engine import set_plan_columns
        from chameleon_recsys_b200.plan import SEG_ACR
        fp = self.fp
        p = FeaturePlanC()
        p.n_segments, p.row_ld = len(fp.segments), fp.Fp
        for i, s in enumerate(fp.segments):
            sg = p.seg[i]
            sg.kind, sg.col, sg.width, sg.card, sg.src = s.kind, s.int_col, s.width, s.card, s.src
            sg.ld, sg.table, sg.grad = 0, None, None
            if s.kind == SEG_ACR:
                sg.ld, sg.table = fp.acr_ld, self.acr_dev.data_ptr()
            elif s.param is not None:
                off, _, ld = self.tab[s.param]
                sg.ld, sg.table = ld, self.flat_dev.data_ptr() + 4 * off
                sg.grad = None if grad_dev is None else grad_dev.data_ptr() + 4 * off
        for i, t in enumerate(self.ctx_int_dev):
            p.ctx_int[i] = t.data_ptr()
        for i, t in enumerate(self.ctx_float_dev):
            p.ctx_float[i] = t.data_ptr()
        for i, t in enumerate(self.meta_dev):
            p.meta[i] = t.data_ptr()
        p.created_at_ts, p.pop_norm = self.dev['created'].data_ptr(), self.dev['pop'].data_ptr()
        p.gamma = self.flat_dev.data_ptr() + 4 * self.gamma_off
        p.beta = self.flat_dev.data_ptr() + 4 * self.beta_off
        p.stats = stats_dev.data_ptr()
        p.log_base_recency, p.log_base_novelty = LB_REC, LB_NOV
        set_plan_columns(p, fp)
        return p

    def rows(self, layout):
        """(row_pos, row_item, (n_rows, n_input, n_cand, n_positive, n_full)) of one row layout of ops.row_layout."""
        rs = np.random.RandomState(100 + LAYOUTS.index(layout))
        pos_idx = np.sort(rs.choice(N_POS, L, replace=False)).astype(np.int32)
        if layout == 'train':
            rp, ri = _ref_build_rows(pos_idx, self.item_clicked, self.label_next, self.negatives, K)
            return rp, ri, (rp.size, L, K + 1, 0, rp.size)
        if layout == 'base':
            uitems = rs.choice(self.pool, size=U).astype(np.int64)
            rp, ri = _ref_build_base_rows(pos_idx, self.item_clicked, self.label_next, uitems, U - 6, U)
            return rp, ri, (rp.size, L, 0, L, 2 * L)
        if layout == 'recommend':
            rp = np.concatenate([pos_idx, np.full(N_CAND, pos_idx[0], np.int32)])
            ri = np.concatenate([self.item_clicked[pos_idx], rs.choice(self.pool, size=N_CAND)]).astype(np.int64)
            return rp, ri, (rp.size, L, 0, 0, L)
        assert layout == 'one_row'
        return pos_idx[:1].copy(), np.array([self.pool[-2]], np.int64), (1, 0, 1, 0, 1)


_CASES = {}


def _case(name):
    if name not in _CASES:
        _CASES[name] = Case(_feature_plan(PLANS[name]()), seed=sorted(PLANS).index(name) + 1)
    return _CASES[name]


# ----------------------------------------------------------------------------------------------------------- reference
def _rec_raw(ts_ref, created):
    """nar_model.py:1055-1060 (int64 -> float32 before the subtraction, float32 division) + log_1p, the log in fp64."""
    days = (np.asarray(ts_ref, np.int64).astype(np.float32) - np.asarray(created, np.int64).astype(np.float32)) \
        / np.float32(MS_PER_DAY)
    return np.log1p(np.maximum(days, np.float32(0)).astype(np.float64)) / np.log(LB_REC)


def _nov_raw(pop):
    return -np.log(np.asarray(pop, np.float32).astype(np.float64)) / np.log(LB_NOV)


def _moments(x):
    m = x.mean()
    sd = np.sqrt(((x - m) ** 2).mean() + 1e-24)
    return [m, sd, (x.min() - m) / sd, (x.max() - m) / sd]


def _ref_stats(rec, nov):
    """{rec mean, sd, zmin, zmax, nov mean, sd, zmin, zmax} (nar_model.py:1011-1039, population variance)."""
    return _moments(np.asarray(rec, np.float64)) + _moments(np.asarray(nov, np.float64))


def _normalize(x, st):
    """normalize_values + min_max_normalization (nar_model.py:996-1039) with given statistics st = (mean, sd, zmin, zmax)."""
    st = np.asarray(st, np.float64)
    z = (x - st[..., 0]) / st[..., 1]
    return (z - st[..., 2] + 1e-24) / np.maximum(st[..., 3] - st[..., 2], 2e-24) * 2.0 - 1.0


def _groups(n_rows, n_input, n_cand, n_positive):
    r = np.arange(n_rows)
    g = np.full(n_rows, 2)
    if n_cand > 0:
        g[(r - n_input) % n_cand == 0] = 1
    else:
        g[r < n_input + n_positive] = 1
    g[r < n_input] = 0
    return g


def _ref_build_rows(pos_idx, item_clicked, label_next, negatives, K):
    n_cand = K + 1
    Lr = pos_idx.size
    rp = np.concatenate([pos_idx, np.repeat(pos_idx, n_cand)]).astype(np.int32)
    cand = np.concatenate([label_next[pos_idx][:, None], negatives.reshape(-1, K)[pos_idx]], axis=1) if K else \
        label_next[pos_idx][:, None]
    ri = np.concatenate([item_clicked[pos_idx], cand.reshape(-1)]).astype(np.int64)
    assert rp.size == Lr * (K + 2)
    return rp, ri


def _ref_build_base_rows(pos_idx, item_clicked, label_next, uitems, n_unique, U):
    u = np.where(np.arange(U) < n_unique, uitems[:U], 0)
    rp = np.concatenate([pos_idx, pos_idx, np.full(U, pos_idx[0])]).astype(np.int32)
    ri = np.concatenate([item_clicked[pos_idx], label_next[pos_idx], u]).astype(np.int64)
    return rp, ri


def _ref_features(c, row_pos, row_item, lay, stats):
    """fp64 reference of one gather.  Returns the scaled rows, the raw (unscaled) values, the class of every entry
    (0: exactly 0, 1: within one float32 rounding, 2: normalised recency / novelty) and which entries carry a gradient."""
    from chameleon_recsys_b200 import plan as P
    fp = c.fp
    n_rows, n_input, n_cand, n_positive, n_full = lay
    grp = _groups(n_rows, n_input, n_cand, n_positive)
    ts_ref = np.where(np.arange(n_rows) < n_input, c.event_ts[row_pos], c.max_ts)
    raw = np.zeros((n_rows, fp.Fp))
    cls = np.zeros((n_rows, fp.Fp), np.int8)
    for s in fp.segments:
        j = np.arange(s.width)
        if s.kind in (P.SEG_CTX_OHE, P.SEG_META_OHE):
            ids = c.ctx_int[s.src][row_pos] if s.kind == P.SEG_CTX_OHE else c.meta[s.src][row_item]
            v = (ids[:, None] == j[None, :]).astype(np.float64)
        elif s.kind in (P.SEG_CTX_EMBED, P.SEG_META_EMBED):
            ids = c.ctx_int[s.src][row_pos] if s.kind == P.SEG_CTX_EMBED else c.meta[s.src][row_item]
            v = c.table(s.param)[np.clip(ids, 0, s.card - 1)][:, :s.width]
        elif s.kind == P.SEG_CTX_NUM:
            v = c.ctx_float[s.src][row_pos][:, None]
        elif s.kind == P.SEG_CTX_ZERO:
            v = np.zeros((n_rows, 1))
        elif s.kind == P.SEG_META_NUM:
            v = c.meta[s.src][row_item].astype(np.float32)[:, None]
        elif s.kind == P.SEG_ACR:
            v = c.acr[row_item, :s.width]
        elif s.kind == P.SEG_ITEM_EMB:
            v = c.table('items_embedding')[row_item, :s.width]
        elif s.kind == P.SEG_RECENCY:
            v = _normalize(_rec_raw(ts_ref, c.created[row_item]), stats[grp, 0:4])[:, None]
        else:
            assert s.kind == P.SEG_NOVELTY
            v = _normalize(_nov_raw(c.pop[row_item]), stats[grp, 4:8])[:, None]
        cols = s.int_col + j
        raw[:, cols] = v
        cls[:, cols] = 2 if s.kind in (P.SEG_RECENCY, P.SEG_NOVELTY) else 1
    live = cls > 0
    live[n_full:, fp.ctx_col0:] = False           # item-only rows: no context
    cls[~live] = 0
    val = np.where(live, raw * c.gamma().astype(np.float64) + c.beta().astype(np.float64), 0.0)
    return val, raw, cls, live


def _gather(c, row_pos, row_item, lay, stats, plan=None):
    """Run the gather on a NaN-prefilled output and return it (fp64)."""
    import torch
    from chameleon_recsys_b200 import ops
    n_rows, n_input, n_cand, n_positive, n_full = lay
    stats_dev = torch.from_numpy(np.ascontiguousarray(stats, np.float32).reshape(-1)).cuda()
    plan = plan if plan is not None else c.plan_c(stats_dev)
    out = torch.full((n_rows, c.fp.Fp), float('nan'), device='cuda')
    ops.gather_features(plan, torch.from_numpy(row_pos).cuda(), torch.from_numpy(row_item).cuda(),
                        ops.row_layout(n_rows, n_input, n_cand, n_positive, n_full, c.fp.ctx_col0),
                        c.dev['event_ts'], c.dev['max_ts'], out)
    return out.cpu().numpy().astype(np.float64), stats_dev


def _check_forward(c, row_pos, row_item, lay, stats, got, what):
    """Padding / item-only context entries exactly 0, table / one-hot / numeric entries within one float32 rounding of
    the fp64 raw*gamma+beta, normalised entries within NORM_BAR*max(1, |ref|).  Returns the measured ratios to the bars."""
    ref, _, cls, _ = _ref_features(c, row_pos, row_item, lay, stats)
    assert not np.isnan(got).any(), (what, 'unwritten entries', np.argwhere(np.isnan(got))[:8].tolist())
    z = cls == 0
    assert (got[z] == 0).all(), (what, 'padding / item-only context entries', np.argwhere(z & (got != 0))[:8].tolist())
    err = np.abs(got - ref)
    v = cls == 1
    bar1 = ONE_ROUNDING * np.abs(ref) * (1 + 1e-9) + 1e-44
    bad = v & (err > bar1)
    assert not bad.any(), (what, 'table / one-hot / numeric', [(int(r), int(k), got[r, k], ref[r, k])
                                                                for r, k in np.argwhere(bad)[:8]])
    nrm = cls == 2
    bar2 = NORM_BAR * np.maximum(1.0, np.abs(ref))
    bad = nrm & (err > bar2)
    assert not bad.any(), (what, 'recency / novelty', [(int(r), int(k), got[r, k], ref[r, k]) for r, k in np.argwhere(bad)[:8]])
    r1 = float((err[v] / bar1[v]).max()) if v.any() else 0.0
    r2 = float((err[nrm] / bar2[nrm]).max()) if nrm.any() else 0.0
    print('agreement %s: one-rounding entries max err/bar %.3f, normalised entries max err/bar %.3g (max err %.3g)'
          % (what, r1, r2, float(err[nrm].max()) if nrm.any() else 0.0))


LAYOUTS = ('train', 'base', 'recommend', 'one_row')


# --------------------------------------------------------------------------------------------------------------- tests
def test_normalization_reference_matches_oracle():
    """The test's normalisation (statistics + normalize_values) against NarOracle._normalize_values: within 1e-12 (fp64
    both sides; measured 0)."""
    import torch
    from oracle.nar_oracle import NarOracle
    rs = np.random.RandomState(3)
    sample = rs.uniform(0, 12, size=500)
    x = rs.uniform(-2, 14, size=300)
    mine = _normalize(x, _ref_stats(sample, sample)[:4])
    theirs = NarOracle._normalize_values(None, torch.from_numpy(x), torch.from_numpy(sample)).numpy()
    assert np.abs(mine - theirs).max() < 1e-12


@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('plan', sorted(PLANS))
def test_gather_forward(plan, layout):
    """Every column of every row against fp64, each row group read with its own statistics.
    Bars: padding and the context columns of item-only rows exactly 0; table, one-hot and numeric columns within one
    float32 rounding of raw*gamma+beta (the kernel's fma rounds once); recency / novelty within 4e-6*max(1, |ref|), a few
    float32 roundings of O(1) values (float32 elapsed days, logf, the normalisation's divisions).
    Measured: one-rounding entries at most 0.995 of their bar (the fma rounds exactly once); normalised entries at most
    5.1e-7, 0.10 of their bar."""
    c = _case(plan)
    row_pos, row_item, lay = c.rows(layout)
    got, _ = _gather(c, row_pos, row_item, lay, c.group_stats)
    _check_forward(c, row_pos, row_item, lay, c.group_stats, got, '%s/%s' % (plan, layout))


@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('plan', sorted(PLANS))
def test_gather_backward(plan, layout):
    """d_beta, d_gamma and the context / metadata / item embedding gradients against fp64, accumulated onto nonzero
    gradients.  Every gradient lives in one flat buffer with the parameters' offsets; the entries no row reaches (padding
    columns, the rest of every table, the ACR, which has no gradient) must keep their prefill exactly.
    Bar: 1e-5 of each entry's absolute sum (prefill included): float32 atomics in an unspecified order.
    Measured: at most 0.03 of the bar (3e-7 of the absolute sum)."""
    import torch
    from chameleon_recsys_b200 import ops
    from chameleon_recsys_b200 import plan as P
    c = _case(plan)
    fp = c.fp
    row_pos, row_item, lay = c.rows(layout)
    n_rows, n_input, n_cand, n_positive, n_full = lay
    rs = np.random.RandomState(11)
    d_out = rs.standard_normal((n_rows, fp.Fp)).astype(np.float32)
    prefill = rs.uniform(-1, 1, size=c.total).astype(np.float32)
    grad_dev = torch.from_numpy(prefill).cuda()
    stats_dev = torch.from_numpy(c.group_stats.reshape(-1)).cuda()
    ops.gather_features_bwd(c.plan_c(stats_dev, grad_dev), torch.from_numpy(row_pos).cuda(), torch.from_numpy(row_item).cuda(),
                            ops.row_layout(n_rows, n_input, n_cand, n_positive, n_full, fp.ctx_col0),
                            c.dev['event_ts'], c.dev['max_ts'], torch.from_numpy(d_out).cuda(),
                            grad_dev[c.gamma_off:c.gamma_off + fp.Fp], grad_dev[c.beta_off:c.beta_off + fp.Fp])
    got = grad_dev.cpu().numpy().astype(np.float64)
    # fp64 reference
    _, raw, _, live = _ref_features(c, row_pos, row_item, lay, c.group_stats)
    d = np.where(live, d_out.astype(np.float64), 0.0)
    exp = prefill.astype(np.float64)
    mag = np.abs(exp)
    touched = np.zeros(c.total, bool)
    cols = np.arange(fp.Fp)
    has = live.any(axis=0)
    for off, v, a in ((c.beta_off, d.sum(0), np.abs(d).sum(0)), (c.gamma_off, (d * raw).sum(0), np.abs(d * raw).sum(0))):
        exp[off + cols] += v
        mag[off + cols] += a
        touched[off + cols[has]] = True
    gam = c.gamma().astype(np.float64)
    for s in fp.segments:
        if s.kind not in (P.SEG_CTX_EMBED, P.SEG_META_EMBED, P.SEG_ITEM_EMB):
            continue
        if s.kind == P.SEG_ITEM_EMB:
            ids = row_item
        else:
            ids = c.ctx_int[s.src][row_pos] if s.kind == P.SEG_CTX_EMBED else c.meta[s.src][row_item]
            ids = np.clip(ids, 0, s.card - 1)
        off, _, ld = c.tab[s.param]
        j = np.arange(s.width)
        v = d[:, s.int_col + j] * gam[s.int_col + j]
        keep = live[:, s.int_col]
        idx = (off + ids[keep, None] * ld + j[None, :]).reshape(-1)
        np.add.at(exp, idx, v[keep].reshape(-1))
        np.add.at(mag, idx, np.abs(v[keep]).reshape(-1))
        touched[idx] = True
    assert (got[~touched] == prefill[~touched]).all(), ('entries no row reaches changed',
                                                        np.flatnonzero(~touched & (got != prefill))[:8].tolist())
    err = np.abs(got - exp)[touched]
    bar = GRAD_BAR * mag[touched]
    worst = np.argmax(err / bar)
    assert (err <= bar).all(), ('gradients', int(np.flatnonzero(touched)[worst]), err[worst], bar[worst])
    print('agreement backward %s/%s: max err/bar %.3g' % (plan, layout, float((err / bar).max())))


def test_descriptor_cache_follows_the_plan():
    """Two plans through one context in the order P1, P2, P1.  P2 has P1's columns, segment count and narrow ranges; its
    small embedding tables sit in the same flat buffer in the reverse order and its city embedding has cardinality 1030
    instead of 1022 (same width, 45).  Only the segment table of the descriptor cache key tells the plans apart, and a
    stale descriptor would read another table (in bounds: the tables of both plans start at the buffer's first float).
    Bars: those of test_gather_forward; measured: normalised entries at most 0.072 of their bar."""
    import torch
    fp1 = _feature_plan(_cfg_adressa(V=5000))
    fp2 = _feature_plan(_cfg_adressa(V=5000, city=1030))
    assert [(s.int_col, s.width) for s in fp1.segments] == [(s.int_col, s.width) for s in fp2.segments]
    n_small = sum(s.param is not None and s.param != 'items_embedding' for s in fp1.segments)
    order2 = list(range(n_small))[::-1]
    total = max(Case.carve(fp1)[3], Case.carve(fp2, order2)[3])
    h = np.random.RandomState(5).standard_normal(total).astype(np.float32)
    flat = (h, torch.from_numpy(h).cuda())
    c1 = Case(fp1, seed=21, flat=flat)
    c2 = Case(fp2, seed=22, order=order2, flat=flat)
    assert c1.tab['ctx_emb/city'][0] == 0 and c2.tab['ctx_emb/city'][0] != 0
    for c in (c1, c2, c1):
        row_pos, row_item, lay = c.rows('train')
        got, _ = _gather(c, row_pos, row_item, lay, c.group_stats)
        _check_forward(c, row_pos, row_item, lay, c.group_stats, got, 'cache/%s' % c.tab['ctx_emb/city'][1])


def test_zero_variance_statistics_are_bit_identical():
    """A buffer holding a single item: the statistics kernel sees one value, so the variance is 0, the sd 1e-12 and
    zmin = zmax = 0.  A row of that item normalises to exactly 0 only if its raw value is bit-identical to the one the
    statistics kernel saw (one ulp of difference becomes ~1e5 after the division by the sd): its novelty column, and the
    recency column of its candidate rows (reference time max_ts, as in the statistics), must equal beta exactly.
    32 items, so that an ulp-level difference in either column (about one value in eight) cannot hide."""
    import torch
    from chameleon_recsys_b200 import ops
    c = _case('meta')
    fp = c.fp
    rec_col = next(s.int_col for s in fp.segments if s.name == 'recency')
    nov_col = next(s.int_col for s in fp.segments if s.name == 'novelty')
    row_pos, row_item0, lay = c.rows('train')
    n_rows, n_input, n_cand, _, _ = lay
    rs = np.random.RandomState(9)
    fresh = [i for i in c.pool if i != 0 and c.created[i] < c.max_ts]
    beta = c.beta()
    for item in rs.choice(fresh, size=32, replace=False):
        buf = np.zeros(700, np.int64)
        buf[123] = item
        row_item = row_item0.copy()
        row_item[rs.rand(n_rows) < 0.4] = item
        stats_dev = torch.zeros(24, device='cuda')
        rp, ri = torch.from_numpy(row_pos).cuda(), torch.from_numpy(row_item).cuda()
        ops.feature_stats(torch.from_numpy(buf).cuda(), 500, c.dev['created'], c.dev['pop'], c.dev['max_ts'], LB_REC, LB_NOV,
                          rp, ri, n_rows, n_input, n_cand, c.dev['event_ts'], stats_dev)
        out = torch.full((n_rows, fp.Fp), float('nan'), device='cuda')
        ops.gather_features(c.plan_c(stats_dev), rp, ri, ops.row_layout(*lay, ctx_col0=fp.ctx_col0), c.dev['event_ts'],
                            c.dev['max_ts'], out)
        o = out.cpu().numpy()
        mine = row_item == item
        cand = mine & (np.arange(n_rows) >= n_input)
        assert (o[mine, nov_col] == beta[nov_col]).all(), (int(item), o[mine, nov_col][:4], beta[nov_col])
        assert (o[cand, rec_col] == beta[rec_col]).all(), (int(item), o[cand, rec_col][:4], beta[rec_col])


STATS_CASES = {
    # name: (buf_len, nonzero entries, n_norm, layout of the rows)
    'empty_train': (2000, 0, 500, 'train'),
    'empty_recommend': (2000, 0, 500, 'recommend'),
    'fewer_than_n_norm': (700, 300, 500, 'train'),
    'more_than_n_norm': (5000, 3000, 2000, 'train'),
    'g1_buffer': (20000, 20000, 2000, 'train'),
}


@pytest.mark.parametrize('name', sorted(STATS_CASES))
def test_feature_stats(name):
    """nar_feature_stats against fp64 over the first n_norm nonzero buffer entries in buffer order, or, with an empty
    buffer, over each row group's own rows that are not item 0.  Buffer lengths below 1024 and not multiples of 1024.
    Bars: mean and sd within 1e-5 relative (float32 sums of up to 2000 terms), zmin and zmax within 1e-4 (O(1) values).
    Measured: mean / sd at most 1.7e-7 relative, zmin / zmax at most 4.3e-7."""
    import torch
    from chameleon_recsys_b200 import ops
    c = _case('g1')
    buf_len, nnz, n_norm, layout = STATS_CASES[name]
    rs = np.random.RandomState(buf_len + nnz)
    buf = np.zeros(buf_len, np.int64)
    where = np.sort(rs.choice(buf_len, nnz, replace=False))
    buf[where] = rs.choice(c.pool[1:], size=nnz)
    row_pos, row_item, lay = c.rows(layout)
    n_rows, n_input, n_cand, _, _ = lay
    stats_dev = torch.full((24,), float('nan'), device='cuda')
    ops.feature_stats(torch.from_numpy(buf).cuda(), n_norm, c.dev['created'], c.dev['pop'], c.dev['max_ts'], LB_REC, LB_NOV,
                      torch.from_numpy(row_pos).cuda(), torch.from_numpy(row_item).cuda(), n_rows, n_input, n_cand,
                      c.dev['event_ts'], stats_dev)
    got = stats_dev.cpu().numpy().astype(np.float64).reshape(3, 8)
    if nnz:
        ids = buf[buf != 0][:n_norm]
        ref = [_ref_stats(_rec_raw(c.max_ts, c.created[ids]), _nov_raw(c.pop[ids]))] * 3
        groups = [0, 1, 2]
    else:
        grp = _groups(n_rows, n_input, n_cand, 0)       # the statistics kernel: n_cand == 0 -> every candidate row is group 2
        ts = np.where(np.arange(n_rows) < n_input, c.event_ts[row_pos], c.max_ts)
        ref, groups = [None] * 3, []
        for g in range(3):
            m = (grp == g) & (row_item != 0)
            if m.any():
                ref[g] = _ref_stats(_rec_raw(ts[m], c.created[row_item[m]]), _nov_raw(c.pop[row_item[m]]))
                groups.append(g)
        assert groups == ([0, 1, 2] if layout == 'train' else [0, 2])
    worst_ms, worst_z = 0.0, 0.0
    for g in groups:
        r = np.asarray(ref[g])
        for k in (0, 1, 4, 5):
            e = abs(got[g, k] - r[k]) / abs(r[k])
            worst_ms = max(worst_ms, e)
            assert e < 1e-5, (name, g, k, got[g, k], r[k])
        for k in (2, 3, 6, 7):
            e = abs(got[g, k] - r[k])
            worst_z = max(worst_z, e)
            assert e < 1e-4, (name, g, k, got[g, k], r[k])
    print('agreement stats %s: mean/sd rel %.3g, zmin/zmax abs %.3g' % (name, worst_ms, worst_z))


@pytest.mark.parametrize('k', [0, K])
def test_build_rows(k):
    """nar_build_rows equals numpy exactly (K = 0: one candidate per position)."""
    import torch
    from chameleon_recsys_b200 import ops
    c = _case('meta')
    pos_idx = np.sort(np.random.RandomState(4).choice(N_POS, L, replace=False)).astype(np.int32)
    neg = np.ascontiguousarray(c.negatives[:, :k]) if k else np.zeros(1, np.int64)
    n = L * (k + 2)
    rp = torch.full((n,), -7, dtype=torch.int32, device='cuda')
    ri = torch.full((n,), -7, dtype=torch.int64, device='cuda')
    ops.build_rows(torch.from_numpy(pos_idx).cuda(), L, c.dev['item_clicked'], c.dev['label_next'],
                   torch.from_numpy(neg).cuda(), k, rp, ri)
    erp, eri = _ref_build_rows(pos_idx, c.item_clicked, c.label_next, c.negatives[:, :k], k)
    assert np.array_equal(rp.cpu().numpy(), erp) and np.array_equal(ri.cpu().numpy(), eri)


@pytest.mark.parametrize('n_unique', [0, U - 6, U])
def test_build_base_rows(n_unique):
    """nar_build_base_rows equals numpy exactly: clicked rows, positive rows, then the unique-negative table, whose unused
    entries (u >= n_unique) hold item 0 at the first position."""
    import torch
    from chameleon_recsys_b200 import ops
    c = _case('meta')
    rs = np.random.RandomState(6)
    pos_idx = np.sort(rs.choice(N_POS, L, replace=False)).astype(np.int32)
    uitems = rs.choice(np.arange(1, c.V), size=U).astype(np.int64)
    n = 2 * L + U
    bp = torch.full((n,), -7, dtype=torch.int32, device='cuda')
    bi = torch.full((n,), -7, dtype=torch.int64, device='cuda')
    ops.build_base_rows(torch.from_numpy(pos_idx).cuda(), L, c.dev['item_clicked'], c.dev['label_next'],
                        torch.from_numpy(uitems).cuda(), torch.tensor([n_unique], dtype=torch.int32, device='cuda'), U,
                        torch.zeros(L * K, dtype=torch.int32, device='cuda'), K, bp, bi)
    erp, eri = _ref_build_base_rows(pos_idx, c.item_clicked, c.label_next, uitems, n_unique, U)
    assert np.array_equal(bp.cpu().numpy(), erp) and np.array_equal(bi.cpu().numpy(), eri)


BUDGET = {'ctx_ids': 12, 'ctx_floats': 8, 'meta': 8}


@pytest.mark.parametrize('over', [0, 1])
@pytest.mark.parametrize('source', sorted(BUDGET))
def test_lane_budget(source, over):
    """The gather's scalar lanes: at most 12 context ids, 8 context floats and 8 metadata arrays.  A plan at the limit
    matches fp64 (bars of test_gather_forward; measured: normalised entries at most 0.086 of their bar); one more raises
    NarError (NAR_ERR_UNSUPPORTED)."""
    from chameleon_recsys_b200._lib import NAR_MAX_SEGMENTS, NarError
    n = BUDGET[source] + over
    fp = _feature_plan(_cfg_budget(**{{'ctx_ids': 'n_ci', 'ctx_floats': 'n_cf', 'meta': 'n_me'}[source]: n}))
    assert len(fp.segments) <= NAR_MAX_SEGMENTS
    c = Case(fp, seed=30 + n)
    row_pos, row_item, lay = c.rows('train')
    if over:
        with pytest.raises(NarError, match='failed: -2 '):
            _gather(c, row_pos, row_item, lay, c.group_stats)
    else:
        got, _ = _gather(c, row_pos, row_item, lay, c.group_stats)
        _check_forward(c, row_pos, row_item, lay, c.group_stats, got, 'budget/%s' % source)
