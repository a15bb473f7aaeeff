"""The batched IVFFlat step at the shape thresholds of its route choices, against the oracle.

ivf_scan_topk picks, per sub-batch, the tensor-core filter level (0, 1 or 2), slab selection or full selection, the refine
with its own selection or after a selection launch, the list-major or the per-query exact kernel, or the fused one-query
kernels.  Each choice is a threshold on k, probes, nq, the candidate capacity cap (the sum of the `probes` longest lists),
the query row stride or the list lengths.  The indexes here are loaded list by list with IvfflatIndex.load, so list
lengths and cap are exact, and every case sits on one side of one threshold and asserts that side through what the library
counts: filter launches and bytes (tc_traffic), queries refined at level 0 (tc_level0_rescored), launches (launch_count)
and the certificate fallbacks.

Rows and queries are low-rank rows rounded to multiples of 1/16 (|x| < 8): every product, square and partial sum of a
distance is then an exact fp32 value, so every summation order gives the oracle's distance bit for bit.  Ids are the
oracle's except inside a run of equal distances; in the run that straddles position k, every returned row must be one
the oracle's probed lists hold at that distance.
"""
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_headline import low_rank

THREADS = os.cpu_count() or 8
gpu = pytest.mark.gpu

# ------------------------------------------------------------------------------ the route thresholds, restated on the host
# (vb_list_tc.cu list_tc_kp / cta_refine_smem_bytes, vb_slab_select.cuh ss_select_smem_bytes, vb_ivf_one.cu one_scan_smem)

SS_CAND, SMEM_MAX, ONE_MAX_Q = 2048, 200 * 1024, 16


def kp_of(k, level):
    if level == 0:
        return 128 if k <= 10 else 1 << 20
    if level == 1:
        return 64 if k <= 10 else 128 if k <= 40 else 1 << 20
    return 32 if k <= 10 else 48 if k <= 24 else 64 if k <= 40 else 1 << 20


def qstride(elem, dim):
    """stride of the fp32 query image the batched step builds (halfvec queries are widened to fp32)"""
    raw = 4 * dim if elem == O.VECTOR else 2 * dim
    pad = (raw + 15) & ~15
    return pad * 2 if elem == O.HALFVEC else pad


def slab_cap(cap, probes):
    return cap // 32 + 2 * probes + 2


def refine_smem(kp, qs, cap, probes):
    """shared memory of the one-CTA-per-query refine that selects from the slab minima"""
    cs = slab_cap(cap, probes)
    return SS_CAND * 8 + kp * 16 + qs + cs * 8 + (2 * probes + 2) * 4 + probes * 16 + 16 + kp * 4 + 16


def slabs_fit(k, level, qs, cap, probes):
    kp = kp_of(k, level)
    return kp <= 128 and refine_smem(kp, qs, cap, probes) <= SMEM_MAX


def one_scan_fits(cap, qs, probes, k):
    def pow2(x):
        p = 2
        while p < x:
            p <<= 1
        return p
    c = (cap + 3) & ~3
    smem = qs + probes * 8 + ((probes + 2) & ~1) * 4 + ((c + 1) & ~1) * 4 + pow2(min(k, c)) * 8
    return 1 <= k <= SS_CAND and smem <= SMEM_MAX


def largest_fitting_cap(fits, lo, hi):
    """the largest cap in [lo, hi) for which fits(cap) holds (fits monotone)"""
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid)
    return lo


def test_threshold_model_puts_the_cases_where_they_belong():
    """the shapes below sit where their names say: dim 64, probes 8: 700k rows fit the slab refine at every k, 800k and
    1.0M do not although the former bound (cap_s * 4 + 20 KiB <= 160 KiB) accepted them, 1.2M is past both; the widest
    query rows lower that edge"""
    qs = qstride(O.VECTOR, 64)
    old = lambda cap, p: slab_cap(cap, p) * 4 + 20 * 1024 <= 160 * 1024
    for k in WINDOW_K:
        lv = 0 if k <= 10 else 1
        assert slabs_fit(k, lv, qs, 700_000, 8)
        for n in (800_000, 1_000_000):
            assert not slabs_fit(k, lv, qs, n, 8) and old(n, 8), (k, n)
        assert not old(1_200_000, 8)
    assert not slabs_fit(10, 0, qs, 1_000_000, 1000) and old(1_000_000, 1000)
    assert slabs_fit(10, 0, qs, 720_000, 8) and not slabs_fit(10, 0, qstride(O.HALFVEC, 4000), 720_000, 8)


# ----------------------------------------------------------------------------------------------------------- data law

def grid_rows(n, dim, seed):
    """low-rank rows on the 1/16 grid"""
    return np.clip(np.rint(low_rank(n, dim, 16, seed=seed) * 16.0), -120, 120).astype(np.float32) / np.float32(16.0)


def as_elem(elem, y, dim):
    """rows of `dim` dimensions whose first y.shape[1] are y and the rest zero (wide rows at a modest host cost), in the
    element's payload layout"""
    if elem == O.HALFVEC:
        y = y.astype(np.float16).view(np.uint16)
    if y.shape[1] == dim:
        return np.ascontiguousarray(y)
    out = np.zeros((y.shape[0], dim), y.dtype)
    out[:, :y.shape[1]] = y
    return out


ACTIVE = 64   # dimensions that carry values; past them rows, queries and centres are zero


class Case:
    """an index of given list lengths over grid rows, its oracle twin and its queries.  Image row r holds x[r] (its
    first ACTIVE dimensions); its heap id is n - 1 - r (the library must map positions to ids)"""

    def __init__(self, pv, opclass, dim, lens, nq, seed=1):
        self.pv = pv
        self.elem, self.metric, _, _ = pv.OPCLASSES[opclass]
        lens = np.asarray(lens, np.int64)
        self.n, self.lists = int(lens.sum()), len(lens)
        self.off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        a = min(dim, ACTIVE)
        self.x = grid_rows(self.n, a, seed)
        self.q = grid_rows(nq, a, seed + 1000)
        rng = np.random.default_rng(seed)
        # centres: grid rows of their own, so probe selection is exact on both sides
        c = grid_rows(self.lists, a, seed + 2000) + np.float32(rng.integers(-8, 9, (self.lists, 1)) / 16)
        self.ids = (self.n - 1 - np.arange(self.n)).astype(np.int64)
        self.xe, self.qe, self.ce = as_elem(self.elem, self.x, dim), as_elem(self.elem, self.q, dim), as_elem(self.elem, c, dim)
        self.l0_failed = False   # a level-0 failure may rest level 0 for the next batches of this index
        self.ix = pv.IvfflatIndex(opclass, dim, self.lists).load(self.ce, self.off, self.xe, self.ids)
        self.oix = O.Ivf(self.elem, self.metric, self.ce, self.off, self.xe, self.ids)

    def cap(self, probes):
        return int(np.sort(np.diff(self.off))[::-1][:probes].sum())

    def want(self, probes, k, sample=None):
        q = self.qe if sample is None else self.qe[sample]
        return self.oix.search_batch(q, probes, k, threads=THREADS)

    def exact(self, r, j):
        """the fp32 distance of row r to query j, computed exactly (every term is on the grid)"""
        d = self.x[r].astype(np.float64) - self.q[j].astype(np.float64)
        return float(d @ d) if self.metric == O.L2_SQUARED else -float(self.x[r].astype(np.float64) @ self.q[j].astype(np.float64))

    def check(self, got, want, probes, queries=None, allowed=None):
        """bit for bit the oracle's distances; its ids outside runs of equal distance; in the run at position k, rows of
        the probed lists (and of `allowed`) at exactly that distance"""
        gi, gd = (np.asarray(a.cpu() if hasattr(a, "cpu") else a) for a in got)
        wi, wd = want
        queries = np.arange(len(gi)) if queries is None else queries
        assert gi.shape == wi.shape
        wd_cmp = wd.astype(np.float32) if gd.dtype == np.float32 else wd
        bad = np.flatnonzero(~(gd == wd_cmp).all(axis=1))
        assert bad.size == 0, ("distances", bad[:5], gd[bad[:1]], wd[bad[:1]])
        k = wi.shape[1]
        for jj, j in enumerate(queries):
            d = wd[jj]
            starts = np.flatnonzero(np.concatenate([[True], d[1:] != d[:-1]]))
            for a, b in zip(starts, list(starts[1:]) + [k]):
                if b < k or not np.isfinite(d[a]):
                    assert sorted(gi[jj, a:b]) == sorted(wi[jj, a:b]), (j, a, b, gi[jj, a:b], wi[jj, a:b])
                    continue
                # the straddling run: distinct rows of the probed lists at the run's distance
                rows = self.n - 1 - gi[jj, a:b]
                assert len(set(rows)) == b - a and (rows >= 0).all() and (rows < self.n).all(), (j, gi[jj, a:b])
                lists, _ = self.oix.scan_lists(self.qe[j], probes)
                row_list = np.searchsorted(self.off, rows, side="right") - 1
                assert np.isin(row_list, lists).all(), (j, row_list, lists)
                if allowed is not None:
                    assert np.isin(gi[jj, a:b], allowed).all(), j
                ref = self.exact(self.n - 1 - wi[jj, a], j)
                assert all(self.exact(r, j) == ref for r in rows), (j, a, b)

    def free(self):
        self.ix.free()


# ----------------------------------------------------------------------------------------------------------- routes

@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)
    for name, v in DEFAULTS.items():
        pv.set_option(name, v)


DEFAULTS = {"scan_impl": int(os.environ.get("VB_TEST_SCAN_IMPL", "2")), "tc_level0": 1, "tc_level1": 1, "slab_select": 1,
            "one_query": 1}


class options:
    """set library options for a block, restore the defaults after it"""

    def __init__(self, pv, **kw):
        self.pv, self.kw = pv, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.pv.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            self.pv.set_option(k, DEFAULTS[k])


def traced(pv, case, fn):
    """fn()'s result and what the search did: launches, filter launches and A-tile bytes read once (tc_traffic), queries
    refined at level 0, and the level 0 / level 1 / exact fallbacks it added"""
    ix = case.ix
    f = (ix.tc_level0_fallbacks(), ix.tc_level1_fallbacks(), ix.tc_fallbacks())
    pv.tc_traffic(True, read=True)
    pv.tc_level0_rescored()
    n0 = pv.launch_count()
    out = fn()
    pv.synchronize()
    r = {"launches": pv.launch_count() - n0, "l0_queries": int(pv.tc_level0_rescored()[2])}
    t = pv.tc_traffic(False, read=True)
    r.update(filters=int(t[3]), a_once=int(t[1]), f0=ix.tc_level0_fallbacks() - f[0], f1=ix.tc_level1_fallbacks() - f[1],
             fx=ix.tc_fallbacks() - f[2])
    case.l0_failed |= r["f0"] > 0
    return out, r


def slab_route(pv, case, q, probes, k, **kw):
    """(launches with slab_select on, launches with it off) of the same level-1 search: equal exactly when the search
    declines the slab minima (the full selection then runs either way), fewer with them (no selection launch)"""
    ix = case.ix
    with options(pv, tc_level0=0):
        ix.search(q, k=k, probes=probes, **kw)   # (the first batched search of an index builds its filter image)
    with options(pv, tc_level0=0, slab_select=1):
        got1, r1 = traced(pv, case, lambda: ix.search(q, k=k, probes=probes, **kw))
    with options(pv, tc_level0=0, slab_select=0):
        got0, r0 = traced(pv, case, lambda: ix.search(q, k=k, probes=probes, **kw))
    assert r1["filters"] > 0 and r0["filters"] > 0, (r1, r0)
    assert r1["fx"] == r0["fx"] == r1["f1"] == r0["f1"] == 0, (r1, r0)
    return got1, got0, r1["launches"], r0["launches"]


WINDOW_K = (1, 10, 11, 40)


@gpu
@pytest.mark.parametrize("n", [700_000, 800_000, 1_000_000, 1_200_000])
def test_slab_window_dim64_probes8(pv, n):
    """vector_l2_ops, dim 64, lists = probes = 8 in equal lists, nq = 64 (batched): below the slab refine's shared-memory
    edge (700k) slab selection and level 0 run; at 800k and 1.0M (which the former bound let through to a refine that
    refused them) and past 1.2M the search takes the full selection, never level 0, and still answers from the filter"""
    probes, nq = 8, 64
    case = Case(pv, "vector_l2_ops", 64, [n // 8] * 8, nq, seed=n // 1000)
    try:
        cap, qs = case.cap(probes), qstride(O.VECTOR, 64)
        want = case.want(probes, max(WINDOW_K))
        for k in WINDOW_K:
            level = 0 if k <= 10 else 1
            fit = slabs_fit(k, level, qs, cap, probes)
            rested = case.l0_failed
            got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
            case.check(got, (want[0][:, :k], want[1][:, :k]), probes)
            assert r["filters"] > 0, (n, k, r)
            if k <= 10 and fit and not rested:
                assert r["l0_queries"] == nq, (n, k, r)
            if not fit:
                assert r["l0_queries"] == 0, (n, k, r)
            g1, g0, l1, l0 = slab_route(pv, case, case.qe, probes, k)
            case.check(g1, (want[0][:, :k], want[1][:, :k]), probes)
            case.check(g0, (want[0][:, :k], want[1][:, :k]), probes)
            assert (l1 < l0) if fit else (l1 == l0), (n, k, fit, l1, l0)
    finally:
        case.free()


@gpu
def test_slab_window_probes_1000_and_exact_scan(pv):
    """ivfflat.probes = lists on a 1M-row, 1000-list index (cap_s ~ 33 250): even one query takes the batched step
    (the one-query kernels decline a million candidates), and the full selection answers it; also against
    Table.exact_topk over the same rows"""
    lists, probes = 1000, 1000
    case = Case(pv, "vector_l2_ops", 64, [1000] * lists, 64, seed=7)
    try:
        cap = case.cap(probes)
        assert not slabs_fit(10, 0, qstride(O.VECTOR, 64), cap, probes)
        assert not one_scan_fits(cap, qstride(O.VECTOR, 64), probes, 10)
        want = case.want(probes, 40)
        for k in (10, 40):
            got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
            case.check(got, (want[0][:, :k], want[1][:, :k]), probes)
            assert r["filters"] > 0 and r["l0_queries"] == 0, (k, r)
            one = case.ix.search(case.qe[:1], k=k, probes=probes)
            case.check(one, (want[0][:1, :k], want[1][:1, :k]), probes)
        t = pv.Table(O.VECTOR, 64).append(case.x)
        ti, td = t.exact_topk(O.L2_SQUARED, case.q, 40)
        t.free()
        # exact_topk numbers rows by table position; the index's ids are n - 1 - position
        case.check((np.where(ti >= 0, case.n - 1 - ti, -1), td), want, probes)
    finally:
        case.free()


@gpu
def test_slab_window_filtered_and_inner_product(pv):
    """inside the window (800k rows, dim 64, probes = lists = 8): a filtered search allowing about half the rows, and
    vector_ip_ops, whose refine bound differs, both take the full selection and answer as the oracle does"""
    n, probes, nq, k = 800_000, 8, 64, 10
    case = Case(pv, "vector_l2_ops", 64, [n // 8] * 8, nq, seed=3)
    try:
        allowed = np.flatnonzero(np.random.default_rng(5).random(n) < 0.5).astype(np.int64)
        f = case.ix.filter(allowed)
        keep = np.zeros(n, bool)
        keep[case.n - 1 - allowed] = True
        # the oracle over the allowed rows only: its order restricted to them is the filtered order
        off = np.concatenate([[0], np.cumsum([keep[case.off[l]:case.off[l + 1]].sum() for l in range(8)])]).astype(np.int64)
        oix = O.Ivf(O.VECTOR, O.L2_SQUARED, case.ce, off, case.xe[keep], case.ids[keep])
        want = oix.search_batch(case.qe, probes, k, threads=THREADS)
        g1, g0, l1, l0 = slab_route(pv, case, case.qe, probes, k, filter=f)
        case.check(g1, want, probes, allowed=allowed)
        case.check(g0, want, probes, allowed=allowed)
        assert l1 == l0, (l1, l0)
        with options(pv, tc_level0=1):
            got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes, filter=f))
        case.check(got, want, probes, allowed=allowed)
        assert r["filters"] > 0 and r["l0_queries"] == 0, r
        f.free()
    finally:
        case.free()
    case = Case(pv, "vector_ip_ops", 64, [n // 8] * 8, nq, seed=4)
    try:
        want = case.want(probes, 40)
        for k in (10, 40):
            got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
            case.check(got, (want[0][:, :k], want[1][:, :k]), probes)
            assert r["filters"] > 0 and r["l0_queries"] == 0, (k, r)
    finally:
        case.free()


@gpu
@pytest.mark.parametrize("elem,dim", [(O.VECTOR, 2000), (O.HALFVEC, 4000)])
def test_widest_rows_at_the_refine_limit(pv, elem, dim):
    """vector at 2000 and halfvec at 4000 dimensions (query images of 8000 and 16 000 bytes): eight lists just under the
    slab refine's shared-memory edge at k' = 128 and a ninth small list that takes cap past it.  probes = 8: slab
    selection (and level 0 at k = 10); probes = 9: the full selection, at k = 10 and 40"""
    opclass = "vector_l2_ops" if elem == O.VECTOR else "halfvec_l2_ops"
    qs = qstride(elem, dim)
    # the largest multiple of 8 * 32 rows whose eight lists still fit the refine at probes 8, and 2048 rows more at 9
    cap8 = largest_fitting_cap(lambda c: refine_smem(128, qs, c, 8) <= SMEM_MAX, 1, 1 << 22) // 256 * 256
    lens = [cap8 // 8] * 8 + [2048]
    assert slabs_fit(10, 0, qs, cap8, 8) and refine_smem(128, qs, cap8, 8) > SMEM_MAX - 8192
    assert not slabs_fit(10, 0, qs, cap8 + 2048, 9) and not slabs_fit(40, 1, qs, cap8 + 2048, 9)
    nq = 32
    case = Case(pv, opclass, dim, lens, nq, seed=dim)
    try:
        sample = np.arange(0, nq, 4)
        for probes, fit in ((8, True), (9, False)):
            assert case.cap(probes) == (cap8 if probes == 8 else cap8 + 2048)
            want = case.want(probes, 40, sample)
            for k in (10, 40):
                rested = case.l0_failed
                got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
                case.check((got[0][sample], got[1][sample]), (want[0][:, :k], want[1][:, :k]), probes, queries=sample)
                assert r["filters"] > 0, (probes, k, r)
                if k == 10 and fit and not rested:
                    assert r["l0_queries"] == nq, (probes, k, r)
                if not fit:
                    assert r["l0_queries"] == 0, (probes, k, r)
            g1, g0, l1, l0 = slab_route(pv, case, case.qe, probes, 40)
            case.check((g1[0][sample], g1[1][sample]), (want[0], want[1]), probes, queries=sample)
            assert (l1 < l0) if fit else (l1 == l0), (probes, l1, l0)
    finally:
        case.free()


@gpu
def test_k_steps_of_the_filter(pv):
    """k across the steps of list_tc_kp: level 0 up to k = 10, level 1 up to k = 40 (half the A-tile bytes of a forced
    level 2), no filter at 41 (list_tc_supported), and the exact kernels at 2048 / 2049 (2049: the sort-everything
    selection).  k' itself (64 or 128 at level 1, 32 / 48 / 64 at level 2) changes no counter: a step of it that keeps
    the level and the filter's support is seen only through these results."""
    probes, nq = 8, 64
    case = Case(pv, "vector_l2_ops", 64, [4000] * 16, nq, seed=11)
    try:
        want = case.want(probes, 2049)
        for k in (10, 11, 24, 25, 40, 41, 2048, 2049):
            sub = (want[0][:, :k], want[1][:, :k])
            rested = case.l0_failed
            got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
            case.check(got, sub, probes)
            if k > 40:
                assert r["filters"] == 0, (k, r)
                continue
            assert r["filters"] > 0 and r["f1"] == 0, (k, r)
            if k > 10 or not rested:
                assert r["l0_queries"] == (nq if k <= 10 else 0), (k, r)
            with options(pv, tc_level0=0):
                _, r1 = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
            with options(pv, tc_level0=0, tc_level1=0):
                g2, r2 = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
            case.check(g2, sub, probes)
            assert r1["f1"] == 0 and 2 * r1["a_once"] == r2["a_once"] > 0, (k, r1, r2)
    finally:
        case.free()


@gpu
def test_batched_threshold(pv):
    """nq * probes = 255 takes the per-query scans, 256 the batched step (tensor-core filter at k = 10); both answer as
    the oracle does"""
    case = Case(pv, "vector_l2_ops", 64, [3000] * 16, 64, seed=13)
    try:
        for nq, probes in ((51, 5), (85, 3), (64, 4), (32, 8)):
            q = case.qe[:nq]
            want = case.oix.search_batch(q, probes, 10, threads=THREADS)
            got, r = traced(pv, case, lambda: case.ix.search(q, k=10, probes=probes))
            case.check(got, want, probes)
            assert (r["filters"] > 0) == (nq * probes >= 256), (nq, probes, r)
    finally:
        case.free()


@gpu
def test_one_query_kernels_at_their_edges(pv):
    """the fused one-query kernels take at most 16 queries, a run of candidates that fits their shared memory and
    k <= 2048; one query past each edge (17 queries, 4 more candidates, k = 2049) takes the general path.  Which path ran
    is told by the launches of the same search with the one-query kernels switched off: fewer, or the same"""
    probes, k = 8, 10
    qs = qstride(O.VECTOR, 64)
    edge = largest_fitting_cap(lambda c: one_scan_fits(c, qs, probes, k), 1, 1 << 20)
    edge2048 = largest_fitting_cap(lambda c: one_scan_fits(c, qs, probes, 2048), 1, 1 << 20)
    assert one_scan_fits(edge, qs, probes, k) and not one_scan_fits(edge + 4, qs, probes, k)

    def lens_for(cap):   # probes lists summing to cap, eight shorter ones beside them
        base = cap // probes
        return [base + (1 if i < cap - base * probes else 0) for i in range(probes)] + [base // 2] * 8

    def run(case, nq, k, one_fits):
        q = case.qe[:nq]
        want = case.oix.search_batch(q, probes, k, threads=THREADS)
        with options(pv, one_query=1):
            got, r1 = traced(pv, case, lambda: case.ix.search(q, k=k, probes=probes))
        with options(pv, one_query=0):
            got0, r0 = traced(pv, case, lambda: case.ix.search(q, k=k, probes=probes))
        case.check(got, want, probes)
        case.check(got0, want, probes)
        applies = nq <= ONE_MAX_Q and one_fits
        assert (r1["launches"] < r0["launches"]) if applies else (r1["launches"] == r0["launches"]), (nq, k, r1, r0)

    for cap, kk in ((edge, k), (edge + 4, k), (edge2048, 2048)):
        case = Case(pv, "vector_l2_ops", 64, lens_for(cap), 17, seed=cap % 1000)
        try:
            assert case.cap(probes) == cap
            fits = one_scan_fits(cap, qs, probes, kk)
            for nq in (1, 16, 17):
                run(case, nq, kk, fits)
            if kk == 2048:
                run(case, 16, 2049, False)
        finally:
            case.free()


@gpu
def test_sub_batches(pv):
    """cap = 1M (eight lists of 125 000 rows, probes 8) limits a sub-batch to 268 queries: 600 queries run as 268 + 268 +
    64 through search, search_host_into, search_into (device buffers) and prefetch_queries + search_prefetched_into, each
    against Table.exact_topk over the same rows and the oracle on a sample.  Then 900 queries over two 350 000-row lists
    and 62 short ones (probes 2, cap 700k, 383 queries per sub-batch), where slab selection fits and level 0 runs: any
    query it could not certify is searched again and must land at its own row of its sub-batch.  (This law rarely leaves
    a query uncertified at level 0, so the re-run's offset is not pinned by it.)"""
    import torch
    probes, k, nq = 8, 10, 600
    case = Case(pv, "vector_l2_ops", 64, [125_000] * 8, nq, seed=17)
    try:
        assert (1 << 30) // (4 * case.cap(probes)) == 268
        t = pv.Table(O.VECTOR, 64).append(case.x)
        ti, td = t.exact_topk(O.L2_SQUARED, case.q, k)
        t.free()
        whole = (np.where(ti >= 0, case.n - 1 - ti, -1), td)
        sample = np.concatenate([np.arange(0, nq, 20), [267, 268, 535, 536, 599]])
        wsample = case.want(probes, k, sample)
        outs = {"search": case.ix.search(case.qe, k=k, probes=probes)}
        ids, dist = np.empty((nq, k), np.int64), np.empty((nq, k), np.float64)
        case.ix.search_host_into(np.ascontiguousarray(case.qe), k, probes, ids, dist)
        outs["host_into"] = (ids, dist)
        qd = torch.from_numpy(case.qe).cuda()
        di, dd = torch.empty((nq, k), dtype=torch.int64, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda")
        case.ix.search_into(qd, k, probes, di, dd)
        pv.synchronize()
        outs["into"] = (di, dd)
        pinned = torch.from_numpy(case.qe).pin_memory().numpy()
        ids2, dist2 = np.empty((nq, k), np.int64), np.empty((nq, k), np.float64)
        case.ix.prefetch_queries(pinned, 1)
        case.ix.search_prefetched_into(1, k, probes, ids2, dist2)
        outs["prefetched"] = (ids2, dist2)
        for name, got in outs.items():
            gi, gd = (np.asarray(a.cpu() if hasattr(a, "cpu") else a) for a in got)
            case.check((gi, gd), whole, probes)
            case.check((gi[sample], gd[sample]), wsample, probes, queries=sample)
    finally:
        case.free()

    lens = [350_000, 350_000] + [1000] * 62
    nq, probes = 900, 2
    case = Case(pv, "vector_l2_ops", 64, lens, nq, seed=19)
    try:
        cap = case.cap(probes)
        assert slabs_fit(k, 0, qstride(O.VECTOR, 64), cap, probes) and (1 << 30) // (4 * cap) == 383
        want = case.want(probes, k)
        got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
        case.check(got, want, probes)
        assert r["l0_queries"] >= nq, r
        got, r = traced(pv, case, lambda: _search_into(pv, case, probes, k))
        case.check(got, want, probes)
    finally:
        case.free()


def _search_into(pv, case, probes, k):
    import torch
    qd = torch.from_numpy(case.qe).cuda()
    di = torch.empty((len(qd), k), dtype=torch.int64, device="cuda")
    dd = torch.empty((len(qd), k), dtype=torch.float32, device="cuda")
    case.ix.search_into(qd, k, probes, di, dd)
    pv.synchronize()
    return di, dd


TC_ARMS = [(l0, l1, slab) for l0 in (1, 0) for l1 in (1, 0) for slab in (1, 0)]


@gpu
def test_list_lengths_at_tile_and_slab_edges(pv):
    """lists of 0, 1, 31, 32, 33, 127, 128, 129 rows and one of 6000, all probed by 64 queries, under every combination
    of tc_level0, tc_level1 and slab_select on the tensor-core scan (scan_impl 4) and on the list-major kernel
    (scan_impl 3)"""
    lens = [0, 1, 31, 32, 33, 127, 128, 129, 6000]
    probes = len(lens)
    case = Case(pv, "vector_l2_ops", 64, lens, 64, seed=23)
    try:
        want = case.want(probes, 40)
        for k in (10, 40):
            sub = (want[0][:, :k], want[1][:, :k])
            for l0, l1, slab in TC_ARMS:
                rested = case.l0_failed
                with options(pv, scan_impl=4, tc_level0=l0, tc_level1=l1, slab_select=slab):
                    got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
                case.check(got, sub, probes)
                assert r["filters"] > 0 and r["f1"] == 0, (k, l0, l1, slab, r)
                if not rested:
                    assert r["l0_queries"] == (case.q.shape[0] if (l0 and l1 and slab and k <= 10) else 0), (k, l0, l1, slab, r)
            with options(pv, scan_impl=3):
                got, r = traced(pv, case, lambda: case.ix.search(case.qe, k=k, probes=probes))
            case.check(got, sub, probes)
            assert r["filters"] == 0, r
    finally:
        case.free()
