"""avg / sum of vector and halfvec rows on the GPU (vb_table_aggregate): the reference's known answers, test/t/018's
serial and Partial Aggregate results, bit identity with the oracle's run plan (results, counts, float8 states) over
types, dimensions, run lengths and groupings, -0, overflow decided by the plan, the _dev variant, and the errors."""
import ctypes as C
import math
import re

import numpy as np
import pytest

from tests import aggregate_oracle as A
from tests.test_aggregate_oracle import KAT, _want_vals, rows_018

pytestmark = pytest.mark.gpu
EINVAL, ENOMEM = -1, -4


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def table(pv, half, rows):
    rows = np.asarray(rows)
    t = pv.Table(pv.HALFVEC if half else pv.VECTOR, rows.shape[1])
    if rows.shape[0]:
        t.append(rows.astype(np.float16) if half and rows.dtype != np.float16 else rows)
    return t


def device_agg(t, agg, groups, ngroups, R, state=False):
    return t.avg(groups, ngroups, run_rows=R, state=state) if agg == A.AVG else t.sum(groups, ngroups, run_rows=R)


@pytest.mark.parametrize("run_rows", [0, 1, 2])
@pytest.mark.parametrize("case", KAT["table"], ids=lambda c: c["statement"])
def test_table_kats(pv, case, run_rows):
    import torch
    half = case["type"] == "halfvec"
    agg = A.AVG if case["agg"] == "avg" else A.SUM
    rows = np.array(case["rows"], dtype=np.float32).reshape(-1, case["dim"])
    t = table(pv, half, rows)
    groups = np.array(case["groups"], dtype=np.int32)
    want = case["expect"]
    for g in (groups, torch.from_numpy(groups).cuda()):
        if isinstance(want, dict):
            with pytest.raises(pv.VecB200Error, match=want["error"]) as e:
                device_agg(t, agg, g, 1, run_rows)
            assert e.value.code == EINVAL and str(e.value).endswith(want["error"])
            continue
        vals, counts = device_agg(t, agg, g, 1, run_rows)
        vals, counts = (vals.cpu().numpy(), counts.cpu().numpy()) if torch.is_tensor(vals) else (vals, counts)
        if want is None:
            assert counts[0] == 0 and not vals.any()
        else:
            assert counts[0] == (groups == 0).sum()
            np.testing.assert_array_equal(vals[0], _want_vals(half, want))


@pytest.mark.parametrize("half", [False, True])
def test_state_kats_through_a_table(pv, half):
    """vector_accum('{0}', '[1,2,3]') = {1,1,2,3}: the state of a one-row table; '{2,2,4,6}' is the state of two rows
    [1,2,3] and vector_avg of it [1,2,3]"""
    t = table(pv, half, np.array([[1, 2, 3]], np.float32))
    _, _, st = t.avg(state=True)
    assert st[0].tolist() == [1, 1, 2, 3]
    t = table(pv, half, np.array([[1, 2, 3], [1, 2, 3]], np.float32))
    for R in (0, 1):
        vals, _, st = t.avg(run_rows=R, state=True)
        assert st[0].tolist() == [2, 2, 4, 6]
        np.testing.assert_array_equal(vals[0], _want_vals(half, [1, 2, 3]))


def test_018_on_the_device(pv):
    rows = rows_018()
    n = rows.shape[0]
    th = table(pv, True, rows.astype(np.float16))
    vals, _ = th.sum(run_rows=math.ceil(n / 3))
    assert vals[0].astype(np.float32).tolist() == KAT["partial_aggregate_018"]["expect"]
    vals, _ = th.sum(run_rows=0)
    assert vals[0].astype(np.float32).tolist() == [8192, 8192, 16384]
    tv = table(pv, False, rows)
    vals, counts = tv.avg(run_rows=0)
    want = (np.add.accumulate(rows.astype(np.float64), axis=0)[-1] / n).astype(np.float32)   # avg(r_j)::float4
    np.testing.assert_array_equal(vals[0], want)
    assert counts[0] == n


def make_groups(kind, n, rng):
    if kind == "none":
        return None, 1
    if kind == "one_with_excluded":
        return np.where(rng.random(n) < 0.3, -1, 0).astype(np.int32), 1
    if kind == "skewed37":
        return np.minimum(36, np.floor(-np.log(rng.random(n)) * 6)).astype(np.int32), 37
    # 5000 groups, mostly empty: rows fall in 60 of them, a tenth are excluded
    used = rng.choice(5000, 60, replace=False)
    g = used[rng.integers(0, 60, n)].astype(np.int32)
    g[rng.random(n) < 0.1] = -1
    return g, 5000


@pytest.mark.parametrize("groups_kind", ["none", "one_with_excluded", "skewed37", "sparse5000"])
@pytest.mark.parametrize("dim", [1, 3, 17, 768, 1536])
@pytest.mark.parametrize("half", [False, True])
def test_bit_identical_to_the_oracle_plan(pv, half, dim, groups_kind):
    import torch
    rng = np.random.default_rng(dim * 7 + len(groups_kind))
    n = min(300_000, max(2000, 3_000_000 // dim))
    rows = (rng.standard_normal((n, dim)) * (4 if half else 100)).astype(np.float32)
    if half:
        rows = rows.astype(np.float16)
    t = table(pv, half, rows)
    groups, ng = make_groups(groups_kind, n, rng)
    gdev = torch.from_numpy(groups).cuda() if groups is not None else None
    for agg in (A.AVG, A.SUM):
        for R in (0, 1, 5, 1000, n):
            try:
                want = A.table_aggregate(half, agg, rows, dim, groups, ng, R, state=agg == A.AVG)
            except A.AggregateError as e:
                with pytest.raises(pv.VecB200Error, match=str(e)):
                    device_agg(t, agg, groups, ng, R)
                continue
            got = device_agg(t, agg, groups, ng, R, state=True) if agg == A.AVG else device_agg(t, agg, groups, ng, R)
            assert got[0].tobytes() == want[0].tobytes(), (agg, R)
            np.testing.assert_array_equal(got[1], want[1])
            if agg == A.AVG:
                assert got[2].tobytes() == want[2].tobytes(), (agg, R)
            if gdev is not None and R in (0, 5):     # the _dev variant gives the host variant's bytes
                dg = device_agg(t, agg, gdev, ng, R, state=True) if agg == A.AVG else device_agg(t, agg, gdev, ng, R)
                for a, b in zip(dg, got):
                    assert a.cpu().numpy().tobytes() == b.tobytes()


@pytest.mark.parametrize("half", [False, True])
def test_negative_zero_columns_stay_negative_zero(pv, half):
    n = 1000
    rows = np.zeros((n, 4), np.float32)
    rows[:, 1] = -0.0
    rows[:, 3] = -0.0
    rows[:, 2] = 1.0
    t = table(pv, half, rows)
    for R in (0, 1, 2, 7, 999, n):
        for agg in (A.AVG, A.SUM):
            vals, _ = device_agg(t, agg, None, 1, R)
            v = vals[0].astype(np.float32)
            assert np.signbit(v[1]) and np.signbit(v[3]) and v[1] == 0 and v[3] == 0, (agg, R)
            assert not np.signbit(v[0])


def test_overflow_is_decided_by_the_plan(pv):
    lib = pv.load()
    a = table(pv, False, np.array([[0], [3e38], [3e38], [-3e38]], np.float32))
    b = table(pv, False, np.array([[0], [-3e38], [3e38], [3e38]], np.float32))
    for t, fails in ((a, {0: True, 2: False}), (b, {0: False, 2: True})):
        rows = np.array([[0], [3e38], [3e38], [-3e38]] if t is a else [[0], [-3e38], [3e38], [3e38]], np.float32)
        for R, f in fails.items():
            oracle_fails = False
            try:
                A.table_aggregate(False, A.SUM, rows, 1, run_rows=R)
            except A.AggregateError:
                oracle_fails = True
            assert oracle_fails == f
            out = np.full((1, 1), 7.0, np.float32)
            cnt = np.full(1, 7, np.int64)
            rc = lib.vb_table_aggregate(t.h, A.SUM, None, 1, R, out.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), None)
            if f:
                assert rc == EINVAL and lib.vb_last_error().decode() == "value out of range: overflow"
                assert out[0, 0] == 7.0 and cnt[0] == 7            # the host variant writes nothing
            else:
                assert rc == 0 and out[0, 0] == np.float32(3e38) and cnt[0] == 4
    # halfvec: 65504 + 65504 overflows serially; [65504, -65504 | 65504] does not at R = 2
    h = table(pv, True, np.array([[65504], [-65504], [65504]], np.float32))
    vals, _ = h.sum(run_rows=2)
    assert vals[0, 0] == np.float16(65504)


def test_empty_table_and_empty_groups(pv):
    for half in (False, True):
        t = pv.Table(pv.HALFVEC if half else pv.VECTOR, 5)
        for agg in (A.AVG, A.SUM):
            vals, counts = device_agg(t, agg, None, 1, 0)
            assert counts.tolist() == [0] and not vals.any()
            vals, counts = device_agg(t, agg, np.zeros(0, np.int32), 3, 4)
            assert counts.tolist() == [0, 0, 0] and not vals.any()


def test_validation_errors(pv):
    lib = pv.load()
    t = table(pv, False, np.ones((10, 4), np.float32))
    out = np.zeros((8, 4), np.float32)
    cnt = np.zeros(8, np.int64)
    st = np.zeros((8, 5))
    g = np.zeros(10, np.int32)
    P = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)   # noqa: E731

    def call(agg=A.AVG, groups=None, ng=1, R=0, state=None):
        rc = lib.vb_table_aggregate(t.h, agg, P(groups), ng, R, P(out), P(cnt), P(state))
        return rc, lib.vb_last_error().decode()
    assert call(agg=2) == (EINVAL, "vb_table_aggregate: unknown aggregate 2 (VB_AGG_AVG or VB_AGG_SUM)")
    assert call(ng=0, groups=g)[0] == EINVAL and "ngroups = 0" in call(ng=0, groups=g)[1]
    assert call(R=-1)[0] == EINVAL and "run_rows = -1" in call(R=-1)[1]
    assert call(ng=2)[0] == EINVAL and "group_of_row is NULL" in call(ng=2)[1]
    assert call(agg=A.SUM, state=st)[0] == EINVAL and "out_state = NULL" in call(agg=A.SUM, state=st)[1]
    bad = g.copy()
    bad[6] = 8
    assert call(groups=bad, ng=8) == (EINVAL, "vb_table_aggregate: group_of_row[6] = 8 is not a group (-1..7)")
    bad[6] = -2
    assert call(groups=bad, ng=8)[1] == "vb_table_aggregate: group_of_row[6] = -2 is not a group (-1..7)"
    tb = pv.Table(pv.BIT, 16)
    rc = lib.vb_table_aggregate(tb.h, A.AVG, None, 1, 0, P(out), P(cnt), None)
    assert rc == EINVAL and "bit has no aggregates" in lib.vb_last_error().decode()
    # an ngroups x dim far beyond device memory: VB_ENOMEM naming the bytes, nothing written
    wide = table(pv, False, np.ones((10, 1536), np.float32))
    ng = 1 << 23
    rc = lib.vb_table_aggregate(wide.h, A.AVG, P(g), ng, 0, P(out), P(cnt), P(st))
    msg = lib.vb_last_error().decode()
    assert rc == ENOMEM, msg
    need = int(re.search(r"needs (\d+) bytes", msg).group(1))
    assert need >= ng * 1536 * 4 + ng * 1537 * 8 and "staged results" in msg
    assert not out.any() and not cnt.any()


def test_dev_variant_ignores_out_of_range_groups(pv):
    import torch
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((5000, 33)).astype(np.float32)
    t = table(pv, False, rows)
    g = rng.integers(-1, 4, 5000).astype(np.int32)
    bad = g.copy()
    bad[::7] = 9
    bad[1::11] = -5
    clean = np.where((bad >= 0) & (bad < 4), bad, -1).astype(np.int32)
    for agg in (A.AVG, A.SUM):
        want = device_agg(t, agg, clean, 4, 100)
        got = device_agg(t, agg, torch.from_numpy(bad).cuda(), 4, 100)
        for a, b in zip(got, want):
            assert a.cpu().numpy().tobytes() == b.tobytes()
