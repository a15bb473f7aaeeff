"""CPU checks of the aggregate oracle (tests/aggregate_oracle.c): it reproduces the reference's known answers for
avg / sum of vector and halfvec, the Partial Aggregate result of test/t/018_aggregates.pl, and an independent numpy
statement of the run plan."""
import json
import math
import os

import numpy as np
import pytest

from tests import aggregate_oracle as A

KAT = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aggregate_kat.json")))


def _arg(a):
    if isinstance(a, dict):
        lo, hi = a["series"]
        return list(range(lo, hi + 1))
    return a


def _want_vals(half, want):
    return np.array(want, dtype=np.float32).astype(np.float16) if half else np.array(want, dtype=np.float32)


@pytest.mark.parametrize("run_rows", [0, 1, 2])
@pytest.mark.parametrize("case", KAT["table"], ids=lambda c: c["statement"])
def test_oracle_reproduces_the_table_kats(case, run_rows):
    half = case["type"] == "halfvec"
    agg = A.AVG if case["agg"] == "avg" else A.SUM
    rows = np.array(case["rows"], dtype=np.float32).reshape(-1, case["dim"])
    want = case["expect"]
    if isinstance(want, dict):
        with pytest.raises(A.AggregateError, match=f"^{want['error']}$"):
            A.table_aggregate(half, agg, rows, case["dim"], case["groups"], 1, run_rows)
        return
    vals, counts = A.table_aggregate(half, agg, rows, case["dim"], case["groups"], 1, run_rows)
    if want is None:
        assert counts[0] == 0
        return
    assert counts[0] == sum(g == 0 for g in case["groups"])
    np.testing.assert_array_equal(vals[0], _want_vals(half, want))


@pytest.mark.parametrize("case", KAT["calls"], ids=lambda c: c["statement"])
def test_oracle_reproduces_the_state_function_kats(case):
    half = case["type"] == "halfvec"
    fn = case["function"]
    args = [_arg(a) for a in case["args"]]
    want = case["expect"]

    def call():
        if fn.endswith("_avg"):
            return A.final_avg(half, args[0])
        if fn.endswith("_accum"):
            return A.accum(half, args[0], args[1])
        return A.combine(args[0], args[1])
    if isinstance(want, dict):
        with pytest.raises(A.AggregateError) as e:
            call()
        assert str(e.value) == want["error"]
        return
    got = call()
    if want is None:
        assert got is None
    elif fn.endswith("_avg"):
        np.testing.assert_array_equal(got, _want_vals(half, want))
    else:
        assert got == [float(w) for w in want]


def test_not_applicable_cases_are_the_dimension_mismatches():
    assert len(KAT["not_applicable"]) == 4
    assert all("dimensions" in c["reference"] for c in KAT["not_applicable"])


def rows_018(n=1_000_000, seed=18):
    """test/t/018_aggregates.pl's table: r_j = random() + {1.01, 2.01, 3.01} as real, v = ARRAY[r1, r2, r3]"""
    rng = np.random.default_rng(seed)
    return (rng.random((n, 3)) + np.array([1.01, 2.01, 3.01])).astype(np.float32)


def test_018_partial_aggregate_of_halfvec_sum():
    rows = rows_018()
    h = rows.astype(np.float16)     # v::halfvec (Float4ToHalf, round to nearest even; no value overflows)
    n = h.shape[0]
    want = KAT["partial_aggregate_018"]
    vals, _ = A.table_aggregate(True, A.SUM, h, 3, run_rows=math.ceil(n / want["participants"]))
    assert vals[0].astype(np.float32).tolist() == want["expect"]
    vals, _ = A.table_aggregate(True, A.SUM, h, 3, run_rows=0)
    assert vals[0].astype(np.float32).tolist() == [8192, 8192, 16384]


def test_018_serial_avg_is_the_float8_mean_of_each_column():
    rows = rows_018()
    vals, counts = A.table_aggregate(False, A.AVG, rows, 3, run_rows=0)
    want = (np.add.accumulate(rows.astype(np.float64), axis=0)[-1] / rows.shape[0]).astype(np.float32)
    np.testing.assert_array_equal(vals[0], want)
    assert counts[0] == rows.shape[0]
    assert abs(vals[0] - np.array([1.51, 2.51, 3.51], dtype=np.float32)).max() < 0.01


def numpy_plan(half, agg, rows, groups, ngroups, R):
    """the run plan in numpy: np.add.accumulate (sequential) in float64 / float32 / float16, run by run"""
    dim = rows.shape[1]
    vals = np.zeros((ngroups, dim), dtype=np.float16 if half else np.float32)
    counts = np.zeros(ngroups, dtype=np.int64)
    state = np.zeros((ngroups, dim + 1))
    sum_t = np.float16 if half else np.float32
    for g in range(ngroups):
        S = rows[groups == g]
        counts[g] = len(S)
        if not len(S):
            continue
        r = len(S) if R == 0 or R >= len(S) else R
        runs = [S[i:i + r] for i in range(0, len(S), r)]
        if agg == A.AVG:
            st = np.stack([np.add.accumulate(x.astype(np.float64), axis=0)[-1] for x in runs])
            s = np.add.accumulate(st, axis=0)[-1]
            m = (s / len(S)).astype(np.float32)
            vals[g] = m.astype(np.float16) if half else m
            state[g, 0], state[g, 1:] = len(S), s
        else:
            with np.errstate(over="ignore"):
                parts = [np.add.accumulate(x.astype(sum_t), axis=0) for x in runs]
                st = np.stack([p[-1] for p in parts])
                comb = np.add.accumulate(st, axis=0)
            if any(np.isinf(p).any() for p in parts) or np.isinf(comb).any():
                raise A.AggregateError("value out of range: overflow")
            vals[g] = comb[-1]
    return vals, counts, state


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("agg", [A.AVG, A.SUM])
@pytest.mark.parametrize("R", [0, 1, 3, 64, 1000])
def test_oracle_agrees_with_a_numpy_statement_of_the_plan(half, agg, R):
    rng = np.random.default_rng(7 + R)
    n, dim, ngroups = 3000, 5, 7
    rows = (rng.standard_normal((n, dim)) * (30 if half else 1e3)).astype(np.float32)
    rows[:50, 1] = -0.0
    if half:
        rows = rows.astype(np.float16)
    groups = rng.integers(-1, ngroups - 1, n).astype(np.int32)     # group ngroups - 1 stays empty
    want = numpy_plan(half, agg, rows.astype(np.float32) if not half else rows, groups, ngroups, R)
    if agg == A.AVG:
        vals, counts, st = A.table_aggregate(half, agg, rows, dim, groups, ngroups, R, state=True)
        np.testing.assert_array_equal(st, want[2])
    else:
        vals, counts = A.table_aggregate(half, agg, rows, dim, groups, ngroups, R)
    np.testing.assert_array_equal(counts, want[1])
    assert vals.tobytes() == want[0].tobytes()


def test_sum_overflow_is_decided_by_the_plan():
    a = np.array([[0], [3e38], [3e38], [-3e38]], dtype=np.float32)
    with pytest.raises(A.AggregateError, match="^value out of range: overflow$"):
        A.table_aggregate(False, A.SUM, a, 1, run_rows=0)
    vals, _ = A.table_aggregate(False, A.SUM, a, 1, run_rows=2)
    assert vals[0, 0] == np.float32(3e38)
    b = np.array([[0], [-3e38], [3e38], [3e38]], dtype=np.float32)
    vals, _ = A.table_aggregate(False, A.SUM, b, 1, run_rows=0)
    assert vals[0, 0] == np.float32(3e38)
    with pytest.raises(A.AggregateError, match="^value out of range: overflow$"):
        A.table_aggregate(False, A.SUM, b, 1, run_rows=2)
