"""Every search route against the oracle on hostile but legal values.

Most of the suite draws rows near the origin.  Here the laws are chosen where the project's arithmetic can part from
the reference's:

- offset(t): rows, queries and centres translated together by t * u (u a fixed unit direction, or the all-ones
  direction).  True distances do not move; the norm expansion |x|^2 + |q|^2 - 2 x.q of the tensor-core filters loses
  log2(t^2 / d) bits, so their bounds must fail and the exact path must answer.  At t = 1e6 along the ones direction
  the fp32 grid (0.0625) makes every L2 distance an exact sum, with ties by the hundred: the tie rule is under test.
- big-norm: a ball of radius ~1 around a centre with |c|^2 ~ 2e38 (each |x|^2 finite, |x|^2 + |q|^2 not), and one
  with |c|^2 > 3.4e38 (|x|^2 itself overflows).  The reference's (x - q)^2 stays small and finite in both.
- inf-distance: rows at +-3e38 in a few coordinates (L2 = +inf to every query; inner products of one sign only).
- NaN-distance: zero rows and zero queries under cosine, and rows whose inner-product terms overflow to +inf and -inf
  in different lanes of the per-query scan (the lane reduction adds the two infinities).
- zeros and ties: duplicate rows, rows orthogonal to the query (a negative inner product of -0.0), subnormals.
- halfvec: +-65504, subnormal halves, zero rows under cosine.  sparsevec: values up to 3e38, empty rows, tiny values.

Every value is legal: finite fp32 for vector and sparsevec, |h| <= 65504 for halfvec.

Assertions follow one rule.  A distance is asserted EXACTLY (bit for bit against the oracle) only where its fp32 result
does not depend on the summation order: a NaN term, an infinite term with no infinite term of the other sign, or terms
that are all exact fp32 values on a common grid whose total stays below 2^24 grid steps (every partial sum is then exact).
Everywhere else a result may lie anywhere in the interval `fp32_sum_interval` gives -- the exact fp64 sum of the terms
+- gamma_n * sum |terms| (+ n * 2^-150 for underflow), which holds for every summation order and for fused or separate
multiply-adds -- and every near-tie allowance in this file is derived from that interval.  Never an exact assertion on a
sum whose overflow depends on the order (such as 3e38 + -3e38 + 3e38), and none on products that overflow with both
signs: rounded separately they give inf + -inf = NaN, fused (as every kernel here and an FMA build of the reference
accumulate) the running +-inf absorbs the other product, so such a sum may be -inf, +inf or NaN.
"""
import math
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_headline import low_rank
from tests.util import build_ivf_arrays, f32_to_half_bits, half_bits_to_f32, mixture

U32 = 2.0 ** -24                 # unit roundoff of fp32
ETA = 2.0 ** -150                # the absolute error of one fp32 product that underflows
F32_MAX = float(np.finfo(np.float32).max)
HALF_MAX = 65504.0
THREADS = os.cpu_count() or 8
OFFSETS = [0.0, 1e2, 1e4, 1e6]
HOSTILE = (1e4, 1e6)             # offsets at which every tensor-core bound must fail


def tname(t):
    """the offset as law names spell it: 0, 1e2, 1e4, 1e6"""
    return "0" if t == 0 else f"1e{int(round(math.log10(t)))}"


# ----------------------------------------------------------------------------------------------------------- data laws

def direction(dim, kind):
    """the translation direction: a fixed unit vector, or all ones (t * ones moves every element by t)"""
    if kind == "ones":
        return np.ones(dim)
    u = np.random.default_rng(12345).standard_normal(dim)
    return u / np.linalg.norm(u)


def offset(x, t, kind):
    return (np.asarray(x, np.float64) + t * direction(x.shape[1], kind)).astype(np.float32)


def base_law(law, n, dim, seed):
    if law == "lowrank":
        return low_rank(n, dim, 16, seed=seed)
    return mixture(n, dim, 24, seed=seed)[0]


def offset_law(law, t, kind, n, nq, dim, seed):
    """(rows, queries) of the low-rank or the mixture law, translated by t along `kind`"""
    x = base_law(law, n + nq, dim, seed)
    y = offset(x, t, kind)
    return y[:n], y[n:]


def big_norm(n, nq, dim, seed, overflow=False):
    """a ball of radius ~1 around c = (a, a, 0, ...): |c|^2 = 2e38 (finite norms, overflowing |x|^2 + |q|^2) or 3.92e38
    (the norm overflows).  The ball lives in the other coordinates, where the fp32 grid still resolves it."""
    rng = np.random.default_rng(seed)
    a = 1.4e19 if overflow else 1.0e19
    x = rng.standard_normal((n + nq, dim)) / math.sqrt(dim)
    x[:, :2] = a
    x = x.astype(np.float32)
    return x[:n], x[n:]


def inf_rows(x, q, rows, seed):
    """rows at +3e38 in 3 coordinates, where every query is positive: (3e38 - q)^2 and 3e38 * q overflow to +inf for
    every query, so L2 = +inf and the inner product = +inf in any order"""
    rng = np.random.default_rng(seed)
    cols = rng.choice(x.shape[1], 3, replace=False)
    q = q.copy()
    q[:, cols] = np.abs(q[:, cols]) + 2.0
    x = x.copy()
    x[np.asarray(rows)[:, None], cols[None, :]] = 3e38
    return x, q


def halfvec_law(n, nq, dim, seed):
    """half values: +-65504, subnormal halves (6e-8), zeros, ordinary values; zero rows and one zero query (as float32
    arrays of exactly representable halves)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n + nq, dim)).astype(np.float32)
    m = rng.random(x.shape)
    x[m < 0.03] = HALF_MAX
    x[(m >= 0.03) & (m < 0.06)] = -HALF_MAX
    x[(m >= 0.06) & (m < 0.12)] = np.float32(6e-8)
    x[(m >= 0.12) & (m < 0.15)] = 0.0
    x = x.astype(np.float16).astype(np.float32)
    x[: n // 10] = 0.0
    x[n] = 0.0
    return x[:n], x[n:]


def zeros_and_ties(n, nq, dim, seed):
    """duplicate rows, rows orthogonal to every query (disjoint supports: a negative inner product of -0.0), zero rows,
    subnormal elements whose squares underflow (1e-40)"""
    rng = np.random.default_rng(seed)
    h = dim // 2
    x = np.zeros((n, dim), np.float32)
    x[:, h:] = rng.integers(-3, 4, (n, dim - h))            # small integers: exact sums
    x[rng.random(n) < 0.3, h:] = 0.0
    x[::7] = x[3]                                            # duplicates of row 3
    x[1::11, h:] = np.float32(1e-40)
    q = np.zeros((nq, dim), np.float32)
    q[:, :h] = rng.integers(-3, 4, (nq, h))                 # supports disjoint from the rows: orthogonal
    q[1::2, h:] = rng.integers(-2, 3, (nq // 2, dim - h))
    q[-1, :] = 0.0
    return x, q


def dense_laws(dim, n=600, nq=24):
    """name -> (rows, queries) of every dense vector law"""
    out = {}
    for law in ("lowrank", "mixture"):
        for t in OFFSETS:
            for kind in ("unit", "ones"):
                out[f"{law}-{tname(t)}-{kind}"] = offset_law(law, t, kind, n, nq, dim, seed=int(t) % 97 + dim)
    out["bignorm"] = big_norm(n, nq, dim, seed=5)
    out["bignorm-inf"] = big_norm(n, nq, dim, seed=6, overflow=True)
    x, q = offset_law("lowrank", 0.0, "unit", n, nq, dim, seed=7)
    out["inf"] = inf_rows(x, q, np.arange(0, n, 37), seed=7)
    out["zeros-ties"] = zeros_and_ties(n, nq, dim, seed=8)
    return out


# ----------------------------------------------------------------------------------------- rigorous fp32 sum interval

def _grid_exact(t, asum):
    """per row of terms t (exact fp32 values): every partial sum is exact in any order -- all terms are multiples of the
    smallest of their lowest set bits, and the sum of their magnitudes stays below 2^24 of those steps"""
    a = np.abs(t)
    with np.errstate(over="ignore"):
        ok = ((a <= F32_MAX) & (a.astype(np.float32).astype(np.float64) == a)).all(axis=1)
    f, e = np.frexp(np.where(a > 0, a, 1.0))
    m = np.ldexp(f, 24).astype(np.int64)                    # the 24-bit significand: |t| = m 2^(e - 24)
    low = np.where(a > 0, np.ldexp((m & -m).astype(np.float64), e - 24), np.inf)   # the lowest set bit of each term
    return ok & (asum < low.min(axis=1) * 2.0 ** 24)


def fp32_sum_interval(terms):
    """[lo, hi] (fp64, per row of `terms`) that contains the fp32 sum of the row's terms (the exact fp64 values of the
    products each side forms) for every summation order and either fused or separate multiply-adds; lo == hi where the
    result is order-independent (see the module docstring); NaN where it is NaN in every order"""
    t = np.atleast_2d(np.asarray(terms, np.float64))
    n = t.shape[1]
    pinf, ninf = np.isposinf(t).any(axis=1), np.isneginf(t).any(axis=1)
    nan = np.isnan(t).any(axis=1)
    both = pinf & ninf        # +inf and -inf terms: NaN when each product is rounded, +-inf when it is fused -- anything
    fin = np.where(np.isfinite(t), t, 0.0)
    asum = np.abs(fin).sum(axis=1)
    s = fin.sum(axis=1)                                     # exact where the grid rule holds (integers below 2^53)
    g = n * U32 / (1 - n * U32)
    b = g * asum + n * ETA + 2 * n * 2.0 ** -53 * asum      # (+ the fp64 rounding of s itself)
    exact = _grid_exact(fin, asum) | (asum <= ETA)          # (a sum of magnitudes under 2^-150 rounds to zero throughout)
    s = np.where(asum <= ETA, 0.0, s)
    lo = np.where(exact, _fl32(s), _fl32(s - b, -1))
    hi = np.where(exact, _fl32(s), _fl32(s + b, +1))
    lo = np.where(both, -np.inf, np.where(pinf, np.inf, np.where(ninf, -np.inf, lo)))
    hi = np.where(both, np.inf, np.where(pinf, np.inf, np.where(ninf, -np.inf, hi)))
    return np.where(nan, np.nan, lo), np.where(nan, np.nan, hi)


def _fl32(v, direction=0):
    """v rounded to fp32: to nearest, or (direction -1 / +1) to the nearest fp32 value at or below / above v.  An end of
    an interval beyond the largest float can only be met by a sum that overflowed: +-inf"""
    v = np.asarray(v, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = v.astype(np.float32)
        if direction < 0:
            f = np.where(f.astype(np.float64) > v, np.nextafter(f, np.float32(-np.inf)), f)
        if direction > 0:
            f = np.where(f.astype(np.float64) < v, np.nextafter(f, np.float32(np.inf)), f)
    out = f.astype(np.float64)
    if direction:
        out = np.where(np.abs(v) > F32_MAX, np.copysign(np.inf, v), out)
    return out


def _terms(metric, x, q):
    """the fp32 terms a pair sums: (x - q)^2 with x - q rounded to fp32, x q, |x - q|; exact in fp64.  Where fp32
    x - q is inexact the slack of that rounding is added (it is not order-dependent, but a kernel may form it otherwise)"""
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    if metric in (O.L2, O.L2_SQUARED, O.L1):
        with np.errstate(over="ignore", invalid="ignore"):
            d = (x - q).astype(np.float64)
        inexact = (d != x64 - q64) & np.isfinite(d)
        t = d * d if metric != O.L1 else np.abs(d)
        slack = np.where(inexact, (2 * U32 + U32 * U32) * t if metric != O.L1 else U32 * t, 0.0)
        return t, slack
    with np.errstate(over="ignore", invalid="ignore"):
        t = x64 * q64
    # an fp32 product beyond the fp32 range is +-inf whatever the order
    t = np.where(np.abs(t) >= 2.0 ** 128, np.copysign(np.inf, t), t)
    return t, np.zeros_like(t)


def sum_interval(metric, x, q):
    """fp32_sum_interval of the terms of rows x (or one row) against q: (lo, hi) arrays, or floats for one row"""
    one = np.ndim(x) == 1
    t, slack = _terms(metric, np.atleast_2d(x), q)
    lo, hi = fp32_sum_interval(t)
    sl = np.atleast_2d(slack).sum(axis=1)
    lo = np.where(sl > 0, _fl32(lo - sl, -1), lo)
    hi = np.where(sl > 0, _fl32(hi + sl, +1), hi)
    return (float(lo[0]), float(hi[0])) if one else (lo, hi)


def intervals(metric, rows, q):
    """[lo, hi] of the float8 the reference's operator returns for every row (float32) against query q, in any fp32
    order: (lo[n], hi[n])"""
    rows = np.atleast_2d(rows)
    if metric == O.COSINE:
        return _cosine_intervals(rows, q)
    lo, hi = sum_interval(metric, rows, q)
    if metric == O.L2:
        with np.errstate(invalid="ignore"):
            return np.sqrt(lo), np.sqrt(hi)
    if metric == O.NEG_IP:
        return -hi, -lo
    return lo, hi


def distance_interval(metric, x, q):
    lo, hi = intervals(metric, x, q)
    return float(lo[0]), float(hi[0])


def _cosine_intervals(x, q):
    """1 - clamp(ip / sqrt(|x|^2 |q|^2)) in fp64 from the three fp32 sums (src/vector.c:671-696).  With positive norms
    the quotient is monotone in each sum, so its extremes sit at the corners of the three intervals."""
    ip = sum_interval(O.IP, x, q)
    t, _ = _terms(O.IP, x, x)
    na = fp32_sum_interval(t)
    nb = tuple(np.full(len(x), v) for v in sum_interval(O.IP, q, q))
    vals = []
    with np.errstate(all="ignore"):
        for p in ip:
            for a in na:
                for b in nb:
                    s = p / np.sqrt(a * b)
                    vals.append(np.where(np.isnan(s), s, np.clip(s, -1.0, 1.0)))
    v = np.stack(vals)
    allnan, anynan = np.isnan(v).all(axis=0), np.isnan(v).any(axis=0)
    one = (ip[0] == ip[1]) & (na[0] == na[1]) & (nb[0] == nb[1])
    slo, shi = np.nanmin(np.where(anynan, 0.0, v), axis=0), np.nanmax(np.where(anynan, 0.0, v), axis=0)
    slo = np.where(one, slo, np.maximum(-1.0, slo - 4e-16 * np.abs(slo) - 1e-300))
    shi = np.where(one, shi, np.minimum(1.0, shi + 4e-16 * np.abs(shi) + 1e-300))
    lo, hi = 1.0 - shi, 1.0 - slo
    wide = ~one & (anynan | (na[0] <= 0) | (nb[0] <= 0))
    lo, hi = np.where(wide, 0.0, lo), np.where(wide, 2.0, hi)
    return np.where(allnan, np.nan, lo), np.where(allnan, np.nan, hi)


def inside(v, lo, hi, f32=False):
    """v within [lo, hi]; NaN matches NaN only.  f32: v is a float32 result, so the interval is widened to fp32"""
    v, lo, hi = np.asarray(v, np.float64), np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    if f32:
        lo = np.where(np.isfinite(lo), np.nextafter(lo.astype(np.float32), np.float32(-np.inf)).astype(np.float64), lo)
        hi = np.where(np.isfinite(hi), np.nextafter(hi.astype(np.float32), np.float32(np.inf)).astype(np.float64), hi)
        lo = np.where(np.isposinf(lo), F32_MAX, lo)   # an fp32 rounding of a huge double may be the largest float
    nan = np.isnan(lo)
    anything = np.isneginf(lo) & np.isposinf(hi)            # (includes NaN)
    return np.where(nan, np.isnan(v), anything | ((v >= lo) & (v <= hi)))


def same_values(a, b):
    """bit-for-bit equal up to -0 == +0, NaN equal to NaN"""
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


def same_as_returned(metric, got, want):
    """the top-k routes rank and return cosine distances as float32 keys (the other metrics' keys are the fp32 sums
    themselves, finished in fp64): equal to the oracle's float8 after that rounding"""
    if metric == O.COSINE:
        want = np.asarray(want, np.float64).astype(np.float32)
    return same_values(got, want)


# ------------------------------------------------------------------------------ top-k results under the fp32 bound

def _before(lo, hi, rank, a, b):
    """rows a (array) that must come before row b in every order the fp32 bound allows: smaller for sure, or both exact
    and equal (or both NaN) with a winning the tie.  NaN sorts after every number (float8 btree order)."""
    a = np.asarray(a)
    na, nb = np.isnan(lo[a]), bool(np.isnan(lo[b]))
    tie = rank[a] < rank[b]
    if nb:
        return ~na | tie
    exact = (lo[a] == hi[a]) & (lo[a] == lo[b]) & (lo[b] == hi[b])
    return ~na & ((hi[a] < lo[b]) | (exact & tie))


def check_topk(ids, dist, lo, hi, k, allowed=None, f32=False, tie_rule=True):
    """one query's top-k (ids, dist) against the intervals of every row: each distance lies in its row's interval, no
    pair is out of an order the bound forces, no row left out must have been in, and `-1 / +inf` padding follows the
    allowed rows.  Ties rank by position in `allowed` (ascending row numbers by default); tie_rule=False leaves exact
    ties unordered."""
    n = len(lo)
    allowed = np.arange(n) if allowed is None else np.asarray(allowed)
    rank = np.full(n, n + 1, dtype=np.int64)
    rank[allowed] = np.arange(len(allowed)) if tie_rule else 0
    m = min(k, len(allowed))
    ids, dist = np.asarray(ids), np.asarray(dist, np.float64)
    assert np.all(ids[m:] == -1) and np.all(np.isposinf(dist[m:])), (ids[m:], dist[m:])
    got = ids[:m]
    assert np.all(got >= 0) and len(set(got.tolist())) == m, got
    assert np.all(rank[got] <= n), "a row outside the allowed set"
    assert inside(dist[:m], lo[got], hi[got], f32).all(), [(int(i), dist[j], lo[i], hi[i]) for j, i in enumerate(got)
                                                            if not inside(dist[j], lo[i], hi[i], f32)][:5]
    if f32:     # the route ranks by float32 keys (cosine): values are compared after that rounding, equal keys are ties
        with np.errstate(over="ignore"):
            lo, hi = lo.astype(np.float32).astype(np.float64), hi.astype(np.float32).astype(np.float64)
    # in order: no later row is smaller for sure (suffix minimum of hi), NaN only at the end, exact ties by rank
    glo, ghi, nan = lo[got], hi[got], np.isnan(lo[got])
    assert not (nan[:-1] & ~nan[1:]).any(), "a number after a NaN"
    later = np.minimum.accumulate(np.where(nan, np.inf, ghi)[::-1])[::-1]
    bad = ~nan[:-1] & (later[1:] < glo[:-1])
    assert not bad.any(), ("out of order at", int(np.argmax(bad)))
    ex = np.flatnonzero((glo == ghi) | nan)
    same = (glo[ex[1:]] == glo[ex[:-1]]) | (nan[ex[1:]] & nan[ex[:-1]])
    assert not (same & (rank[got[ex[1:]]] < rank[got[ex[:-1]]])).any(), "an exact tie out of row order"
    if m:
        taken = np.zeros(n, bool)
        taken[got] = True
        out = allowed[~taken[allowed]]
        bad = _before(lo, hi, rank, out, got[-1])
        assert not bad.any(), ("left out", int(out[np.argmax(bad)]) if bad.any() else None, "before", int(got[-1]))


def exact_query(lo, hi, rows):
    return bool(np.all((lo[rows] == hi[rows]) | np.isnan(lo[rows])))


# -------------------------------------------------------------------------------------------- CPU checks of the helpers

@pytest.mark.parametrize("dim", [32, 128])
def test_laws_produce_only_legal_values(dim):
    for name, (x, q) in dense_laws(dim, n=300, nq=8).items():
        for a in (x, q):
            assert a.dtype == np.float32 and np.isfinite(a).all(), name
    x, q = halfvec_law(300, 8, dim, seed=1)
    for a in (x, q):
        assert np.isfinite(a).all() and np.abs(a).max() <= HALF_MAX
        assert np.array_equal(a.astype(np.float16).astype(np.float32), a), "halves round-trip"
    assert (half_bits_to_f32(f32_to_half_bits(x)) == x).all()
    xs, qs = sparse_law(200, 8, dim, seed=1)
    assert np.isfinite(xs).all() and np.isfinite(qs).all() and np.abs(xs).max() <= 3e38
    # the big-norm laws are what they claim: finite norms whose sum overflows, and an overflowing norm
    x, q = big_norm(50, 5, dim, seed=2)
    nx = np.array([float(np.sum(r.astype(np.float32) ** 2, dtype=np.float32)) for r in x])
    assert np.isfinite(nx).all() and (nx > 1.7e38).all() and (nx + nx > F32_MAX).all()
    x, _ = big_norm(50, 5, dim, seed=2, overflow=True)
    with np.errstate(over="ignore"):
        assert np.isinf(np.sum(x[0] * x[0], dtype=np.float32))


def _seq32(t):
    acc = np.float32(0)
    with np.errstate(over="ignore", invalid="ignore"):
        for v in t:
            acc = np.float32(acc + v)
    return float(acc)


def _orders(t):
    """fp32 sums of t in several orders: sequential, reversed, numpy's pairwise, sorted by magnitude both ways,
    and a few permutations"""
    t32 = np.asarray(t, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        out = [_seq32(t32), _seq32(t32[::-1]), float(np.sum(t32, dtype=np.float32)),
               _seq32(t32[np.argsort(np.abs(t32))]), _seq32(t32[np.argsort(-np.abs(t32))])]
        rng = np.random.default_rng(0)
        out += [_seq32(t32[rng.permutation(t32.size)]) for _ in range(4)]
    return out


def _fp32_products(metric, x, q):
    """the fp32 terms a plain fp32 loop forms (each product rounded)"""
    with np.errstate(over="ignore", invalid="ignore"):
        if metric == O.L2_SQUARED:
            d = x - q
            return d * d
        return x * q


@pytest.mark.parametrize("dim", [32, 128, 1536])
def test_order_independent_cases_are_order_independent(dim):
    """Where fp32_sum_interval says lo == hi, every summation order gives that one fp32 value (sequential, reversed,
    pairwise, sorted, shuffled); where it gives an interval, every order falls inside it."""
    exact_seen = 0
    for name, (x, q) in dense_laws(dim, n=40, nq=4).items():
        for metric in (O.L2_SQUARED, O.IP):
            for r in range(0, len(x), 7):
                lo, hi = sum_interval(metric, x[r], q[r % len(q)])
                sums = _orders(_fp32_products(metric, x[r], q[r % len(q)]))
                if lo == hi or (lo != lo):
                    exact_seen += 1
                    assert all(same_values(s, lo) for s in sums), (name, metric, r, lo, sums)
                else:
                    assert all(lo <= s <= hi for s in sums), (name, metric, r, lo, hi, sums)
    assert exact_seen > 20
    # the offset law at 1e6 along the ones direction is exact for L2 (the fp32 grid of the elements is 0.0625)
    x, q = offset_law("lowrank", 1e6, "ones", 20, 4, dim, seed=1)
    assert all(sum_interval(O.L2_SQUARED, x[i], q[0])[0] == sum_interval(O.L2_SQUARED, x[i], q[0])[1] for i in range(20))
    # same-sign overflowing products: +inf in any order; opposite signs: NaN in any order
    a = np.array([3e38, 1.0, -2.0, 3e38], np.float32)
    b = np.array([2.0, 1.0, 1.0, 5.0], np.float32)
    assert sum_interval(O.IP, a, b) == (math.inf, math.inf)
    with np.errstate(over="ignore"):
        assert all(s == math.inf for s in _orders(a * b))
    # products that overflow with both signs: NaN when rounded one by one, +-inf when fused -- never asserted exactly
    c = np.array([3e38, -3e38, 1.0], np.float32)
    assert sum_interval(O.IP, c, np.array([2.0, 2.0, 1.0], np.float32)) == (-math.inf, math.inf)
    assert all(s != s for s in _orders(np.float32([np.inf, -np.inf, 1.0])))
    # and the warning case: 3e38 + -3e38 + 3e38 depends on the order, so it gets an interval, never an exact value
    t = np.array([3e38, -3e38, 3e38], np.float64)
    lo, hi = fp32_sum_interval(t)
    assert lo < hi and len(set(_orders(t))) > 1
    # subnormal squares underflow in fp32: the interval is not exact but holds every order
    x = np.full(dim, 1e-40, np.float32)
    lo, hi = sum_interval(O.L2_SQUARED, x, np.zeros(dim, np.float32))
    assert lo <= 0.0 <= hi and all(lo <= s <= hi for s in _orders(_fp32_products(O.L2_SQUARED, x, np.zeros(dim, np.float32))))


def test_oracle_orders_nan_last_before_padding():
    """the oracle's exact top-k sorts NaN after +inf and pads with (-1, +inf) after the NaN results (float8 btree order,
    oracle/pgv_distance.c cmp_distid); its IVFFlat scan sorts NaN last too (pgv_ivfflat.c item_less)"""
    rng = np.random.default_rng(2)
    dim = 8
    x = rng.standard_normal((20, dim)).astype(np.float32)
    x[[3, 11]] = 0.0                         # cosine: 0 / 0
    x[[5, 6]] = 0.0
    x[5, 0] = x[6, 0] = 3e38                 # cosine: inf / sqrt(inf ...) = NaN; L2: +inf
    q = np.abs(rng.standard_normal(dim)).astype(np.float32) + 1
    ids, dist = O.exact_topk(O.VECTOR, O.COSINE, q, x, 25)
    assert list(ids[16:20]) == [3, 5, 6, 11] and np.isnan(dist[16:20]).all()
    assert np.all(ids[20:] == -1) and np.all(np.isposinf(dist[20:]))
    assert not np.isnan(dist[:16]).any()
    ids, dist = O.exact_topk(O.VECTOR, O.L2, q, x, 20)
    assert list(ids[18:]) == [5, 6] and np.isposinf(dist[18:]).all()
    # inner product NaN rows (+inf and -inf products): last in the IVFFlat scan order too
    x[7, :2] = (3e38, -3e38)
    centers = x[:2].copy()
    centers[:] = 1.0
    lists = np.zeros(20, np.int32)
    grouped, gids, off = build_ivf_arrays(x, lists, 2)
    oix = O.Ivf(O.VECTOR, O.NEG_IP, centers, off, grouped, gids)
    i, d, n = oix.search(q, 2, 0)
    assert n == 20 and int(i[-1]) == 7 and np.isnan(d[-1]) and not np.isnan(d[:-1]).any()


def test_intervals_hold_the_oracle():
    """the oracle's own distances (one fp32 order) lie in the intervals, for every metric and law"""
    for name, (x, q) in dense_laws(64, n=80, nq=3).items():
        for metric in (O.L2_SQUARED, O.L2, O.NEG_IP, O.IP, O.COSINE, O.L1):
            want = O.distance_batch(O.VECTOR, metric, q[0], x)
            lo, hi = intervals(metric, x, q[0])
            assert inside(want, lo, hi).all(), (name, metric)


# ------------------------------------------------------------------------------------------------------- sparse law

def sparse_law(n, nq, dim, seed):
    """dense images of sparsevec rows: values up to 3e38 (L2 overflows), empty rows (cosine NaN), tiny values"""
    rng = np.random.default_rng(seed)
    x = np.where(rng.random((n + nq, dim)) < 0.15, rng.standard_normal((n + nq, dim)), 0.0).astype(np.float32)
    x[rng.random((n + nq, dim)) < 0.01] = np.float32(1e-40)
    big = rng.choice(n, n // 20, replace=False)
    x[big, rng.integers(0, dim, big.size)] = 3e38
    x[rng.choice(n, n // 20, replace=False)] = 0.0
    x[n + 1] = 0.0
    return x[:n], x[n:]


# ===================================================================================================== GPU routes

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)
    for name, v in (("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2"))), ("tc_level0", 1), ("tc_level1", 1),
                    ("slab_select", 1), ("one_query", 1), ("tensor_cores", 1)):
        pv.set_option(name, v)


class options:
    """set library options for a block, restore the defaults after it"""
    DEFAULT = {"scan_impl": int(os.environ.get("VB_TEST_SCAN_IMPL", "2")), "tc_level0": 1, "tc_level1": 1, "slab_select": 1,
               "one_query": 1, "tensor_cores": 1}

    def __init__(self, pv, **kw):
        self.pv, self.kw = pv, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.pv.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            self.pv.set_option(k, self.DEFAULT[k])


DIST_METRICS = [O.L2_SQUARED, O.L2, O.NEG_IP, O.IP, O.COSINE, O.L1]


@gpu
@pytest.mark.parametrize("elem", [O.VECTOR, O.HALFVEC])
def test_distance_batch_every_metric_on_every_law(pv, elem):
    """distance_batch against the oracle: exact where the fp32 result is order-independent, inside the fp32 interval
    elsewhere, for every metric and law"""
    dim = 72
    laws = dense_laws(dim, n=160, nq=4) if elem == O.VECTOR else {"halfvec": halfvec_law(300, 6, dim, seed=3)}
    exact_seen = 0
    for name, (x, q) in laws.items():
        xe, qe = (x, q) if elem == O.VECTOR else (f32_to_half_bits(x), f32_to_half_bits(q))
        for metric in DIST_METRICS:
            for j in range(len(q)):
                got = pv.distance_batch(elem, metric, qe[j], xe)
                want = O.distance_batch(elem, metric, qe[j], xe)
                lo, hi = intervals(metric, x, q[j])
                exact = (lo == hi) | np.isnan(lo)
                exact_seen += int(exact.sum())
                assert same_values(got[exact], want[exact]), (name, metric, j)
                assert same_values(want[exact], lo[exact]), (name, metric, j, "the interval of an exact case")
                assert inside(got, lo, hi).all(), (name, metric, j, np.flatnonzero(~inside(got, lo, hi))[:5])
                assert inside(want, lo, hi).all(), (name, metric, j)
    assert exact_seen > 100


@gpu
def test_sparse_distance_batch_and_exact_topk(pv):
    """sparsevec distances and the exact scan on values up to 3e38, empty rows and tiny values"""
    S = pv.sparsevec
    dim = 96
    x, q = sparse_law(700, 6, dim, seed=4)
    rows = S.SparseRows.from_dense(x)
    t = S.SparseTable(dim).append(rows)
    for metric in (O.L2, O.NEG_IP, O.COSINE, O.L1):
        qs = [S.SparseVector.from_dense(v) for v in q]
        ids, dist = t.exact_topk(metric, qs, 720)
        for j, qv in enumerate(qs):
            got = S.distance_batch(metric, qv, rows)
            want = O.sparse_distance_batch(metric, (qv.indices, qv.values), rows.row_off, rows.idx, rows.val)
            lo, hi = intervals(metric, x, q[j])
            exact = (lo == hi) | np.isnan(lo)
            assert same_values(got[exact], want[exact]), (metric, j)
            assert inside(got, lo, hi).all() and inside(want, lo, hi).all(), (metric, j)
            check_topk(ids[j], dist[j], lo, hi, 720, f32=metric == O.COSINE)
    t.free()


def _table_laws(elem, dim, n, nq):
    if elem == O.HALFVEC:
        return {"halfvec": halfvec_law(n, nq, dim, seed=9)}
    laws = {}
    for law, t, kind in (("lowrank", 0.0, "unit"), ("lowrank", 1e2, "unit"), ("mixture", 1e4, "ones"), ("lowrank", 1e6, "ones"),
                         ("mixture", 1e6, "unit")):
        laws[f"{law}-{tname(t)}-{kind}"] = offset_law(law, t, kind, n, nq, dim, seed=11)
    laws["bignorm"] = big_norm(n, nq, dim, seed=12)
    laws["bignorm-inf"] = big_norm(n, nq, dim, seed=13, overflow=True)
    x, q = offset_law("lowrank", 0.0, "unit", n, nq, dim, seed=14)
    x, q = inf_rows(x, q, np.arange(5, n, 97), seed=14)
    x[np.arange(9, n, 89)] = 0.0                       # zero rows: cosine NaN
    x[np.arange(0, n, 50)] = x[2]                       # duplicates
    laws["inf-nan"] = (x, q)
    laws["zeros-ties"] = zeros_and_ties(n, nq, dim, seed=15)
    return laws


@gpu
@pytest.mark.parametrize("elem,dim,scan_impl", [(O.VECTOR, 128, 0), (O.VECTOR, 128, 1), (O.HALFVEC, 256, 0), (O.HALFVEC, 256, 1)])
def test_exact_topk_radix_segmented_and_padding(pv, elem, dim, scan_impl):
    """Table.exact_topk under the LDG (0) and bulk-copy (1) scans, k = 10 (radix selection), 2048, 2049 (segmented
    sort) and n + 5 (padding): ties to the smaller row id, NaN after +inf, (-1, +inf) padding after NaN; bit for bit the
    oracle's on order-independent queries"""
    n, nq = 3000, 4
    for name, (x, q) in _table_laws(elem, dim, n, nq).items():
        xe, qe = (x, q) if elem == O.VECTOR else (f32_to_half_bits(x), f32_to_half_bits(q))
        t = pv.Table(elem, dim).append(xe)
        for metric in (O.L2, O.NEG_IP, O.COSINE):
            bounds = [intervals(metric, x, q[j]) for j in range(nq)]
            for k in (10, 2048, 2049, n + 5):
                with options(pv, scan_impl=scan_impl):
                    ids, dist = t.exact_topk(metric, qe, k)
                for j in range(nq):
                    lo, hi = bounds[j]
                    check_topk(ids[j], dist[j], lo, hi, k, f32=metric == O.COSINE)
                    if exact_query(lo, hi, np.arange(n)) and metric != O.COSINE:   # (cosine ranks by float32 keys)
                        # -0.0 (an orthogonal row under negative inner product) comes back as +0.0: the float8 btree
                        # order and the tie rule treat them as one value, and == compares them equal
                        wi, wd = O.exact_topk(elem, metric, qe[j], xe, k)
                        assert np.array_equal(ids[j], wi) and same_as_returned(metric, dist[j], wd), (name, metric, k, j)
        t.free()


@gpu
def test_exact_topk_filtered_and_rerank(pv):
    """the filtered exact scan and the candidate re-rank on the same laws: the filter's rows in ascending order, the
    candidates in their given order, NaN rows allowed beside rejected ones"""
    dim, n, nq, k = 128, 2500, 4, 40
    rng = np.random.default_rng(21)
    for name, (x, q) in _table_laws(O.VECTOR, dim, n, nq).items():
        t = pv.Table(O.VECTOR, dim).append(x)
        allowed = np.sort(rng.choice(n, n // 3, replace=False))
        cand = np.stack([rng.permutation(n)[: 300] for _ in range(nq)]).astype(np.int64)
        cand[:, ::17] = -1
        f = t.filter(allowed)
        for metric in (O.L2, O.NEG_IP, O.COSINE):
            fi, fd = t.exact_topk(metric, q, k, filter=f)
            ri, rd = t.rerank(metric, q, cand, k)
            for j in range(nq):
                lo, hi = intervals(metric, x, q[j])
                check_topk(fi[j], fd[j], lo, hi, k, allowed=allowed, f32=metric == O.COSINE)
                c = cand[j][cand[j] >= 0]
                check_topk(ri[j], rd[j], lo, hi, k, allowed=c, f32=metric == O.COSINE)
                if exact_query(lo, hi, allowed):
                    wi, wd = O.exact_topk(O.VECTOR, metric, q[j], x[allowed], k)
                    assert np.array_equal(fi[j], np.where(wi >= 0, allowed[np.maximum(wi, 0)], -1)), (name, metric, j)
                    assert same_as_returned(metric, fd[j], wd)
        f.free()
        t.free()


# ------------------------------------------------------------------------------------------------------------- IVFFlat

IVF_DIM, IVF_N, IVF_LISTS, IVF_NQ, IVF_PROBES, IVF_K = 256, 16000, 32, 256, 8, 10
TC_ARMS = [(l0, l1, slab) for l0 in (1, 0) for l1 in (1, 0) for slab in (1, 0)]


def ivf_law(name, lists=IVF_LISTS):
    """(rows, queries, centres) of an IVFFlat law; the centres are rows of the law itself"""
    rng = np.random.default_rng(len(name))
    if name.startswith("bignorm"):
        x, q = big_norm(IVF_N, IVF_NQ, IVF_DIM, seed=31, overflow=name == "bignorm-inf")
    else:
        law, t, kind = name.split("-")
        x, q = offset_law(law, float(t), kind, IVF_N, IVF_NQ, IVF_DIM, seed=32)
    c = x[rng.choice(IVF_N, lists, replace=False)].copy()
    return x, q, c


def ivf_pair(pv, opclass, x, c):
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    assign = O.ivf_assign(elem, metric, x, c, threads=THREADS)
    grouped, ids, off = build_ivf_arrays(x, assign, len(c))
    return (lambda: pv.IvfflatIndex(opclass, x.shape[1], len(c)).load(c, off, grouped, ids)), O.Ivf(elem, metric, c, off, grouped, ids)


def ivf_intervals(metric, x, q):
    return [intervals(metric, x, q[j]) for j in range(len(q))]


def check_ivf(ids, dist, oix, x, q, metric, probes, k, f32=False, every=1):
    """every `every`-th query's result against the oracle's probed lists: the fp32 bound on every distance and order,
    and bit for bit the oracle's where the query's distances are order-independent"""
    sample = np.arange(0, len(q), every)
    ids, dist, q = ids[sample], dist[sample], q[sample]
    wi, wd = oix.search_batch(q, probes, k, threads=THREADS)
    for j in range(len(q)):
        lists, _ = oix.scan_lists(q[j], probes)
        probed = np.concatenate([oix.ids[oix.offsets[l]:oix.offsets[l + 1]] for l in lists])
        lo, hi = intervals(metric, x[probed], q[j])
        # positions of the probed rows: ties rank by (distance, list number) then position, as the oracle's total order
        pos = {int(r): i for i, r in enumerate(probed)}
        loc = np.array([pos[int(r)] if r >= 0 else -1 for r in ids[j]])
        check_topk(np.where(ids[j] >= 0, loc, -1), dist[j], lo, hi, k, f32=f32)
        if exact_query(lo, hi, np.arange(len(probed))):
            assert np.array_equal(ids[j], wi[j]) and same_values(dist[j], wd[j]), j


IVF_LAWS = [f"{law}-{tname(t)}-{kind}" for law in ("lowrank", "mixture") for t in OFFSETS for kind in ("unit", "ones")] + ["bignorm", "bignorm-inf"]


def same_as_an_exact_scan(got, base0, base3):
    """each query's row equals the per-query LDG scan's (scan_impl 0: what a certified filter result carries) or the
    list-major kernel's (scan_impl 3: what a batch the filter could not certify is re-run on), bit for bit"""
    for j in range(len(got[0])):
        if not any(np.array_equal(got[0][j], b[0][j]) and same_values(got[1][j], b[1][j]) for b in (base0, base3)):
            return False
    return True


def _hostile(name):
    return name.startswith("bignorm") or any(f"-{tname(t)}-" in name for t in HOSTILE)


@gpu
@pytest.mark.parametrize("name", IVF_LAWS)
def test_ivfflat_tensor_core_arms_equal_the_exact_scan(pv, name):
    """IvfflatIndex.search through the tensor-core list scan (scan_impl 4) under every combination of tc_level0,
    tc_level1 and slab_select equals an exact scan bit for bit -- per query, the per-query LDG scan (scan_impl 0) where
    the filter certified it, the list-major kernel (scan_impl 3) where the batch was re-run -- and both exact scans stay
    within the fp32 bound of the oracle.  On the hostile laws the bounds fail and the counters show the exact path answered
    (or, for an overflowing norm, the image reports non-finite and the filter never launches); on the t = 0 control
    no query needs the exact re-run."""
    x, q, c = ivf_law(name)
    make, oix = ivf_pair(pv, "vector_l2_ops", x, c)
    ix = make()
    with options(pv, scan_impl=0):
        base = ix.search(q, k=IVF_K, probes=IVF_PROBES)
    with options(pv, scan_impl=3):
        base3 = ix.search(q, k=IVF_K, probes=IVF_PROBES)
    # (the arms below are compared with the exact scans on every query; the oracle's bound is checked on a sample of them)
    check_ivf(base[0], base[1], oix, x, q, O.L2_SQUARED, IVF_PROBES, IVF_K, every=16)
    ix.free()
    pv.prof_enable(True)
    try:
        for l0, l1, slab in TC_ARMS:
            ix = make()          # a fresh image per arm: a level-1 failure rests level 1 for the next batches of an index
            with options(pv, scan_impl=4, tc_level0=l0, tc_level1=l1, slab_select=slab):
                pv.prof_read(pv.PROF_LIST_TC)
                got = ix.search(q, k=IVF_K, probes=IVF_PROBES)
                launches = pv.prof_read(pv.PROF_LIST_TC)[1]
            f0, f1, fx = ix.tc_level0_fallbacks(), ix.tc_level1_fallbacks(), ix.tc_fallbacks()
            ix.free()
            arm = (name, l0, l1, slab, f0, f1, fx, launches)
            assert same_as_an_exact_scan(got, base, base3), arm
            if fx == 0 and launches > 0:
                assert np.array_equal(got[0], base[0]) and np.array_equal(got[1], base[1]), arm
            if name == "bignorm-inf":
                assert launches == 0 and f0 == f1 == fx == 0, arm      # |x|^2 = inf: no bound, exact kernels only
                continue
            assert launches > 0, arm
            if _hostile(name):
                assert fx > 0, arm
                if l1 and l0 and slab:          # (level 0 selects from slab minima: it runs only with slab_select)
                    assert f0 > 0, arm
                if l1 and not l0:
                    assert f1 > 0, arm
            elif name.endswith("-0-unit") or name.endswith("-0-ones"):
                assert fx == 0, arm
    finally:
        pv.prof_enable(False)


@gpu
@pytest.mark.parametrize("name", ["lowrank-1e4-unit", "lowrank-1e6-ones", "bignorm"])
def test_ivfflat_inner_product_and_one_query(pv, name):
    """vector_ip_ops on the hostile laws through every scan arm, and the fused one-query kernels (batches of at most 16
    queries) against the exact scan"""
    x, q, c = ivf_law(name)
    make, oix = ivf_pair(pv, "vector_ip_ops", x, c)
    ix = make()
    with options(pv, scan_impl=0):
        base = ix.search(q, k=IVF_K, probes=IVF_PROBES)
        small = ix.search(q[:16], k=IVF_K, probes=IVF_PROBES)
    with options(pv, scan_impl=3):
        base3 = ix.search(q, k=IVF_K, probes=IVF_PROBES)
    with options(pv, scan_impl=4):
        got = ix.search(q, k=IVF_K, probes=IVF_PROBES)
    assert same_as_an_exact_scan(got, base, base3)
    for one in (1, 0):
        with options(pv, one_query=one, scan_impl=2):
            for m in (1, 5, 16):
                i, d = ix.search(q[:m], k=IVF_K, probes=IVF_PROBES)
                assert np.array_equal(i, small[0][:m]) and np.array_equal(d, small[1][:m]), (name, one, m)
    ix.free()
    # the one-query kernels on the L2 index too (their own distance arithmetic)
    make, oix = ivf_pair(pv, "vector_l2_ops", x, c)
    ix = make()
    with options(pv, scan_impl=0):
        small = ix.search(q[:16], k=IVF_K, probes=IVF_PROBES)
    with options(pv, one_query=1, scan_impl=2):
        i, d = ix.search(q[:16], k=IVF_K, probes=IVF_PROBES)
    assert np.array_equal(i, small[0]) and np.array_equal(d, small[1])
    check_ivf(i, d, oix, x, q[:16], O.L2_SQUARED, IVF_PROBES, IVF_K)
    ix.free()


@gpu
def test_ivfflat_filtered_allowed_nan_rows_beside_rejected_rows(pv):
    """search(filter=...) where allowed rows have NaN distances beside rejected rows (the masked run's has_nan path):
    an inner-product index whose "mixed" rows hold +3e38 in coordinate 0 and -3e38 in coordinate 64, against queries
    positive there.  The per-query LDG scan (scan_impl 0) sums the two coordinates in different lanes, so each lane
    overflows to one infinity and the lane reduction makes the distance NaN; a sequential fused chain (the list-major
    kernel) lets the first infinity absorb the second instead.  With scan_impl 0 the allowed NaN rows must come back
    after every allowed number and before the (-1, +inf) padding, and no rejected row may take their place."""
    rng = np.random.default_rng(41)
    dim, n, lists, nq = 128, 6000, 16, 20
    x, q = offset_law("mixture", 0.0, "unit", n, nq, dim, seed=41)
    q[:, [0, 64, 2]] = np.abs(q[:, [0, 64, 2]]) + 1.5     # 3e38 * 1.5 overflows on its own
    mixed = rng.choice(n, 60, replace=False)
    x[mixed, 0], x[mixed, 64] = 3e38, -3e38
    same_sign = rng.choice(np.setdiff1d(np.arange(n), mixed), 30, replace=False)
    x[same_sign, 2] = 3e38                                  # +inf in any order: NEG_IP = -inf
    c = x[rng.choice(np.setdiff1d(np.arange(n), np.concatenate([mixed, same_sign])), lists, replace=False)].copy()
    make, _ = ivf_pair(pv, "vector_ip_ops", x, c)
    ix = make()
    allowed = np.union1d(rng.choice(n, n // 4, replace=False), mixed[::2])
    nan_allowed = set(np.intersect1d(allowed, mixed).tolist())
    f = ix.filter(allowed)
    k = len(allowed) + 7
    with options(pv, scan_impl=0, one_query=0):
        fi, fd = ix.search(q, k=k, probes=lists, filter=f)
        ui, ud = ix.search(q, k=n + 5, probes=lists)        # the unfiltered order the filtered one restricts
    for j in range(nq):
        keep = np.isin(ui[j], allowed)
        wi, wd = ui[j][keep], ud[j][keep]
        nums = ~np.isnan(wd)
        m = int(nums.sum())
        assert set(wi[~nums].tolist()) == nan_allowed, j     # the allowed mixed rows are NaN for this scan
        # the allowed numbers first, as the unfiltered scan orders them (ties may fall either way between the two sorts)
        assert same_values(fd[j, :m], wd[:m]) and set(fi[j, :m].tolist()) == set(wi[:m].tolist()), j
        # then every allowed NaN row, then padding
        assert np.isnan(fd[j, m:len(allowed)]).all() and set(fi[j, m:len(allowed)].tolist()) == nan_allowed, j
        assert np.all(fi[j, len(allowed):] == -1) and np.isposinf(fd[j, len(allowed):]).all(), j
    f.free()
    ix.free()


@gpu
def test_ivfflat_filtered_tensor_core_scan_on_big_norms(pv):
    """search(filter=...) through the tensor-core list scan (scan_impl 4) on the big-norm law: every |x|^2 is finite, so
    the filter runs, but |x|^2 + |q|^2 - 2 x.q is inf - inf for the true neighbours.  The masked run must not certify
    them: the exact re-run answers (its counter rises), bit for bit an exact scan, and rejected rows never come back."""
    x, q, c = ivf_law("bignorm")
    make, _ = ivf_pair(pv, "vector_l2_ops", x, c)
    ix = make()
    allowed = np.random.default_rng(43).choice(IVF_N, IVF_N // 3, replace=False)
    f = ix.filter(allowed)
    out = {}
    for impl in (0, 3):
        with options(pv, scan_impl=impl):
            out[impl] = ix.search(q, k=IVF_K, probes=IVF_PROBES, filter=f)
    f.free()
    ix.free()
    ix = make()
    f = ix.filter(allowed)
    pv.prof_enable(True)
    try:
        with options(pv, scan_impl=4):
            pv.prof_read(pv.PROF_LIST_TC)
            got = ix.search(q, k=IVF_K, probes=IVF_PROBES, filter=f)
            launches = pv.prof_read(pv.PROF_LIST_TC)[1]
    finally:
        pv.prof_enable(False)
    fx = ix.tc_fallbacks()
    f.free()
    ix.free()
    assert launches > 0 and fx > 0, (launches, fx)
    assert same_as_an_exact_scan(got, out[0], out[3])
    assert np.isin(got[0], allowed).all()


@gpu
@pytest.mark.parametrize("name", ["lowrank-1e6-ones", "mixture-1e4-unit", "bignorm"])
def test_ivfflat_iterative_scan_pages(pv, name):
    """iterative_scan pages on the hostile laws.  The rows are scanned by the per-query chunk scan in every arm; what
    scan_impl 4 changes is the probe order of the 256 queries, selected through the tensor-core centre filter (160
    lists).  On these laws that filter cannot certify (its counter rises) and the exact centre scan answers: the pages
    equal the exact arm's bit for bit, and each query's sequence is its probed rows, each once"""
    x, q, c = ivf_law(name, lists=160)
    make, oix = ivf_pair(pv, "vector_l2_ops", x, c)
    qs = q[:256]
    seqs = {}
    pv.prof_enable(True)
    try:
        for impl in (0, 4):
            ix = make()
            with options(pv, scan_impl=impl):
                pv.prof_read(pv.PROF_CENTRE_TC)
                with ix.iterative_scan(qs, probes=2, max_probes=4, page=64) as s:
                    pages = []
                    for _ in range(200):
                        i, d, cnt = s.next_batch()
                        if not cnt.any():
                            break
                        pages.append((i.copy(), d.copy(), cnt.copy()))
                launches = pv.prof_read(pv.PROF_CENTRE_TC)[1]
            seqs[impl] = pages
            if impl == 4:
                assert launches > 0 and ix.tc_fallbacks() > 0, (launches, ix.tc_fallbacks())
            ix.free()
    finally:
        pv.prof_enable(False)
    assert len(seqs[0]) == len(seqs[4])
    for a, b in zip(seqs[0], seqs[4]):
        assert np.array_equal(a[2], b[2])
        for j in range(len(qs)):
            assert np.array_equal(a[0][j, :a[2][j]], b[0][j, :b[2][j]]) and same_values(a[1][j, :a[2][j]], b[1][j, :b[2][j]])
    for j in (0, 77, 255):
        got = np.concatenate([p[0][j, :p[2][j]] for p in seqs[0]])
        lists, _ = oix.scan_lists(qs[j], 4)
        probed = np.concatenate([oix.ids[oix.offsets[l]:oix.offsets[l + 1]] for l in lists])
        assert sorted(got.tolist()) == sorted(probed.tolist())


@gpu
@pytest.mark.parametrize("lists", [160, 3000])
@pytest.mark.parametrize("name", ["mixture-1e4-ones", "mixture-1e6-ones", "bignorm", "mixture-0-unit"])
def test_probe_selection_on_translated_and_big_norm_centres(pv, name, lists):
    """GetScanLists for 320 queries over >= 128 centres (the tensor-core probe path) on translated and big-norm centres:
    the probed lists and their order as the fp32 bound allows, bit for bit the oracle's where exact, and the exact
    kernels' (scan_impl 3) lists everywhere.  The filter's fallback counter rises on the hostile centres and stays at
    zero on the control."""
    dim = 48
    if name == "bignorm":
        x, q = big_norm(12000, 320, dim, seed=51)
    else:
        law, t, kind = name.split("-")
        x, q = offset_law(law, float(t), kind, 12000, 320, dim, seed=52)
    rng = np.random.default_rng(lists)
    c = x[rng.choice(len(x), lists, replace=False)].copy()
    make, oix = ivf_pair(pv, "vector_l2_ops", x, c)
    ix = make()
    pv.prof_enable(True)
    try:
        with options(pv, scan_impl=3):
            l3, d3 = ix.scan_lists(q, 7)
        with options(pv, scan_impl=4):
            pv.prof_read(pv.PROF_CENTRE_TC)
            f0 = ix.tc_fallbacks()
            l4, d4 = ix.scan_lists(q, 7)
            launches = pv.prof_read(pv.PROF_CENTRE_TC)[1]
            fx = ix.tc_fallbacks() - f0
    finally:
        pv.prof_enable(False)
    assert launches > 0
    if name == "mixture-0-unit":
        assert fx == 0, fx        # the control certifies: l4 came from the filter itself
    else:
        assert fx > 0, fx         # the bound fails and the exact centre scan answers
    assert np.array_equal(l3, l4)
    for j in range(0, 320, 8):
        lo, hi = intervals(O.L2_SQUARED, c, q[j])
        check_topk(l4[j], d4[j], lo, hi, 7)
        if exact_query(lo, hi, np.arange(lists)):
            wl, wd = oix.scan_lists(q[j], 7)
            assert np.array_equal(l4[j], wl) and same_values(d4[j], wd), j
    ix.free()


@gpu
@pytest.mark.parametrize("name", ["lowrank-0-unit", "lowrank-1e2-unit", "lowrank-1e4-ones", "lowrank-1e6-ones", "mixture-1e4-unit",
                                  "bignorm", "bignorm-inf", "inf"])
@pytest.mark.parametrize("metric", [O.L2_SQUARED, O.NEG_IP])
def test_assign_with_and_without_tensor_cores(pv, name, metric):
    """pv.assign equals the oracle's AddTupleToSort loop (strict < against DBL_MAX, src/ivfbuild.c:165-190): rows whose
    distance to every centre is +inf (or -inf) go to list 0.  The tensor-core pass re-checks exactly every row
    its bound cannot separate: nearly all of them on the hostile laws, few on the control."""
    dim, n, k = 96, 4096, 40
    rng = np.random.default_rng(61)
    if name.startswith("bignorm"):
        x, _ = big_norm(n, 1, dim, seed=62, overflow=name == "bignorm-inf")
    elif name == "inf":
        x, _ = offset_law("mixture", 0.0, "unit", n, 1, dim, seed=63)
        x[::9, :3] = 3e38                # (3e38 - c)^2 and 3e38 c overflow to +inf against every (positive) centre
    else:
        law, t, kind = name.split("-")
        x, _ = offset_law(law, float(t), kind, n, 1, dim, seed=64)
    if name == "inf":
        c = np.abs(x[rng.choice(np.flatnonzero(np.arange(n) % 9), k, replace=False)]) + 1.0
    else:
        c = x[rng.choice(n, k, replace=False)].copy()
    want = O.ivf_assign(O.VECTOR, metric, x, c, threads=THREADS)
    t = pv.Table(O.VECTOR, dim).append(x)
    got = {}
    for tc in (1, 0):
        with options(pv, tensor_cores=tc):
            got[tc] = pv.assign(t, metric, c)
            rechecked = pv.last_assign_rechecked()
        if tc and _hostile(name):
            assert rechecked > n // 2, (name, rechecked)
        if tc and name == "lowrank-0-unit":
            assert 0 <= rechecked < n // 10, (name, rechecked)
    t.free()
    for tc in (1, 0):
        if np.array_equal(got[tc], want):
            continue
        # only rows whose two nearest centres are within the fp32 bound may differ
        for r in np.flatnonzero(got[tc] != want):
            lo, hi = intervals(metric, c, x[r])
            a, b = int(got[tc][r]), int(want[r])
            assert not np.isnan(lo[a]), (name, tc, r, a, "a NaN distance won")
            assert not (hi[b] < lo[a]) and not (lo[a] == hi[a] == lo[b] == hi[b]), (name, tc, r, a, b, lo[a], hi[a], lo[b], hi[b])
    if name == "inf":     # every distance +inf (L2) or -inf (negative inner product): the first centre, list 0
        assert (want[::9] == 0).all() and (got[1][::9] == 0).all() and (got[0][::9] == 0).all()


@gpu
def test_in_place_insert_and_delete_keep_the_finite_flag_as_a_load_does(pv):
    """an insert of a row whose |x|^2 overflows turns the tensor-core list scan off for the whole index, as a load with
    that row does; deleting it turns it back on; results equal the exact scan throughout"""
    x, q, c = ivf_law("lowrank-0-unit")
    make, _ = ivf_pair(pv, "vector_l2_ops", x, c)
    ix = make()
    big = x[:3].copy()
    big[:, 0] = 2e19
    pv.prof_enable(True)

    def arms():
        with options(pv, scan_impl=0):
            base = ix.search(q, k=IVF_K, probes=IVF_PROBES)
        with options(pv, scan_impl=3):
            base3 = ix.search(q, k=IVF_K, probes=IVF_PROBES)
        with options(pv, scan_impl=4):
            pv.prof_read(pv.PROF_LIST_TC)
            got = ix.search(q, k=IVF_K, probes=IVF_PROBES)
            launches = pv.prof_read(pv.PROF_LIST_TC)[1]
        assert same_as_an_exact_scan(got, base, base3)
        return launches

    try:
        assert arms() > 0
        ix.insert(big, np.array([10**9, 10**9 + 1, 10**9 + 2]))
        assert arms() == 0
        assert ix.delete(np.array([10**9, 10**9 + 1, 10**9 + 2])) == 3
        assert arms() > 0
    finally:
        pv.prof_enable(False)
    ix.free()


@gpu
@pytest.mark.parametrize("t", [0.0, 1e6])
def test_hnsw_search_on_an_oracle_graph_under_the_offset_law(pv, t):
    """HNSW search on an oracle-built graph of translated rows: at t = 1e6 along the ones direction every distance is an
    exact fp32 sum, so the walk, its distance count and its results equal the oracle's bit for bit"""
    x, q = offset_law("lowrank", t, "ones", 3000, 64, 32, seed=71)
    og = O.Hnsw(O.VECTOR, O.L2_SQUARED, x, m=16, ef_construction=64, seed=7)
    g = og.export()
    gi = pv.HnswIndex("vector_l2_ops", 32, m=16).load(x[g["elem_row"]], g["levels"], g["nbr0"], g["upper_off"], g["upper"], g["entry"])
    ids, dist, nd = gi.search(q, k=10, ef_search=40)
    wi, wd, wnd = og.search_batch(q, 40, 10, ties=O.TIES_TOTAL, threads=THREADS)
    if t:
        assert np.array_equal(ids, wi) and same_values(dist, wd) and np.array_equal(nd, wnd)
    else:
        same_q = np.all(ids == wi, axis=1)
        assert same_q.mean() > 0.95
        erows = x[g["elem_row"]]
        for j in range(len(q)):
            lo, hi = intervals(O.L2_SQUARED, erows[ids[j]], q[j])
            assert inside(dist[j], lo, hi, f32=True).all(), j
    gi.free()
