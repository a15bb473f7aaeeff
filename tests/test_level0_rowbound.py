"""Per-row error bound of filter level 0 (vb_list_tc.cu: pack_rows_i8_kernel's R_x, l0_query_kernel's coefficients and the
level-0 refine's E_i): for rows with mixed int8 residuals -- ordinary rows, rows with one spike coordinate, huge and zero
rows -- the fp32 d~ of the level-0 epilogue is within E(x, q) of the float64 distance, for L2 and the inner product.
E is evaluated here in round-to-nearest fp32, which is below the kernel's round-up evaluation, so the check is the
stricter one.  No GPU needed."""
import numpy as np
import pytest

f32 = np.float32


def up(v):
    """float64 -> the smallest fp32 >= v (__double2float_ru)"""
    r = np.float32(v)
    return np.where(r.astype(np.float64) < v, np.nextafter(r, np.float32(np.inf)), r).astype(np.float32)


def quant_rows(x):
    amax = np.abs(x).max(axis=1).astype(f32)
    sx = (amax / f32(127)).astype(f32)
    safe = np.where(sx > 0, sx, f32(1))
    x8 = np.where(sx[:, None] > 0, np.clip(np.rint((x / safe[:, None]).astype(f32)), -127, 127), 0).astype(f32)
    res = np.sqrt(((x.astype(np.float64) - sx[:, None].astype(np.float64) * x8) ** 2).sum(1))
    r8 = up(res * (1.0 + 1.0 / 1048576.0))
    xn = (x * x).sum(1, dtype=f32)
    return sx, x8, r8, xn


def quant_query(q):
    tq = f32(np.abs(q).max() / f32(127))
    h = np.clip(np.rint((q / tq).astype(f32)), -127, 127).astype(f32)
    r = (q.astype(np.float64) - np.float64(tq) * h).astype(f32)                      # fma(-t_q, h, q)
    lo = np.clip(np.rint(((r * f32(254)).astype(f32) / tq).astype(f32)), -127, 127).astype(f32)
    return tq, h, lo


def coefficients(q, tq, h, lo, is_l2, c_sum):
    """l0_query_kernel: (a, b, c, d) of E = a R_x + b X_x + c X_x^2 + d, and eps(q) with the global rmax / xmax"""
    qd = q.astype(np.float64)
    n2 = float((qd * qd).sum())
    qnorm = np.sqrt(n2)
    rq = np.sqrt(((qd - np.float64(tq) * (h.astype(np.float64) + lo.astype(np.float64) / 254.0)) ** 2).sum())
    qabs = float(tq) * (np.sqrt((h.astype(np.float64) ** 2).sum()) + np.sqrt((lo.astype(np.float64) ** 2).sum()) / 254.0)
    w, dq = 1.0 + 1.0 / 1024.0, rq + qabs / 1048576.0
    ca = 2.0 * qnorm if is_l2 else qnorm
    cb = 2.0 * dq if is_l2 else dq + qnorm / 131072.0
    cc = float(c_sum) if is_l2 else 0.0
    cd = 2e-30 + float(c_sum) * n2 if is_l2 else 1e-30
    coef = tuple(f32(v * w) for v in (ca, cb, cc, cd))

    def eps(xmax, rmax):
        X = xmax * w + rmax
        dot = rmax * qnorm + X * rq + X * qabs / 1048576.0 + 1e-30
        return (2.0 * dot + float(c_sum) * (X * X + n2) if is_l2 else dot + X * qnorm / 131072.0) * w
    return coef, eps


@pytest.mark.parametrize("is_l2", [True, False])
def test_level0_per_row_bound_holds(is_l2):
    rng = np.random.default_rng(7)
    n, dim, nq = 600, 384, 12
    c_sum = f32(max(1.0 / 65536.0, 3.0 * (dim / 32.0 + 8.0) / 16777216.0))
    basis = rng.standard_normal((16, dim)).astype(f32)
    x = (rng.standard_normal((n, 16)).astype(f32) @ basis / 4.0).astype(f32)
    x += 0.05 * rng.standard_normal((n, dim)).astype(f32)
    spikes = rng.choice(n, 40, replace=False)
    x[spikes, rng.integers(0, dim, 40)] = rng.choice([3.0, 30.0, -300.0], 40).astype(f32)   # one dominant coordinate
    x[rng.choice(n, 20, replace=False)] *= f32(1e3)                                           # huge rows
    x[rng.choice(n, 5, replace=False)] = 0.0                                                  # zero rows
    x = x.astype(f32)
    q = (rng.standard_normal((nq, 16)).astype(f32) @ basis / 4.0).astype(f32)
    sx, x8, r8, xn = quant_rows(x)
    assert r8.max() > 50 * np.median(r8), "the table must mix small and large residuals"
    xmax, rmax = float(np.sqrt(xn.max())), float(r8.max())
    xd = x.astype(np.float64)
    X = (np.sqrt(xn) * f32(1.0 + 1.0 / 1024.0)).astype(f32) + r8                               # X_x (fp32)
    for j in range(nq):
        tq, h, lo = quant_query(q[j])
        (a, b, c, d), eps = coefficients(q[j], tq, h, lo, is_l2, c_sum)
        ihi, ilo = x8.astype(np.float64) @ h, x8.astype(np.float64) @ lo                      # exact int32 products
        inner = (ilo.astype(f32).astype(np.float64) * np.float64(f32(1.0 / 254.0)) + ihi.astype(f32)).astype(f32)
        dot = (sx * (tq * inner).astype(f32)).astype(f32)
        qn = (q[j] * q[j]).sum(dtype=f32)
        approx = (np.float64(-2.0) * dot + (xn + qn).astype(f32)).astype(f32) if is_l2 else -dot
        exact = ((xd - q[j]) ** 2).sum(1) if is_l2 else -(xd @ q[j].astype(np.float64))
        E = (a * r8 + (b * X + ((c * (X * X).astype(f32)).astype(f32) + d)).astype(f32)).astype(f32)
        err = np.abs(approx.astype(np.float64) - exact)
        assert np.all(err <= E), (j, float((err / E).max()))
        # the per-row bound never exceeds the global one the certificate uses, and is far tighter on ordinary rows
        assert np.all(E <= eps(xmax, rmax) * (1 + 1e-5))
        assert np.median(E) < 0.5 * eps(xmax, rmax)
