"""The lower bound of filter level P (vb_list_proj.cu lp_bound_kernel), emulated on the CPU step by step as the kernels
compute it: the basis P in fp32, sigma^2 from a Gershgorin bound on P P^T, the projections accumulated in double and
rounded to fp32, the fp32 fmaf chain of the list-major kernel over the r components, and the bound's fp32 steps each
rounded down.  For random, non-orthonormal and nearly singular P, on rows with common offsets and mixed scales, the bound
must never exceed the fp32 distance, and the listing refine's rule with it (re-score the k smallest, then every other
listed candidate with LB <= T1, certify LB_{k'} > T) must return the exact top k of every query it certifies."""
import numpy as np
import pytest

U = 2.0 ** -24
F32 = np.float32


def down(v):
    """float64 -> the fp32 value at or below it"""
    f = np.asarray(v, np.float64).astype(F32)
    return np.where(f.astype(np.float64) > v, np.nextafter(f, F32(-np.inf)), f)


def up(v):
    f = np.asarray(v, np.float64).astype(F32)
    return np.where(f.astype(np.float64) < v, np.nextafter(f, F32(np.inf)), f)


def constants(p, dim):
    """(c1, c2, ce) as list_proj_prepare computes them"""
    r = p.shape[0]
    pd = p.astype(np.float64)
    g = pd @ pd.T
    pn = (pd * pd).sum(1)
    sigma2 = (np.abs(g) + dim * np.ldexp(pn.max(), -52)).sum(1).max() * (1 + 2.0 ** -40)
    c1 = np.nextafter(F32(1.0 - (r + 4) * U), F32(0))
    c2 = np.nextafter(F32((1.0 - (dim + 8) * U) / sigma2), F32(0))
    ce = up(U * np.sqrt(sigma2) * (1 + U) + dim * 2.0 ** -52 * np.sqrt(pn.sum()) * 1.01)
    return c1, c2, np.nextafter(ce, F32(np.inf)), sigma2


def project(p, x):
    return (x.astype(np.float64) @ p.astype(np.float64).T).astype(F32)


def fma_chain(yx, yq):
    """fl(sum_j fl(yx_j - yq_j)^2), one fmaf rounding per component, in order"""
    s = np.zeros(yx.shape[0], F32)
    for j in range(yx.shape[1]):
        d = (yx[:, j] - yq[j]).astype(F32)
        s = (d.astype(np.float64) ** 2 + s.astype(np.float64)).astype(F32)
    return s


def lower_bound(s, qn, xmax, c1, c2, ce):
    s = np.minimum(s, F32(np.finfo(F32).max))
    delta = up(ce.astype(np.float64) * up(xmax.astype(np.float64) + up(up(np.sqrt(np.float64(qn))) * (1 + 1 / 1024)).astype(np.float64)))
    t = down(down(np.sqrt(down(s.astype(np.float64) * c1).astype(np.float64))).astype(np.float64) - np.float64(delta))
    t = np.where(t < 0, F32(0), t)
    return down(down(t.astype(np.float64) ** 2).astype(np.float64) * np.float64(c2))


def fp32_distance(x, q):
    """the fp32 sum of squared differences, sequential (the oracle's order)"""
    acc = np.zeros(x.shape[0], F32)
    for i in range(x.shape[1]):
        d = (x[:, i] - q[i]).astype(F32)
        acc = (acc + d * d).astype(F32)
    return acc


def bases(rng, dim, r, rows):
    yield "principal", np.linalg.svd(rows[:1000].astype(np.float64), full_matrices=False)[2][:r].astype(F32)
    q = np.linalg.qr(rng.standard_normal((dim, r)))[0].T
    yield "orthonormal", q.astype(F32)
    yield "scaled", (q * rng.uniform(0.2, 3.0, (r, 1))).astype(F32)
    yield "random", rng.standard_normal((r, dim)).astype(F32)
    near = q.copy()
    near[1] = near[0] + 1e-4 * near[1]      # two nearly equal directions: ||P||_2 close to sqrt(2)
    yield "near_singular", near.astype(F32)
    yield "sigma_near_one", (q * F32(1 - 1e-7)).astype(F32)


def data(rng, dim, law):
    n, nq = 3000, 24
    if law == "lowrank":
        frame = np.linalg.qr(rng.standard_normal((dim, 8)))[0]
        z = rng.standard_normal((n + nq, 8))
        a = (z @ frame.T + 0.02 * rng.standard_normal((n + nq, dim))).astype(F32)
    elif law == "offset":
        a = (1000.0 + 0.01 * rng.standard_normal((n + nq, dim))).astype(F32)
    else:
        a = (rng.standard_normal((n + nq, dim)) * np.exp(rng.uniform(-6, 6, (n + nq, 1)))).astype(F32)
    return a[:n], a[n:]


@pytest.mark.parametrize("law", ["lowrank", "offset", "mixed_scales"])
def test_bound_below_the_fp32_distance_and_certified_results_exact(law):
    rng = np.random.default_rng(7)
    dim, r, k, kp = 96, 16, 10, 64
    rows, queries = data(rng, dim, law)
    xmax = F32(np.sqrt(down((rows.astype(np.float64) ** 2).sum(1).max())))
    for name, p in bases(rng, dim, r, rows):
        c1, c2, ce, _ = constants(p, dim)
        y = project(p, rows)
        certified = 0
        for q in queries:
            qn = F32((q.astype(np.float64) ** 2).sum())
            lb = lower_bound(fma_chain(y, project(p, q[None])[0]), qn, xmax, c1, c2, ce)
            d = fp32_distance(rows, q)
            assert (lb <= d).all(), (law, name, float((lb - d).max()))
            # the listing refine's rule with d~ = LB, zero per-row terms and eps(q) = 0
            order = np.lexsort((np.arange(len(lb)), lb))
            listed = order[:kp]
            t1 = d[listed[:k]].max()
            sel = np.concatenate([listed[:k], listed[k:][~(lb[listed[k:]] > t1)]])
            top = sel[np.lexsort((sel, d[sel]))][:k]
            if lb[listed[kp - 1]] > d[top[-1]]:
                certified += 1
                truth = np.lexsort((np.arange(len(d)), d))[:k]
                assert np.array_equal(top, truth) and np.array_equal(d[top], d[truth]), (law, name)
        if law == "lowrank" and name == "principal":
            assert certified > 0
