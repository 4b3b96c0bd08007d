"""Iterative refinement stopped by the componentwise backward error, with double-double residuals
(b200ldlt_solve_refined / _device).

The header (include/b200ldlt.h) states the residual's order of operations, the backward errors and the stopping rule
exactly, so the numpy replay below reproduces every returned bit: x, steps, status, omega1, omega2 and omega_first."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.capi import Refined
from ipopt_b200.kkt import to_scipy

from test_error_analysis import rows_of
from test_partial_solve import LARGE, SYSTEMS, assert_bits, factored

NEW_SYMBOLS = ["b200ldlt_solve_refined", "b200ldlt_solve_refined_device"]
EPS = 2.0 ** -52
FIELDS = [k for k, _ in Refined._fields_]
LANE = np.arange(32)


def tridiag(n=2000):
    """the tridiagonal system with a 1e-10 diagonal: the factorisation lifts pivots (num_forced > 0)"""
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    return n, irn, jcn, val


ALL = dict(SYSTEMS, mbndry400=LARGE, tridiag=tridiag)


# ---- error-free transformations in numpy (every float64 operation rounds once, nothing is fused) ----------------------
def two_sum(a, b):
    s = a + b
    v = s - a
    return s, (a - (s - v)) + (b - v)


def two_prod(a, b):
    """(p, e) with p = fl(a b) and p + e = a b exactly (Dekker's splitting; the same e as fma(a, b, -p))"""
    p = a * b
    f = 134217729.0   # 2^27 + 1
    ta, tb = f * a, f * b
    ah, bh = ta - (ta - a), tb - (tb - b)
    al, bl = a - ah, b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def fma(a, b, c):
    """correctly rounded a b + c: RN(th + RO(tl + ul)) with (uh, ul) = a b, (th, tl) = c + uh exactly and RO rounding to
    odd (Boldo and Melquiond, 'Emulation of FMA and correctly rounded sums', 2008)"""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, np.float64) for v in (a, b, c)))
    uh, ul = two_prod(a, b)
    th, tl = two_sum(c, uh)
    v, err = two_sum(tl, ul)
    bits = np.atleast_1d(v).view(np.uint64)
    even = (bits & np.uint64(1)) == 0
    fix = (err != 0) & even
    v = np.where(fix, np.nextafter(v, np.where(err > 0, np.inf, -np.inf)), v)
    return th + v


# ---- the header's residual, s and omegas, replayed ------------------------------------------------------------------
def lanes(rows, r0, r1, k):
    ptr = rows[0]
    idx = ptr[r0:r1, None] + 32 * k + LANE[None, :]
    return idx, idx < ptr[r0 + 1:r1 + 1, None]


def dd_residual(rows, b, x):
    """r = b - A x in the header's double-double order, and s = |A| |x| in error_analysis's (lane sums by fma)"""
    ptr, col, a = rows
    n = len(ptr) - 1
    L = np.diff(ptr)
    r, s = np.zeros(n), np.zeros(n)
    for r0 in range(0, n, 1 << 15):
        r1 = min(n, r0 + (1 << 15))
        h = np.zeros((r1 - r0, 32))
        h[:, 0] = b[r0:r1]
        lo = np.zeros_like(h)
        sx = np.zeros_like(h)
        for k in range(max(1, -(-int(L[r0:r1].max(initial=0)) // 32))):
            idx, m = lanes(rows, r0, r1, k)
            ae, xe = a[idx[m]], x[col[idx[m]]]
            p, e = two_prod(-ae, xe)
            hh, t = two_sum(h[m], p)
            h[m] = hh
            lo[m] = lo[m] + (t + e)
            sx[m] = fma(np.abs(ae), np.abs(xe), sx[m])
        for o in (16, 8, 4, 2, 1):
            hh, t = two_sum(h, h[:, LANE ^ o])
            lo = (lo + lo[:, LANE ^ o]) + t
            h = hh
            sx = sx + sx[:, LANE ^ o]
        r[r0:r1] = h[:, 0] + lo[:, 0]
        s[r0:r1] = sx[:, 0]
    return r, s


def dd_residual_scalar(terms):
    """one row in pure Python floats: terms[0] = b_i, then the (a_ij, x_j) pairs in column order"""
    b, pairs = terms[0], terms[1:]
    h, lo = [0.0] * 32, [0.0] * 32
    h[0] = b
    for q, (aij, xj) in enumerate(pairs):
        ln = q % 32
        p = -aij * xj
        e = float(Fraction(-aij) * Fraction(xj) - Fraction(p))   # exact: the error of a product is a double
        s = h[ln] + p
        v = s - h[ln]
        t = (h[ln] - (s - v)) + (p - v)
        h[ln], lo[ln] = s, lo[ln] + (t + e)
    for o in (16, 8, 4, 2, 1):
        nh, nl = [0.0] * 32, [0.0] * 32
        for ln in range(32):
            a2, b2 = h[ln], h[ln ^ o]
            s = a2 + b2
            v = s - a2
            t = (a2 - (s - v)) + (b2 - v)
            nh[ln], nl[ln] = s, (lo[ln] + lo[ln ^ o]) + t
        h, lo = nh, nl
    return h[0] + lo[0]


def omegas(rows, b, x, r, s):
    """omega1, omega2 of error_analysis's class rule (k_ea_class) for the residual r and s"""
    ptr, col, a = rows
    n = len(ptr) - 1
    aa = np.abs(a)
    amax = np.zeros(n)
    ne = ptr[1:] > ptr[:-1]
    amax[ne] = np.maximum.reduceat(aa, ptr[:-1][ne])
    ax = np.abs(x)
    xn = np.where(np.isnan(ax), np.inf, ax).max()
    ab = np.abs(b)
    axn = amax * xn
    tau = (1000.0 * n * EPS) * (axn + ab)
    in2 = s + ab <= tau
    w = np.where(in2, s + axn, s + ab)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.abs(r / w)
    t = np.where(np.isnan(t), np.inf, t)
    t = np.where(r != 0, t, 0.0)
    return float(t[~in2].max(initial=0.0)), float(t[in2].max(initial=0.0))


def rule(oms, max_steps, tol):
    """the header's stopping rule on the omegas (omega1, omega2) of x_0, x_1, ... (as many as it reads): (status, steps,
    nres, omega1, omega2, omega_first), steps being the index of the returned iterate"""
    first = oms[0][0] + oms[0][1]
    for k, (o1, o2) in enumerate(oms):
        om = o1 + o2
        prev = oms[k - 1][0] + oms[k - 1][1] if k else None
        if not math.isfinite(om):
            return (3, 0, 1, o1, o2, first) if k == 0 else (3, k - 1, k + 1) + tuple(oms[k - 1]) + (first,)
        if om <= tol:
            return 0, k, k + 1, o1, o2, first
        if k >= 1 and om > prev / 2:
            return (1, k, k + 1, o1, o2, first) if om < prev else (1, k - 1, k + 1) + tuple(oms[k - 1]) + (first,)
        if k == max_steps:
            return 2, k, k + 1, o1, o2, first
    raise AssertionError("the rule needs more iterates")


def replay(s, rows, b, max_steps, tol):
    """the refinement in numpy, with the library's single-column solve for x_0 and each d_k"""
    def solve(v):
        y = np.array(v, np.float64)
        assert s.solve(y, 1) == SYMSOLVER_SUCCESS, s.last_error()
        return y
    xs, oms = [solve(b)], []
    while True:
        r, sv = dd_residual(rows, b, xs[-1])
        oms.append(omegas(rows, b, xs[-1], r, sv))
        try:
            out = rule(oms, max_steps, tol)
            break
        except AssertionError:
            xs.append(xs[-1] + solve(r))
    status, steps, nres, o1, o2, first = out
    return xs[steps], dict(omega_first=first, omega1=o1, omega2=o2, steps=steps, status=status, nres=nres)


def assert_outcome(got, c, ref, tag):
    for k in FIELDS:
        g = np.asarray(got[k])[c]
        if k.startswith("omega"):
            assert_bits(np.float64(g), np.float64(ref[k]), (tag, k, g, ref[k]))
        else:
            assert g == ref[k], (tag, k, g, ref[k])


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


def test_fma_emulation_is_correctly_rounded():
    rng = np.random.default_rng(3)
    a = rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)
    b = rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)
    c = np.where(rng.random(4000) < 0.5, -(a * b), rng.standard_normal(4000))   # cancellation in half of them
    c = c * (1 + rng.integers(-2, 3, 4000) * EPS)
    got = fma(a, b, c)
    for i in range(4000):
        assert got[i] == float(Fraction(a[i]) * Fraction(b[i]) + Fraction(c[i])), i


def cancelling_rows(rng, nrows):
    """rows (b, [(a, x) ...]) whose terms cancel to far below their size"""
    out = []
    for _ in range(nrows):
        m = int(rng.integers(1, 90))
        a = rng.standard_normal(m) * 2.0 ** rng.integers(-20, 20, m)
        x = rng.standard_normal(m) * 2.0 ** rng.integers(-20, 20, m)
        exact = sum(Fraction(ai) * Fraction(xi) for ai, xi in zip(a, x))
        b = float(exact) * (1 + float(rng.integers(-3, 4)) * EPS)
        out.append((b, list(zip(a.tolist(), x.tolist()))))
    return out


def test_double_double_replay_matches_scalar_and_bound():
    rng = np.random.default_rng(11)
    rows = cancelling_rows(rng, 200)
    ptr = np.r_[0, np.cumsum([len(p) for _, p in rows])]
    a = np.array([ai for _, p in rows for ai, _ in p])
    xv = np.array([xi for _, p in rows for _, xi in p])
    col = np.arange(len(a))   # one x entry per term
    b = np.array([bi for bi, _ in rows])
    r, _ = dd_residual((ptr, col, a), b, xv)
    worst = 0.0
    for i, (bi, pairs) in enumerate(rows):
        assert_bits(np.float64(r[i]), np.float64(dd_residual_scalar([bi] + pairs)), i)
        exact = Fraction(bi) - sum(Fraction(ai) * Fraction(xi) for ai, xi in pairs)
        size = abs(bi) + sum(abs(ai * xi) for ai, xi in pairs)
        m = len(pairs)
        bound = Fraction(2.0 ** -53) * abs(exact) + Fraction((m + 32) ** 2) * Fraction(2.0 ** -105) * Fraction(size)
        err = abs(Fraction(r[i]) - exact)
        assert err <= bound, (i, float(err), float(bound))
        if size:
            worst = max(worst, float(err / Fraction(size)))
    # the working-precision sum of the same rows is far less accurate: the double-double really is one
    assert worst < 1e-28


NAN, INF = float("nan"), float("inf")


@pytest.mark.parametrize("oms,max_steps,tol,expect", [
    ([(NAN, 0.0)], 10, EPS, (3, 0, 1)),                                   # non-finite x_0: x_0, omega +inf
    ([(0.0, INF)], 10, EPS, (3, 0, 1)),
    ([(1e-8, 0.0), (1e-12, 0.0), (NAN, 0.0)], 10, EPS, (3, 1, 3)),        # non-finite later: the last finite iterate
    ([(0.0, 0.0)], 10, 0.0, (0, 0, 1)),                                   # a zero column converges at step 0
    ([(1e-8, 0.0), (1e-17, 1e-17)], 10, EPS, (0, 1, 2)),
    ([(1e-8, 0.0), (EPS, 0.0)], 10, EPS, (0, 1, 2)),                      # omega == tol converges
    ([(1e-8, 0.0), (1e-8, 0.0)], 10, EPS, (1, 0, 2)),                     # a tie: the older iterate
    ([(1e-8, 0.0), (2e-8, 0.0)], 10, EPS, (1, 0, 2)),                     # worse: rolled back
    ([(1e-8, 0.0), (0.6e-8, 0.0)], 10, EPS, (1, 1, 2)),                   # better but not halved: kept
    ([(1e-8, 0.0), (0.5e-8, 0.0), (0.25e-8, 0.0)], 2, EPS, (2, 2, 3)),    # exact halving goes on, to the limit
    ([(1e-8, 0.0)], 0, EPS, (2, 0, 1)),                                   # max_steps = 0: job 0
    ([(1e-20, 0.0)], 0, EPS, (0, 0, 1)),
    ([(1e-8, 1e-8), (1e-9, 0.0), (1e-9, 0.0)], 10, EPS, (1, 1, 3)),       # a tie after a good step
])
def test_stopping_rule(oms, max_steps, tol, expect):
    status, steps, nres, o1, o2, first = rule(oms, max_steps, tol)
    assert (status, steps, nres) == expect
    assert first == oms[0][0] + oms[0][1] or not math.isfinite(first)
    assert (o1, o2) == tuple(oms[steps]) or (status == 3 and steps == 0)
    if math.isfinite(o1 + o2):
        assert o1 + o2 <= first


# ---- GPU ------------------------------------------------------------------------------------------------------------
def refined(s, B, max_steps=10, tol=EPS, device=False):
    """the library's refinement of the columns (rows of B): (X rows, dict of per-column arrays)"""
    if not device:
        X, d = s.solve_refined(B.T, max_steps, tol)
        return np.ascontiguousarray(X.T), d
    import torch
    db = torch.tensor(np.ascontiguousarray(B).ravel(), dtype=torch.float64, device="cuda")
    dx = torch.zeros_like(db)
    st, d = s.solve_refined_device(db.data_ptr(), dx.data_ptr(), B.shape[0], max_steps, tol)
    assert st == SYMSOLVER_SUCCESS, s.last_error()
    assert_bits(db.cpu().numpy(), np.ascontiguousarray(B).ravel(), "b untouched")
    return dx.cpu().numpy().reshape(B.shape), d


def columns(dim, seed, k=3):
    return np.random.default_rng(seed).standard_normal((k, dim))


@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(ALL))
def test_bit_exact_replay(system):
    dim, irn, jcn, val = ALL[system]()
    s = factored(dim, irn, jcn, val)
    if system == "tridiag":
        assert s.info()["num_forced"] > 0
    rows = rows_of(dim, irn, jcn, val)
    B = columns(dim, 5)
    X, got = refined(s, B)
    for c in range(B.shape[0]):
        x_ref, ref = replay(s, rows, B[c], 10, EPS)
        assert_bits(X[c], x_ref, (system, c, "x"))
        assert_outcome(got, c, ref, (system, c))
    s.close()


def exact_omegas(rows, b, x):
    """omega1, omega2 with exact (Fraction) residuals, under the library's s, classes and weights"""
    ptr, col, a = rows
    n = len(ptr) - 1
    _, s = dd_residual(rows, b, x)
    aa = np.abs(a)
    amax = np.zeros(n)
    ne = ptr[1:] > ptr[:-1]
    amax[ne] = np.maximum.reduceat(aa, ptr[:-1][ne])
    xn = np.abs(x).max()
    ab = np.abs(b)
    axn = amax * xn
    in2 = s + ab <= (1000.0 * n * EPS) * (axn + ab)
    w = np.where(in2, s + axn, s + ab)
    om = [Fraction(0), Fraction(0)]
    for i in range(n):
        e = Fraction(b[i]) - sum(Fraction(a[q]) * Fraction(x[col[q]]) for q in range(ptr[i], ptr[i + 1]))
        if e:
            k = int(in2[i])
            om[k] = max(om[k], abs(e) / Fraction(w[i]))
    return float(om[0]), float(om[1]), int(np.diff(ptr).max())


@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(SYSTEMS) + ["tridiag"])
def test_accuracy_against_exact_residuals(system):
    dim, irn, jcn, val = ALL[system]()
    s = factored(dim, irn, jcn, val)
    rows = rows_of(dim, irn, jcn, val)
    B = columns(dim, 9, 2)
    X, got = refined(s, B)
    for c in range(2):
        e1, e2, m = exact_omegas(rows, B[c], X[c])
        for k, e in (("omega1", e1), ("omega2", e2)):
            g = got[k][c]
            assert abs(g - e) <= 2.0 ** -51 * e + (m + 32) ** 2 * 2.0 ** -103, (system, c, k, g, e)
        assert got["omega1"][c] + got["omega2"][c] <= got["omega_first"][c]
    s.close()


@pytest.mark.gpu
def test_lifted_tridiagonal_converges():
    """job 0 solves the perturbed matrix (num_forced > 0): omega_first far above eps; refinement reaches eps"""
    s = factored(*tridiag())
    assert s.info()["num_forced"] > 0
    B = columns(2000, 21, 4)
    X, got = refined(s, B)
    assert np.all(got["omega_first"] > 1e3 * EPS), got["omega_first"]
    assert np.all(got["status"] == 0), got
    assert np.all(got["steps"] <= 5), got["steps"]
    assert np.all(got["omega1"] + got["omega2"] <= EPS)
    s.close()


@pytest.mark.gpu
def test_large_within_tol_or_says_why():
    s = factored(*LARGE())
    B = columns(s.dim, 2, 2)
    X, got = refined(s, B)
    om = got["omega1"] + got["omega2"]
    assert np.all(om <= got["omega_first"])
    for c in range(2):
        assert om[c] <= EPS or got["status"][c] in (1, 2), (c, got)
    s.close()


def block_columns(dim):
    """11 columns that finish at different steps: a zero column (step 0), random ones, and two that meet max_steps"""
    rng = np.random.default_rng(17)
    B = rng.standard_normal((11, dim)) * np.logspace(-3, 3, 11)[:, None]
    B[3] = 0.0
    return B


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["tridiag", "MBndryCntrl1_30"])
def test_blocks_and_entry_points(system, monkeypatch):
    """every column bit-identical to the call on it alone, to the device entry point, to a repeated call and to
    B200_SOLVE_BLOCK=1; on the lifted tridiagonal the columns finish at different steps"""
    dim, irn, jcn, val = ALL[system]()
    B = block_columns(dim)
    s = factored(dim, irn, jcn, val)
    for max_steps in (10, 1):
        X, got = refined(s, B, max_steps)
        assert got["status"][3] == 0 and got["steps"][3] == 0 and not np.any(X[3])
        Xd, gd = refined(s, B, max_steps, device=True)
        X2, g2 = refined(s, B, max_steps)
        for c in range(B.shape[0]):
            Xc, gc = refined(s, B[c:c + 1], max_steps)
            assert_bits(X[c], Xc[0], (max_steps, c, "alone"))
            for other, tag in ((gd, "device"), (g2, "repeat"), (gc, "alone")):
                assert_outcome(got, c, {k: np.asarray(other[k])[0 if tag == "alone" else c] for k in FIELDS},
                               (max_steps, c, tag))
        assert_bits(Xd, X, (max_steps, "device"))
        assert_bits(X2, X, (max_steps, "repeat"))
        if system == "tridiag":
            assert len(set(got["nres"].tolist())) > 1, got["nres"]
            if max_steps == 1:
                assert np.any(got["status"] == 2), got["status"]
    s.close()
    monkeypatch.setenv("B200_SOLVE_BLOCK", "1")
    s1 = factored(dim, irn, jcn, val)
    X1, g1 = refined(s1, B)
    s1.close()
    s = factored(dim, irn, jcn, val)
    X, got = refined(s, B)
    s.close()
    assert_bits(X1, X, "B200_SOLVE_BLOCK=1")
    for c in range(B.shape[0]):
        assert_outcome(got, c, {k: np.asarray(g1[k])[c] for k in FIELDS}, (c, "block 1"))


@pytest.mark.gpu
def test_plain_solve_and_no_side_effects():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = factored(dim, irn, jcn, val)
    B = columns(dim, 4)
    X0 = B.copy()
    assert s.solve(X0.ravel(), 3) == SYMSOLVER_SUCCESS
    ea0 = s.error_analysis(B.T, X0.T, True)
    X, got = refined(s, B, max_steps=0)
    assert_bits(X, X0, "max_steps = 0")
    assert np.all(got["steps"] == 0) and np.all(got["nres"] == 1)
    refined(s, B)
    X1 = B.copy()
    assert s.solve(X1.ravel(), 3) == SYMSOLVER_SUCCESS
    assert_bits(X1, X0, "solve after")
    ea1 = s.error_analysis(B.T, X0.T, True)
    for k in ea0:
        assert_bits(np.asarray(ea0[k], np.float64), np.asarray(ea1[k], np.float64), ("error_analysis", k))
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1"])
def test_launch_counts(block, monkeypatch):
    """one column: nres (L0 + 3); one block: 1 + E (L0 + 3) - 1, E the block's largest nres"""
    if block is not None:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*tridiag())
    B = block_columns(2000)[:8]
    x = B[0].copy()
    assert s.solve(x, 1) == SYMSOLVER_SUCCESS
    L0 = s.info()["launches_solve"]
    for device in (False, True):
        _, got = refined(s, B[:1], device=device)
        assert s.info()["launches_solve"] == got["nres"][0] * (L0 + 3)
        assert s.info()["ms_solve_gpu"] > 0.0
        _, got = refined(s, B, device=device)
        want = (got["nres"].max() * (L0 + 3) if block is None
                else 1 + int(np.sum(got["nres"] * (L0 + 3) - 1)))
        assert s.info()["launches_solve"] == want, (s.info()["launches_solve"], want, got["nres"])
    s.close()


@pytest.mark.gpu
def test_kept_singular_factors():
    from test_fredholm import handle, zeroed
    dim, irn, jcn, val, _ = zeroed("MBndryCntrl1_30", 2)
    s, st, _ = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR
    y = columns(dim, 6, 2)
    B = (to_scipy(dim, irn, jcn, val) @ y.T).T        # consistent columns
    X, got = refined(s, B)
    for c in range(2):
        assert got["status"][c] in (0, 1), got
        assert got["omega1"][c] + got["omega2"][c] <= got["omega_first"][c]
    s.close()


@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    L = s._L
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    b, x = np.ones(dim), np.full(dim, 42.0)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
    out = (Refined * 2)()

    def refused(nrhs, pb, px, max_steps, tol, match, device=False):
        for o in out:
            for k in FIELDS:
                setattr(o, k, 42)
        f = L.b200ldlt_solve_refined_device if device else L.b200ldlt_solve_refined
        assert f(s._h, nrhs, pb, px, max_steps, tol, out) == SYMSOLVER_FATAL_ERROR and match in s.last_error(), \
            s.last_error()
        assert all(getattr(o, k) == 42 for o in out for k in FIELDS)
        assert np.all(x == 42.0)

    refused(1, dp(b), dp(x), 10, EPS, "no factors")
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    refused(-1, dp(b), dp(x), 10, EPS, "nrhs")
    refused(1, dp(b), dp(x), -1, EPS, "max_steps")
    refused(1, dp(b), dp(x), 10, -1.0, "tol")
    refused(1, dp(b), dp(x), 10, NAN, "tol")
    refused(1, None, dp(x), 10, EPS, "NULL")
    refused(1, dp(b), None, 10, EPS, "NULL")
    refused(1, None, None, 10, EPS, "NULL", device=True)
    refused(1, dp(x), dp(x), 10, EPS, "x must not be b")
    assert L.b200ldlt_solve_refined(s._h, 1, dp(b), dp(x), 10, EPS, None) == SYMSOLVER_FATAL_ERROR
    assert np.all(x == 42.0)
    # nrhs = 0: success, nothing written, nothing launched
    for o in out:
        o.status = 42
    assert L.b200ldlt_solve_refined(s._h, 0, None, None, 10, EPS, out) == SYMSOLVER_SUCCESS and out[0].status == 42
    assert s.info()["launches_solve"] == 0
    # Schur mode: the shared refusal
    assert s.set_schur(np.arange(dim - 5, dim)) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    refused(1, dp(b), dp(x), 10, EPS, "solve_refined: Schur mode")
    assert s.set_schur([]) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    X, got = s.solve_refined(b)
    assert got["status"][0] in (0, 1, 2)
    # sharded handle
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    refused(1, dp(b), dp(x), 10, EPS, "sharded")
    s.close()
