"""Error analysis and condition estimation (b200ldlt_error_analysis / _device, b200ldlt_condest).

Per column, with r = b - A x, s = |A||x|, a_i = max_j |a_ij| and tau_i = 1000 n 2^-52 (a_i ||x|| + |b_i|): I2 = {i : s_i +
|b_i| <= tau_i}, I1 the rest; omega1 = max_I1 |r_i| / (s_i + |b_i|), omega2 = max_I2 |r_i| / (s_i + a_i ||x||); cond_k =
est ||M diag(w_k)||_inf / ||x||, w1 = s + |b| on I1, w2 = s + a ||x|| on I2; ferr = omega1 cond1 + omega2 cond2.  The
estimator is LAPACK's dlacn2 (Higham).  The numpy reference below uses the same definitions; A's duplicates are summed in
triplet order before absolute values are taken, and the row sums of |A| and |A||x| follow the kernel's fixed order, so
anorm, xnorm and |I2| compare exactly."""
import ctypes as C

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.capi import Errors
from ipopt_b200.kkt import mbndry_kkt, to_scipy

from test_partial_solve import LARGE, SYSTEMS, assert_bits, factored

NEW_SYMBOLS = ["b200ldlt_error_analysis", "b200ldlt_error_analysis_device", "b200ldlt_condest"]
ALL = dict(SYSTEMS, mbndry400=LARGE)
EPS = 2.0 ** -52
FIELDS = [k for k, _ in Errors._fields_]


# ---- the numpy reference -------------------------------------------------------------------------------------------
def dlacn2(n, matvec, rmatvec):
    """Higham's 1-norm estimate of the operator B (B v = matvec(v), B^T v = rmatvec(v)) exactly as LAPACK dlacn2 runs it:
    (est, products taken)"""
    y = matvec(np.full(n, 1.0 / n))
    if n == 1:
        return abs(y[0]), 1
    est, nprod = np.abs(y).sum(), 1
    xi = np.where(y >= 0, 1.0, -1.0)
    z = rmatvec(xi)
    nprod += 1
    j, it = int(np.argmax(np.abs(z))), 2
    while True:
        e = np.zeros(n)
        e[j] = 1.0
        y = matvec(e)
        nprod += 1
        old, est = est, np.abs(y).sum()
        sg = np.where(y >= 0, 1.0, -1.0)
        if np.array_equal(sg, xi) or est <= old:
            break
        xi = sg
        z = rmatvec(xi)
        nprod += 1
        jlast, j = j, int(np.argmax(np.abs(z)))
        if not (z[jlast] != abs(z[j]) and it < 5):
            break
        it += 1
    i = np.arange(n)
    y = matvec(np.where(i % 2, -1.0, 1.0) * (1.0 + i / (n - 1)))
    nprod += 1
    t = 2.0 * (np.abs(y).sum() / (3.0 * n))
    return (t if t > est else est), nprod


def rows_of(dim, irn, jcn, val):
    """|A|'s row structure as the library builds it: duplicates summed in triplet order (0.0 + v0 + v1 ...), both
    triangles of the unique entries, each row's columns ascending.  (ptr, col, a)"""
    i, j = np.asarray(irn, np.int64) - 1, np.asarray(jcn, np.int64) - 1
    lo, hi = np.minimum(i, j), np.maximum(i, j)
    key = lo * dim + hi
    order = np.argsort(key, kind="stable")
    ks, vs = key[order], np.asarray(val, np.float64)[order]
    start = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    cnt = np.diff(np.r_[start, len(ks)])
    a = np.zeros(len(start))
    for k in range(int(cnt.max())):
        m = cnt > k
        a[m] += vs[start[m] + k]
    ur, uc = ks[start] // dim, ks[start] % dim
    off = ur != uc
    R, Cc, V = np.r_[ur, uc[off]], np.r_[uc, ur[off]], np.r_[a, a[off]]
    o = np.lexsort((Cc, R))
    ptr = np.r_[0, np.cumsum(np.bincount(R, minlength=dim))]
    return ptr, Cc[o], V[o]


def warp_sums(ptr, v):
    """the row sums of k_ea_rows: lane l adds the row's entries l, l + 32, ... in order, then a shuffle-xor tree"""
    n = len(ptr) - 1
    out = np.zeros(n)
    L = np.diff(ptr)
    lane = np.arange(32)
    for r0 in range(0, n, 1 << 15):
        r1 = min(n, r0 + (1 << 15))
        acc = np.zeros((r1 - r0, 32))
        for k in range(max(1, -(-int(L[r0:r1].max(initial=0)) // 32))):
            idx = ptr[r0:r1, None] + 32 * k + lane[None, :]
            m = idx < ptr[r0 + 1:r1 + 1, None]
            acc[m] += v[idx[m]]
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[:, lane ^ o]
        out[r0:r1] = acc[:, 0]
    return out


def row_sums_ld(ptr, v):
    """exact-ish row sums in extended precision"""
    n = len(ptr) - 1
    out = np.zeros(n, np.longdouble)
    ne = ptr[1:] > ptr[:-1]
    if ne.any():
        out[ne] = np.add.reduceat(v.astype(np.longdouble), ptr[:-1][ne])
    return out


def ref_errors(rows, b, x, Minv=None):
    """the definitions for one column (b, x 1-D); with Minv (dense), also the exact cond1, cond2 and ferr"""
    ptr, col, a = rows
    n = len(ptr) - 1
    aa = np.abs(a)
    amax = np.zeros(n)
    ne = ptr[1:] > ptr[:-1]
    amax[ne] = np.maximum.reduceat(aa, ptr[:-1][ne])
    s = warp_sums(ptr, aa * np.abs(x[col]))
    r = np.asarray(b, np.longdouble) - row_sums_ld(ptr, a.astype(np.longdouble) * x[col])
    xn = np.abs(x).max()
    ab = np.abs(b)
    tau = (1000.0 * n * EPS) * (amax * xn + ab)
    in2 = s + ab <= tau
    w1 = np.where(in2, 0.0, s + ab)
    w2 = np.where(in2, s + amax * xn, 0.0)
    ar = np.abs(r)
    with np.errstate(divide="ignore", invalid="ignore"):
        t1 = np.where(~in2 & (r != 0), ar / np.where(in2, 1.0, w1), 0.0)
        t2 = np.where(in2 & (r != 0), ar / np.where(in2, w2, 1.0), 0.0)
    out = dict(anorm=warp_sums(ptr, aa).max(), xnorm=xn, rnorm=float(ar.max()), omega1=float(t1.max(initial=0.0)),
               omega2=float(t2.max(initial=0.0)), n_i2=int(in2.sum()), w1=w1, w2=w2, r=r.astype(np.float64),
               den=np.where(in2, w2, w1))
    if Minv is not None:
        if xn == 0.0:
            c = 0.0 if not np.any(b) else np.inf
            out.update(cond1=c, cond2=c, ferr=c)
        else:
            aM = np.abs(Minv)
            out["cond1"] = (aM @ w1).max() / xn
            out["cond2"] = (aM @ w2).max() / xn
            out["ferr"] = out["omega1"] * out["cond1"] + out["omega2"] * out["cond2"]
    return out


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


def test_dlacn2_port_matches_lapack_dsycon():
    from scipy.linalg import lapack
    rng = np.random.default_rng(11)
    worst = 0.0
    for t in range(120):
        n = int(rng.integers(2, 60))
        G = rng.standard_normal((n, n)) * np.exp(rng.uniform(-3, 3, (n, 1)))
        A = G + G.T
        lu, ipiv, info = lapack.dsytrf(A)
        assert info == 0
        anorm = np.abs(A).sum(axis=0).max()
        rcond, info = lapack.dsycon(lu, ipiv, anorm)
        assert info == 0

        def solve(v):
            x, info2 = lapack.dsytrs(lu, ipiv, v)
            assert info2 == 0
            return x

        est, nprod = dlacn2(n, solve, solve)
        assert nprod <= 11
        kappa = anorm * est
        rel = abs(kappa - 1.0 / rcond) / (1.0 / rcond)
        worst = max(worst, rel)
    assert worst <= 1e-14, worst


def test_reference_edge_cases():
    # 3 x 3 with an all-zero third row / column (the pattern keeps a zero diagonal entry)
    irn = np.array([1, 2, 2, 3, 3], np.int32)
    jcn = np.array([1, 1, 2, 3, 3], np.int32)
    val = np.array([2.0, 1.0, -3.0, 0.5, -0.5])    # the duplicates of (3, 3) sum to 0
    rows = rows_of(3, irn, jcn, val)
    Minv = np.eye(3)
    # x = 0, b = 0: nothing to trust less -- every row in I2, no error, cond = ferr = 0
    e = ref_errors(rows, np.zeros(3), np.zeros(3), Minv)
    assert e["n_i2"] == 3 and e["omega1"] == e["omega2"] == 0.0 and e["cond1"] == e["cond2"] == e["ferr"] == 0.0
    # x = 0, b != 0: the rows with b_i != 0 are in I1 with omega1 = 1; cond = ferr = +inf
    e = ref_errors(rows, np.array([1.0, 0.0, -2.0]), np.zeros(3), Minv)
    assert e["n_i2"] == 1 and e["omega1"] == 1.0 and e["omega2"] == 0.0
    assert np.isinf(e["cond1"]) and np.isinf(e["ferr"])
    # an all-zero row with b_i = 0 lies in I2 with r_i = 0 (a zero denominator only then); with b_i != 0 it is in I1
    x = np.array([1.0, 2.0, 5.0])
    b = np.array([4.0 + 1e-3, -5.0, 0.0])
    e = ref_errors(rows, b, x, Minv)
    assert e["w2"][2] == 0.0 and e["w1"][2] == 0.0 and e["den"][2] == 0.0 and e["r"][2] == 0.0
    assert e["n_i2"] == 1 and e["omega2"] == 0.0
    assert e["omega1"] == pytest.approx(1e-3 / (4.0 + 4.0 + 1e-3), rel=1e-12)
    assert e["anorm"] == 4.0 and e["xnorm"] == 5.0
    b[2] = 1.0
    e = ref_errors(rows, b, x, Minv)
    assert e["n_i2"] == 0 and e["omega1"] == 1.0 and e["w1"][2] == 1.0
    # the numpy estimator on a small dense case: a lower bound of the exact 1-norm, at most 3x below it
    rng = np.random.default_rng(0)
    G = rng.standard_normal((40, 40))
    Mi = np.linalg.inv(G + G.T)
    est, nprod = dlacn2(40, lambda v: Mi @ v, lambda v: Mi.T @ v)
    exact = np.abs(Mi).sum(axis=0).max()
    assert exact / 3 <= est <= exact * (1 + 1e-12) and nprod <= 11


# ---- GPU helpers ---------------------------------------------------------------------------------------------------
def solved(s, B):
    """X = A^-1 B through the library (B: nrhs x dim rows = columns)"""
    X = np.ascontiguousarray(B, np.float64).copy()
    assert s.solve(X.ravel(), B.shape[0]) == SYMSOLVER_SUCCESS, s.last_error()
    return X


def ea(s, B, X, cond=True, device=False):
    """the library's error analysis of the columns (rows of B, X): dict of per-column arrays"""
    if not device:
        return s.error_analysis(B.T, X.T, cond)
    import torch
    db = torch.tensor(np.ascontiguousarray(B).ravel(), dtype=torch.float64, device="cuda")
    dx = torch.tensor(np.ascontiguousarray(X).ravel(), dtype=torch.float64, device="cuda")
    st, d = s.error_analysis_device(db.data_ptr(), dx.data_ptr(), B.shape[0], int(cond))
    assert st == SYMSOLVER_SUCCESS, s.last_error()
    return d


def assert_struct_bits(a, b, cols_a=None, tag=""):
    for k in FIELDS:
        va = np.asarray(a[k]) if cols_a is None else np.asarray(a[k])[cols_a]
        vb = np.asarray(b[k])
        if va.dtype == np.float64:
            assert_bits(va, vb, (tag, k))
        else:
            assert np.array_equal(va, vb), (tag, k, va, vb)


def check_against_ref(got, c, ref, maxrow, tag):
    assert got["anorm"][c] == ref["anorm"], (tag, got["anorm"][c], ref["anorm"])
    assert got["xnorm"][c] == ref["xnorm"], tag
    assert got["n_i2"][c] == ref["n_i2"], (tag, got["n_i2"][c], ref["n_i2"])
    tol = (maxrow + 2) * EPS
    dw = 0.0
    for k in ("omega1", "omega2"):
        d = abs(got[k][c] - ref[k])
        dw = max(dw, d)
        assert d <= tol + 1e-12 * ref[k], (tag, k, got[k][c], ref[k])
    assert abs(got["rnorm"][c] - ref["rnorm"]) <= tol * ref["den"].max() + 1e-12 * ref["rnorm"], tag
    return dw



# ---- 1. backward errors and 3. estimates against the exact values ----------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(ALL))
def test_backward_errors_and_estimates(system):
    dim, irn, jcn, val = ALL[system]()
    s = factored(dim, irn, jcn, val)
    rows = rows_of(dim, irn, jcn, val)
    maxrow = int(np.diff(rows[0]).max())
    rng = np.random.default_rng(7)
    B = rng.standard_normal((2, dim))
    X = solved(s, B)
    X[1] += 1e-6 * np.abs(X[1]).max() * rng.standard_normal(dim)
    small = dim <= 2000
    Minv = np.linalg.inv(to_scipy(dim, irn, jcn, val).toarray()) if small else None
    got = ea(s, B, X, cond=True)
    dw, ratios = 0.0, []
    for c in range(2):
        ref = ref_errors(rows, B[c], X[c], Minv)
        dw = max(dw, check_against_ref(got, c, ref, maxrow, (system, c)))
        assert 0 < got["nprod"][c] <= 22
        for k in ("cond1", "cond2"):
            if small:
                if ref[k] == 0.0:
                    assert got[k][c] == 0.0, (system, c, k)
                    continue
                ratio = got[k][c] / ref[k]
                ratios.append(ratio)
                assert ref[k] / 3 <= got[k][c] <= ref[k] * (1 + 1e-6), (system, c, k, got[k][c], ref[k])
            else:
                assert np.isfinite(got[k][c]) and got[k][c] >= 0.0
        assert got["ferr"][c] == got["omega1"][c] * got["cond1"][c] + got["omega2"][c] * got["cond2"][c]
    # cheap mode: the same norms and backward errors, bit for bit, no estimate
    cheap = ea(s, B, X, cond=False)
    for k in ("anorm", "xnorm", "rnorm", "omega1", "omega2", "n_i2"):
        assert_bits(np.asarray(cheap[k], np.float64), np.asarray(got[k], np.float64), k)
    assert np.all(cheap["cond1"] == -1.0) and np.all(cheap["ferr"] == -1.0) and np.all(cheap["nprod"] == 0)
    if small:
        kappa, anorm1, ainv1, nprod = s.condest()
        exact = np.abs(Minv).sum(axis=0).max()
        assert exact / 3 <= ainv1 <= exact * (1 + 1e-6), (ainv1, exact)
        assert anorm1 == got["anorm"][0] and kappa == anorm1 * ainv1 and 1 <= nprod <= 11
        ratios.append(ainv1 / exact)
    print("\n%s: max |d omega| = %.3e (tolerance %.3e); est/exact in [%s]" % (
        system, dw, (maxrow + 2) * EPS, ", ".join("%.4f" % r for r in (min(ratios), max(ratios))) if ratios else "-"))
    s.close()


# ---- 2. I2 is exercised -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "LukVlE1_1000", "MDistCntrl3a_25"])
def test_second_row_set(system):
    dim, irn, jcn, val = SYSTEMS[system]()
    s = factored(dim, irn, jcn, val)
    rows = rows_of(dim, irn, jcn, val)
    rng = np.random.default_rng(3)
    xt = rng.standard_normal(dim)
    xt[rng.permutation(dim)[: dim // 2]] = 0.0
    b = to_scipy(dim, irn, jcn, val) @ xt
    X = solved(s, b[None, :])
    got = ea(s, b[None, :], X)
    ref = ref_errors(rows, b, X[0])
    check_against_ref(got, 0, ref, int(np.diff(rows[0]).max()), system)
    print("\n%s: |I2| = %d, omega2 = %.3e, cond2 = %.3e" % (system, got["n_i2"][0], got["omega2"][0], got["cond2"][0]))
    assert got["n_i2"][0] > 0 and got["cond2"][0] > 0.0 and np.isfinite(got["omega2"][0]) and got["omega2"][0] >= 0.0
    s.close()


# ---- 3b. exact cases -------------------------------------------------------------------------------------------------
def blockdiag_system(n, two_by_two, seed):
    rng = np.random.default_rng(seed)
    if not two_by_two:
        d = rng.choice([-1.0, 1.0], n) * np.exp(rng.uniform(-4, 4, n))
        i = np.arange(1, n + 1, dtype=np.int32)
        return n, i, i.copy(), d, np.diag(d)
    t = rng.choice([-1.0, 1.0], n // 2) * np.exp(rng.uniform(-4, 4, n // 2))
    irn, jcn, val = [], [], []
    A = np.zeros((n, n))
    for k, tk in enumerate(t):
        p = 2 * k
        for (a, b2, v) in ((p, p, tk), (p + 1, p, 2 * tk), (p + 1, p + 1, tk)):
            irn.append(a + 1), jcn.append(b2 + 1), val.append(v)
            A[a, b2] = A[b2, a] = v
    return n, np.array(irn, np.int32), np.array(jcn, np.int32), np.array(val), A


@pytest.mark.gpu
@pytest.mark.parametrize("two_by_two", [False, True])
def test_condest_exact_on_block_diagonal(two_by_two):
    n, irn, jcn, val, A = blockdiag_system(200, two_by_two, 5)
    s = factored(n, irn, jcn, val)
    kappa, anorm1, ainv1, nprod = s.condest()
    exact = np.abs(A).sum(axis=0).max() * np.abs(np.linalg.inv(A)).sum(axis=0).max()
    assert anorm1 == np.abs(A).sum(axis=0).max()
    assert abs(kappa - exact) <= 1e-15 * exact, (kappa, exact)
    s.close()


# ---- 4. condest takes dlacn2's decisions ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(ALL))
def test_condest_same_decisions_as_numpy_dlacn2(system):
    s = factored(*ALL[system]())
    n = s.dim

    def m(v):
        x = np.ascontiguousarray(v, np.float64).copy()
        assert s.solve(x, 1) == SYMSOLVER_SUCCESS
        return x

    est, nprod_ref = dlacn2(n, m, m)
    kappa, anorm1, ainv1, nprod = s.condest()
    assert nprod == nprod_ref, (nprod, nprod_ref)
    assert abs(ainv1 - est) <= 1e-12 * est, (ainv1, est)
    s.close()


# ---- 5. forward error ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_forward_error_bound_large():
    dim, irn, jcn, val = LARGE()
    s = factored(dim, irn, jcn, val)
    xt = np.random.default_rng(9).standard_normal(dim)
    b = to_scipy(dim, irn, jcn, val) @ xt
    X = solved(s, b[None, :])
    got = ea(s, b[None, :], X)
    fwd = np.abs(X[0] - xt).max() / np.abs(X[0]).max()
    print("\nN=400: forward error %.3e, ferr %.3e (ratio %.3e), omega1 %.3e cond1 %.3e omega2 %.3e cond2 %.3e nprod %d"
          % (fwd, got["ferr"][0], fwd / got["ferr"][0], got["omega1"][0], got["cond1"][0], got["omega2"][0],
             got["cond2"][0], got["nprod"][0]))
    assert fwd <= 10 * got["ferr"][0]
    s.close()


# ---- 6. bits -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("setup", ["default", "graph", "one_stream"])
def test_bits(setup, monkeypatch):
    if setup == "one_stream":
        monkeypatch.setenv("B200_ONE_STREAM", "1")
    opts = {"use_graph": 1 if setup == "graph" else 0}
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = factored(dim, irn, jcn, val, **opts)
    ref = factored(dim, irn, jcn, val, **opts)           # never makes the call
    monkeypatch.setenv("B200_SOLVE_BLOCK", "1")
    one = factored(dim, irn, jcn, val, **opts)
    monkeypatch.delenv("B200_SOLVE_BLOCK")
    rng = np.random.default_rng(12)
    B = rng.standard_normal((11, dim))
    X = solved(s, B)
    X[::2] += 1e-7 * rng.standard_normal((6, dim))
    for nrhs in (1, 3, 4, 5, 11):
        for cond in (True, False):
            full = ea(s, B[:nrhs], X[:nrhs], cond)
            assert_struct_bits(ea(s, B[:nrhs], X[:nrhs], cond, device=True), full, tag=("device", nrhs))
            assert_struct_bits(ea(s, B[:nrhs], X[:nrhs], cond), full, tag=("repeat", nrhs))
            assert_struct_bits(ea(one, B[:nrhs], X[:nrhs], cond), full, tag=("block 1", nrhs))
            for c in range(nrhs):
                assert_struct_bits(full, ea(s, B[c:c + 1], X[c:c + 1], cond), cols_a=[c], tag=("column", nrhs, c))
    c1, c2 = s.condest(), one.condest()
    assert c1 == s.condest() == c2
    # the factors, D and later solves are those of a handle that never made the call
    for nrhs in (1, 5):
        assert_bits(solved(s, B[:nrhs]), solved(ref, B[:nrhs]), ("solve", nrhs))
    assert_bits(s.enquire_indef()[2], ref.enquire_indef()[2], "D")
    for h in (s, ref, one):
        h.close()


# ---- 7. modes and launch counts ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_kept_singular_factors():
    from test_fredholm import handle, zeroed
    dim, irn, jcn, val, _ = zeroed("MBndryCntrl1_30", 2)
    s, st, _ = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR and len(s.enquire_zero_pivots()) == 2
    rows = rows_of(dim, irn, jcn, val)
    rng = np.random.default_rng(4)
    B = rng.standard_normal((3, dim))
    X = rng.standard_normal((3, dim))
    got = ea(s, B, X)
    for c in range(3):
        check_against_ref(got, c, ref_errors(rows, B[c], X[c]), int(np.diff(rows[0]).max()), ("singular", c))
        assert np.isfinite(got["omega1"][c]) and np.isfinite(got["omega2"][c])
    assert np.all(np.isinf(got["cond1"])) and np.all(np.isinf(got["cond2"])) and np.all(np.isinf(got["ferr"]))
    assert np.all(got["nprod"] == 0) and s.info()["launches_solve"] == 3
    kappa, anorm1, ainv1, nprod = s.condest()
    assert np.isinf(kappa) and np.isinf(ainv1) and nprod == 0 and anorm1 == got["anorm"][0]
    s.close()


@pytest.mark.gpu
def test_lifted_pivots_give_finite_estimates():
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    s = factored(n, irn, jcn, val)
    assert s.info()["num_forced"] > 0
    B = np.random.default_rng(4).standard_normal((2, n))
    got = ea(s, B, solved(s, B))
    for k in ("cond1", "cond2", "ferr", "omega1", "omega2"):
        assert np.all(np.isfinite(got[k])), k
    kappa, _, ainv1, nprod = s.condest()
    assert np.isfinite(kappa) and ainv1 > 0 and 1 <= nprod <= 11
    s.close()


@pytest.mark.gpu
def test_alter_d_doubles_the_estimate():
    s = factored(*SYSTEMS["MBndryCntrl1_30"]())
    k0, a0, m0, p0 = s.condest()
    _, _, dinv = s.enquire_indef()
    assert s.alter_d(2.0 * dinv) == SYMSOLVER_SUCCESS
    k1, a1, m1, p1 = s.condest()
    assert m1 == 2.0 * m0 and a1 == a0 and p1 == p0 and k1 == a1 * m1
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1"])
def test_launch_counts(block, monkeypatch):
    """cond = 0: 3; cond = 1: 3 + 10 T; condest: 2 + 10 nprod (job 0: 8 launches, default B200_SOLVE_DIRECT=2)"""
    if block is not None:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*mbndry_kkt(70, sigma_spread=3.0, seed=5)[:4])
    rng = np.random.default_rng(1)
    B = rng.standard_normal((5, s.dim))
    X = solved(s, B)
    for device in (False, True):
        got = ea(s, B, X, cond=False, device=device)
        assert s.info()["launches_solve"] == 3 and s.info()["ms_solve_gpu"] > 0.0
        for nrhs in (1, 5):
            got = ea(s, B[:nrhs], X[:nrhs], device=device)
            L, tot = s.info()["launches_solve"], int(got["nprod"].sum())
            if block == "1":
                assert L == 3 + 10 * tot, (L, tot)
            else:
                # lockstep: per block of 4 columns, the largest product count of its (up to 8) estimators
                assert (L - 3) % 10 == 0 and -(-tot // 8) <= (L - 3) // 10 <= tot, (L, tot)
    k, _, _, nprod = s.condest()
    assert s.info()["launches_solve"] == 2 + 10 * nprod
    s.close()


# ---- 8. refusals ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    L = s._L
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    b, x = np.ones(dim), np.ones(dim)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
    out = (Errors * 2)()

    def untouched():
        return all(getattr(o, k) == 42 for o in out for k in FIELDS)

    def refused(*args, match, device=False):
        for o in out:
            for k in FIELDS:
                setattr(o, k, 42)
        f = L.b200ldlt_error_analysis_device if device else L.b200ldlt_error_analysis
        assert f(s._h, *args, out) == SYMSOLVER_FATAL_ERROR and match in s.last_error(), s.last_error()
        assert untouched()

    refused(1, dp(b), dp(x), 1, match="no factors")
    with pytest.raises(RuntimeError, match="no factors"):
        s.condest()
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    refused(-1, dp(b), dp(x), 1, match="nrhs")
    refused(1, dp(b), dp(x), 2, match="cond")
    refused(1, None, dp(x), 0, match="NULL")
    refused(1, dp(b), None, 0, match="NULL")
    refused(1, None, None, 0, match="NULL", device=True)
    assert L.b200ldlt_error_analysis(s._h, 1, dp(b), dp(x), 1, None) == SYMSOLVER_FATAL_ERROR
    assert L.b200ldlt_condest(s._h, None, None, None, None) == SYMSOLVER_FATAL_ERROR and "kappa1" in s.last_error()
    # nrhs = 0: success, nothing written, nothing launched
    for o in out:
        o.anorm = 42
    assert L.b200ldlt_error_analysis(s._h, 0, None, None, 1, out) == SYMSOLVER_SUCCESS and out[0].anorm == 42
    assert s.info()["launches_solve"] == 0
    # SINGULAR outside keep mode leaves no factors
    v0 = val.copy()
    r = int(irn[0])
    v0[(irn == r) | (jcn == r)] = 0.0
    s.GetValuesArrayPtr()[:] = v0
    assert s.factor(False, 0)[0] == SYMSOLVER_SINGULAR
    refused(1, dp(b), dp(x), 0, match="no factors")
    # Schur mode
    s.GetValuesArrayPtr()[:] = val
    assert s.set_schur(np.arange(dim - 5, dim)) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    refused(1, dp(b), dp(x), 1, match="Schur mode")
    with pytest.raises(RuntimeError, match="Schur mode"):
        s.condest()
    assert s.set_schur([]) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    assert np.isfinite(s.condest()[0])
    # sharded handle
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    refused(1, dp(b), dp(x), 1, match="sharded")
    with pytest.raises(RuntimeError, match="sharded"):
        s.condest()
    s.close()
