"""Zero pivots, keep mode and the Fredholm alternative (b200ldlt_set_singular_action, b200ldlt_enquire_zero_pivots,
b200ldlt_solve_fredholm / _device) and ma97_solve_fredholm_d of the HSL_MA97 shim."""
import ctypes as C

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt, to_scipy

from test_partial_solve import LARGE, SYSTEMS, assert_bits, device_doubles, run

NEW_SYMBOLS = ["b200ldlt_set_singular_action", "b200ldlt_enquire_zero_pivots", "b200ldlt_solve_fredholm",
               "b200ldlt_solve_fredholm_device", "ma97_solve_fredholm_d"]
ALL = dict(SYSTEMS, mbndry400=LARGE)


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


def zeroed(system, k, seed=0):
    """the system with k variables' rows and columns zeroed (values only, same pattern), and those variables -- drawn so
    that the rank drops by exactly k: no other row becomes zero with them and, for n <= 2000, numpy's eigenvalues show
    exactly k zeros (zeroing a variable of LukVlE1 can also leave a constraint dependent on the others)"""
    dim, irn, jcn, val = ALL[system]()
    rng = np.random.default_rng(seed + k)
    while True:
        rows = np.sort(rng.choice(dim, k, replace=False))
        v = val.copy()
        v[np.isin(irn - 1, rows) | np.isin(jcn - 1, rows)] = 0.0
        nz = np.zeros(dim, bool)
        nz[irn[v != 0] - 1] = True
        nz[jcn[v != 0] - 1] = True
        if nz.sum() != dim - k:
            continue
        if dim <= 2000:
            mag = np.abs(np.linalg.eigvalsh(to_scipy(dim, irn, jcn, v).toarray()))
            if np.sum(mag <= 1e-12 * mag.max()) != k:
                continue
        return dim, irn, jcn, v, rows


def handle(dim, irn, jcn, val, keep=1, **opts):
    s = B200Ldlt(**opts)
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    assert s.set_singular_action(keep) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(False, 0)
    return s, st, neg


def fred_device(s, B, tol):
    import torch
    nrhs, dim = B.shape
    X = torch.zeros(2 * nrhs * dim, dtype=torch.float64, device="cuda")
    X[:nrhs * dim] = torch.tensor(B.ravel())
    st, cons = s.solve_fredholm_device(X.data_ptr(), nrhs, tol)
    assert st == SYMSOLVER_SUCCESS, s.last_error()
    x = X.cpu().numpy().reshape(2 * nrhs, dim)
    return x[:nrhs], x[nrhs:], cons


def fred(s, B, tol, device=False):
    """(X, F, consistent) for the columns of B (nrhs x dim, row c = column c)"""
    if device:
        return fred_device(s, B, tol)
    X, F, c = s.solve_fredholm(B.T, tol)
    return X.T, F.T, c


# ---- 1. zeroed rows: exact results ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("system", sorted(ALL))
def test_zeroed_rows_exact(system, k):
    dim, irn, jcn, val, rows = zeroed(system, k)
    s, st, neg = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR, s.last_error()
    Z = s.enquire_zero_pivots()
    assert len(Z) == k and s.info()["num_tiny"] == k
    var, ty, dinv = s.enquire_indef()
    assert sorted(var[Z]) == list(rows) and np.all(ty[Z] == 1) and np.all(dinv[Z] == 0.0)
    assert s.NumberOfNegEVals() == neg == s.info()["num_neg"]
    if dim <= 2000:
        ev = np.linalg.eigvalsh(to_scipy(dim, irn, jcn, val).toarray())
        scale = np.abs(ev).max()
        mag = np.sort(np.abs(ev))
        assert mag[k - 1] <= 1e-12 * scale and mag[k] >= 1e3 * mag[k - 1], (mag[k - 1], mag[k])   # a clear gap
        gap = np.sqrt(mag[k - 1] * mag[k])
        assert neg == int(np.sum(ev < -gap))
    rng = np.random.default_rng(1)
    B = rng.standard_normal((3, dim))
    B[:, rows] = 0.0
    X, F, c = fred(s, B, 0.0)
    assert c.all() and not F.any()
    B2 = rng.standard_normal((3, dim))
    X, F, c = fred(s, B2, 0.0)
    assert not c.any()
    S = device_doubles(s.device_ptr("scale"), dim)
    for i in range(3):
        f = np.zeros(dim)
        f[rows] = S[rows] ** 2 * B2[i, rows]
        assert np.array_equal(F[i], f), np.abs(F[i] - f).max()    # exact: S is a power of two
    s.close()


# ---- 2. identities, bit for bit -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1"])
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random", "mbndry400"])
def test_identities_bitwise(system, block, monkeypatch):
    if block:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    dim, irn, jcn, val, rows = zeroed(system, 2)
    s, st, _ = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR
    Z = s.enquire_zero_pivots()
    rng = np.random.default_rng(2)
    B = rng.standard_normal((13, dim))
    B[::3, rows] = 0.0                      # mixed consistent / inconsistent columns
    X, F, c = fred(s, B, 1e-10)
    assert list(c) == [i % 3 == 0 for i in range(13)]
    assert_bits(X, run(s, 0, B, False), "x = job 0")
    Y = run(s, 1, B, False)
    Zv = np.zeros_like(Y)
    Zv[:, Z] = Y[:, Z]
    assert_bits(F, run(s, 3, Zv, False), "f = job 3 (z)")
    A = to_scipy(dim, irn, jcn, val)
    r = A @ X.T + s.lmultiply(0, Zv.ravel(), 13).reshape(13, dim).T - B.T
    ref = (abs(A) @ np.abs(X.T)).max() + np.abs(B).max()
    assert np.abs(r).max() <= 1e-12 * ref, np.abs(r).max() / ref      # A x + S^-1 P L z = b to rounding
    Xd, Fd, cd = fred(s, B, 1e-10, device=True)
    assert_bits(Xd, X, "device x")
    assert_bits(Fd, F, "device f")
    assert (cd == c).all()
    for i in (0, 1, 5, 12):
        xi, fi, ci = fred(s, B[i:i + 1], 1e-10)
        assert_bits(xi[0], X[i], "column %d x" % i)
        assert_bits(fi[0], F[i], "column %d f" % i)
        assert ci[0] == c[i]
    for nrhs in range(1, 13):
        Xn, Fn, cn = fred(s, B[:nrhs], 1e-10)
        assert_bits(Xn, X[:nrhs])
        assert_bits(Fn, F[:nrhs])
    st2, _ = s.refactor()
    assert st2 == SYMSOLVER_SINGULAR
    assert list(s.enquire_zero_pivots()) == list(Z)
    X2, F2, _ = fred(s, B, 1e-10)
    assert_bits(X2, X)
    assert_bits(F2, F)
    s.close()


# ---- 3. dependent rows: a duplicated constraint ---------------------------------------------------------------------
def dup_kkt(nx, nc, seed):
    """[[H, J^T], [J, 0]] with H SPD and the last constraint row a copy of the first: rank deficiency 1, null vector
    (0, e_0 - e_last) in the multipliers"""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    Bm = sp.random(nx, nx, density=0.05, random_state=seed)
    H = sp.tril(Bm @ Bm.T + sp.identity(nx), format="coo")
    J = sp.random(nc - 1, nx, density=0.1, random_state=seed + 1, format="lil")
    for r in range(nc - 1):
        J[r, (r * 7 + 3) % nx] += 2.0 + rng.uniform()
    J = sp.vstack([J, J[0]]).tocoo()
    irn = np.concatenate([H.row, nx + J.row]) + 1
    jcn = np.concatenate([H.col, J.col]) + 1
    val = np.concatenate([H.data, J.data])
    null = np.zeros(nx + nc)
    null[nx], null[nx + nc - 1] = 1.0, -1.0
    return nx + nc, irn.astype(np.int32), jcn.astype(np.int32), val, null


# Which kind each configuration produces (zero pivots: factors kept; lifted zero: SINGULAR without factors) is printed
# by the test; at least one configuration must give zero pivots, and every configuration that does is checked.
@pytest.mark.gpu
def test_dependent_rows():
    kinds, checked = {}, 0
    for (nx, nc, seed) in [(40, 12, 0), (120, 40, 1), (300, 100, 2)]:
        dim, irn, jcn, val, null = dup_kkt(nx, nc, seed)
        A = to_scipy(dim, irn, jcn, val)
        assert np.linalg.matrix_rank(A.toarray()) == dim - 1
        for ordering in (0, 1):
            s, st, _ = handle(dim, irn, jcn, val, ordering=ordering)
            assert st == SYMSOLVER_SINGULAR
            Z = s.enquire_zero_pivots() if "no factors" not in s.last_error() else None
            kinds[(nx, nc, ordering)] = "zero pivots" if Z is not None else "lifted zero"
            if Z is None:
                assert "lifted zero" in s.last_error()
                with pytest.raises(RuntimeError, match="no factors"):
                    s.solve_fredholm(np.ones(dim), 1e-10)
                s.close()
                continue
            checked += 1
            assert len(Z) == 1
            rng = np.random.default_rng(3)
            w = rng.standard_normal(dim)
            b = A @ w
            x, f, c = s.solve_fredholm(b, 1e-10)
            assert c[0]
            res = np.abs(A @ x - b).max() / (abs(A).max() * np.abs(x).max() + np.abs(b).max())
            assert res <= 1e-9, res
            b2 = b + null
            x, f, c = s.solve_fredholm(b2, 1e-10)
            assert not c[0]
            Af = A @ f
            assert np.abs(Af).max() <= 1e-12 * np.abs(abs(A) @ np.abs(f)).max()
            yv = b2.copy()
            assert s.solve_partial(1, yv) == SYMSOLVER_SUCCESS
            assert np.isclose(b2 @ f, np.sum(yv[Z] ** 2), rtol=1e-10)
            cosang = abs(f @ null) / (np.linalg.norm(f) * np.linalg.norm(null))
            assert cosang >= 1 - 1e-10, cosang
            s.close()
    print("dependent-row systems:", kinds)
    assert checked >= 1, kinds


# ---- 4. keep mode on a non-singular matrix ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "mbndry30_wzero"])
def test_keep_mode_nonsingular_unchanged(system):
    dim, irn, jcn, val = ALL[system]()
    s0, st0, neg0 = handle(dim, irn, jcn, val, keep=0)
    s1, st1, neg1 = handle(dim, irn, jcn, val, keep=1)
    assert st0 == st1 == SYMSOLVER_SUCCESS and neg0 == neg1
    assert s0.info()["launches_factor"] == s1.info()["launches_factor"]
    for a, b in zip(s0.enquire_indef(), s1.enquire_indef()):
        assert_bits(a.astype(np.float64), b.astype(np.float64))
    B = np.random.default_rng(4).standard_normal((3, dim))
    for job in range(5):
        assert_bits(run(s0, job, B, False), run(s1, job, B, False), "job %d" % job)
    assert len(s1.enquire_zero_pivots()) == 0
    X, F, c = fred(s1, B, 0.0)
    assert c.all() and not F.any()
    assert_bits(X, run(s0, 0, B, False))
    s0.close()
    s1.close()


# ---- 5. launch counts and refusals ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1"])
def test_launch_counts(block, monkeypatch):
    if block:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    dim, irn, jcn, val, rows = zeroed("mbndry400", 2)
    s, st, _ = handle(dim, irn, jcn, val)
    B = np.random.default_rng(5).standard_normal((8, dim))
    run(s, 1, B[:1], False)
    D = s.info()["launches_solve"] - 3        # job 1: 3 + D
    for nrhs in (1, 8):
        fred(s, B[:nrhs], 1e-10)
        want = -(-nrhs // 4) * (5 + 2 * D) if block is None else nrhs * (8 + 3 * D)
        assert s.info()["launches_solve"] == want, (nrhs, D, s.info()["launches_solve"])
    s.close()


@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val, rows = zeroed("MBndryCntrl1_30", 1)
    s, st, _ = handle(dim, irn, jcn, val, keep=0)
    assert st == SYMSOLVER_SINGULAR
    x, cons = np.zeros(2 * dim), np.zeros(1, np.int32)
    L = s._L
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    xp, cp = x.ctypes.data_as(dp), cons.ctypes.data_as(ip)
    assert L.b200ldlt_solve_fredholm(s._h, 1, 0.0, xp, cp) == SYMSOLVER_FATAL_ERROR and "no factors" in s.last_error()
    with pytest.raises(RuntimeError):
        s.enquire_zero_pivots()
    assert s.set_singular_action(2) == SYMSOLVER_FATAL_ERROR
    assert s.set_singular_action(1) == SYMSOLVER_SUCCESS
    assert s.refactor()[0] == SYMSOLVER_SINGULAR
    x[:dim] = 1.0
    before = x.copy()
    for args in [(-1, 0.0, xp, cp), (1, -1.0, xp, cp), (1, float("nan"), xp, cp), (1, 0.0, None, cp), (1, 0.0, xp, None)]:
        assert L.b200ldlt_solve_fredholm(s._h, *args) == SYMSOLVER_FATAL_ERROR
        assert "solve_fredholm" in s.last_error()
        assert_bits(x, before)
    assert L.b200ldlt_solve_fredholm(s._h, 1, 0.0, xp, cp) == SYMSOLVER_SUCCESS
    s.close()
    # sharded handle
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s, st, _ = handle(dim, irn, jcn, val)
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    x = np.zeros(2 * dim)
    assert L.b200ldlt_solve_fredholm(s._h, 1, 0.0, x.ctypes.data_as(dp), cp) == SYMSOLVER_FATAL_ERROR
    assert "sharded" in s.last_error()
    s.close()


# ---- 6. the HSL_MA97 shim -------------------------------------------------------------------------------------------
CTRL_ACTION, CTRL_CONSIST_TOL = 4, 104          # byte offsets in ma97_control_d
INFO_RANK, INFO_NUM_NEG = 16, 56                # ... in ma97_info_d


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random"])
def test_ma97_shim_fredholm(system, built_lib):
    import scipy.sparse as sp
    dim, irn, jcn, val, rows = zeroed(system, 2)
    Lo = sp.tril(to_scipy(dim, irn, jcn, val)).tocsc()
    Lo.sort_indices()
    ptr, row, cv = Lo.indptr.astype(np.int32), Lo.indices.astype(np.int32), Lo.data.astype(np.float64)
    cols = np.repeat(np.arange(dim), np.diff(ptr)).astype(np.int32)
    ref, st, neg = handle(dim, row + 1, cols + 1, cv, pivtol=0.01, pivtolmax=0.01)
    assert st == SYMSOLVER_SINGULAR
    lib = C.CDLL(built_lib)
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    ctrl, info = C.create_string_buffer(1024), C.create_string_buffer(1024)
    akeep, fkeep = C.c_void_p(), C.c_void_p()
    keeps = (C.byref(akeep), C.byref(fkeep), ctrl, info)
    geti = lambda off: C.cast(C.addressof(info) + off, ip)[0]   # noqa: E731
    lib.ma97_default_control_d(ctrl)
    assert C.cast(C.addressof(ctrl) + CTRL_ACTION, ip)[0] == 1
    C.cast(C.addressof(ctrl) + CTRL_CONSIST_TOL, dp)[0] = 1e-10
    lib.ma97_analyse_d(C.c_int(0), C.c_int(dim), ptr.ctypes.data_as(ip), row.ctypes.data_as(ip), cv.ctypes.data_as(dp),
                       C.byref(akeep), ctrl, info, None)
    assert geti(0) == 0
    fac = lambda: lib.ma97_factor_d(C.c_int(4), ptr.ctypes.data_as(ip), row.ctypes.data_as(ip),  # noqa: E731
                                    cv.ctypes.data_as(dp), C.byref(akeep), C.byref(fkeep), ctrl, info, None)
    fac()
    assert geti(0) == 7 and geti(INFO_RANK) == dim - 2 and geti(INFO_NUM_NEG) == neg
    rng = np.random.default_rng(6)
    B = rng.standard_normal((3, dim))
    B[0, rows] = 0.0
    X = B.copy()
    lib.ma97_solve_d(C.c_int(0), C.c_int(3), X.ctypes.data_as(dp), C.c_int(dim), *keeps)
    assert geti(0) == 0
    assert_bits(X, run(ref, 0, B, False), "ma97_solve_d")
    Xr, Fr, cr = fred(ref, B, 1e-10)
    for ldx in (dim, dim + 3):
        x = np.full((6, ldx), 7.0)
        x[:3, :dim] = B
        flags = np.full(3, -1, np.int32)
        lib.ma97_solve_fredholm_d(C.c_int(3), flags.ctypes.data_as(ip), x.ctypes.data_as(dp), C.c_int(ldx), *keeps)
        assert geti(0) == 0
        assert list(flags) == [1, 0, 0] == list(cr.astype(int))
        assert_bits(x[:3, :dim], Xr)
        assert np.all(x[3, :] == 7.0)                     # consistent column: untouched
        assert_bits(x[4:, :dim], Fr[1:])
        assert np.all(x[:, dim:] == 7.0)
    d = np.zeros(2 * dim)
    lib.ma97_enquire_indef_d(C.byref(akeep), C.byref(fkeep), ctrl, info, None, d.ctypes.data_as(dp))
    assert geti(0) == 0 and np.all(d[2 * ref.enquire_zero_pivots()] == 0.0)
    X = B.copy()
    lib.ma97_factor_solve_d(C.c_int(4), ptr.ctypes.data_as(ip), row.ctypes.data_as(ip), cv.ctypes.data_as(dp),
                            C.c_int(3), X.ctypes.data_as(dp), C.c_int(dim), C.byref(akeep), C.byref(fkeep), ctrl, info, None)
    assert geti(0) == 7
    assert_bits(X, run(ref, 0, B, False), "factor_solve after flag 7")
    C.cast(C.addressof(ctrl) + CTRL_ACTION, ip)[0] = 0
    fac()
    assert geti(0) == -7
    X = B.copy()
    lib.ma97_solve_d(C.c_int(0), C.c_int(1), X.ctypes.data_as(dp), C.c_int(dim), *keeps)
    assert geti(0) == -1
    lib.ma97_finalise_d(C.byref(akeep), C.byref(fkeep))
    ref.close()
