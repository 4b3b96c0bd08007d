"""Multiplication by the factors (b200ldlt_lmultiply / _device) and alteration of D (b200ldlt_alter_d), through the C ABI
and the HSL_MA97 shim (ma97_lmultiply_d, ma97_alter_d, ma97_enquire_posdef_d).

S A S = P L D L^T P^T.  trans 0: y = S^-1 P L x (pivot -> original order, the inverse of job 1); trans 1:
y = L^T P^T S^-1 x (original -> pivot order, the inverse of job 3).  So  lmultiply(0, D lmultiply(1, v)) = A v."""
import ctypes as C

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt, to_scipy

from test_partial_solve import LARGE, SYSTEMS, assert_bits, d_blocks, factored, run

NEW_SYMBOLS = ["b200ldlt_lmultiply", "b200ldlt_lmultiply_device", "b200ldlt_alter_d", "ma97_lmultiply_d",
               "ma97_alter_d", "ma97_enquire_posdef_d"]


def lmul(s, trans, X, device):
    """trans on the columns of X (nrhs x dim, row c = column c), host or device entry point"""
    nrhs, dim = X.shape
    if device:
        import torch
        dx = torch.tensor(X.ravel(), dtype=torch.float64, device="cuda")
        dy = torch.empty_like(dx)
        assert s.lmultiply_device(trans, dx.data_ptr(), dy.data_ptr(), nrhs) == SYMSOLVER_SUCCESS, s.last_error()
        return dy.cpu().numpy().reshape(nrhs, dim)
    return s.lmultiply(trans, X.ravel(), nrhs).reshape(nrhs, dim)


def apply_d(ty, dinv2, V):
    """D V (pivot order, rows of V are vectors) from the D^-1 entries of enquire_indef, without forming D densely"""
    V = np.atleast_2d(V)
    with np.errstate(divide="ignore", invalid="ignore"):   # (2x2 pivots may have a zero diagonal in D^-1: overwritten)
        out = V / dinv2[:, 0]
    two = np.flatnonzero(ty == 2)
    a, b, c = dinv2[two, 0], dinv2[two, 1], dinv2[two + 1, 0]
    det = a * c - b * b                              # D block = [[c, -b], [-b, a]] / det
    v0, v1 = V[:, two], V[:, two + 1]
    out[:, two] = (c * v0 - b * v1) / det
    out[:, two + 1] = (-b * v0 + a * v1) / det
    return out


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


# ---- 1. inverse identities ------------------------------------------------------------------------------------------
# Measured on an H100 (H100 80GB HBM3, both entry points, nrhs 1 and 3): the larger of
# ||job1(lmultiply(0, x)) - x||_inf / ||x||_inf and ||lmultiply(1, job3(b)) - b||_inf / ||b||_inf is 2.1e-16 (hs071_0)
# to 3.4e-15 (MBndryCntrl1_30, mbndry30_wzero).  The tolerance sits about 1e4 above that: room for other matrices' growth
# in L, while a wrong entry of L shows as an O(1) error.
INV_TOL = 1e-11


@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(SYSTEMS))
def test_inverse_identities(system):
    s = factored(*SYSTEMS[system]())
    rng = np.random.default_rng(1)
    worst = 0.0
    for device in (False, True):
        for nrhs in (1, 3):
            X = rng.standard_normal((nrhs, s.dim))
            e1 = np.abs(run(s, 1, lmul(s, 0, X, device), device) - X).max() / np.abs(X).max()
            e3 = np.abs(lmul(s, 1, run(s, 3, X, device), device) - X).max() / np.abs(X).max()
            worst = max(worst, e1, e3)
            assert e1 <= INV_TOL and e3 <= INV_TOL, (device, nrhs, e1, e3)
    print("MEASURED inverse %s %.2e" % (system, worst))
    s.close()


# ---- 2. adjoint -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(SYSTEMS) + ["mbndry400"])
def test_adjoint(system):
    s = factored(*(LARGE() if system == "mbndry400" else SYSTEMS[system]()))
    rng = np.random.default_rng(3)
    for _ in range(2):
        x, y = rng.standard_normal((1, s.dim)), rng.standard_normal((1, s.dim))
        a, b = lmul(s, 0, x, True)[0], lmul(s, 1, y, True)[0]
        lhs, rhs = a @ y[0], x[0] @ b
        assert abs(lhs - rhs) <= 1e-12 * max(np.abs(a * y[0]).sum(), np.abs(x[0] * b).sum()), (lhs, rhs)
    s.close()


# ---- 3. reconstruction of A -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(SYSTEMS))
def test_reconstruction(system):
    dim, irn, jcn, val = SYSTEMS[system]()
    if dim > 2000:
        pytest.skip("dense reconstruction for n <= 2000 only")
    s = factored(dim, irn, jcn, val)
    if s.info()["num_forced"] > 0:
        pytest.skip("lifted pivots: the factors describe a perturbed matrix")
    A = to_scipy(dim, irn, jcn, val).toarray()
    var, ty, dinv2 = s.enquire_indef()
    T = lmul(s, 1, np.eye(dim), False)             # row j = L^T P^T S^-1 e_j
    R = lmul(s, 0, apply_d(ty, dinv2, T), False)   # row j = A e_j
    err = np.abs(R - A).max() / np.abs(A).max()
    print("MEASURED reconstruction %s %.2e" % (system, err))
    assert err <= 1e-13, err
    # the two directions are transposes of each other, entry for entry (a unit vector picks single entries of L)
    M0 = lmul(s, 0, np.eye(dim), True)            # row p = S^-1 P L e_p
    assert np.array_equal(M0, T.T)
    s.close()


# ---- 4. the full-size factor probe ----------------------------------------------------------------------------------
PROBE = [({}, {}), ({"B200_ONE_STREAM": "1"}, {}), ({"B200_CB_AT_END": "1"}, {}), ({"B200_NO_PDL": "1"}, {}),
         ({"B200_NO_WARP2": "1"}, {}), ({}, {"tc_schur_min_r": 256})]


@pytest.mark.gpu
@pytest.mark.parametrize("env,opts", PROBE, ids=["default", "one_stream", "cb_at_end", "no_pdl", "no_warp2", "tc_schur"])
def test_factor_probe_full_size(env, opts, monkeypatch):
    """||A v - S^-1 P L D L^T P^T S^-1 v||_inf / || |A| |v| ||_inf on MBndryCntrl1 N=400 for random v, without a solve"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dim, irn, jcn, val, nc = mbndry_kkt(400)
    s = factored(dim, irn, jcn, val, **opts)
    A = to_scipy(dim, irn, jcn, val)
    var, ty, dinv2 = s.enquire_indef()
    V = np.random.default_rng(7).standard_normal((3, dim))
    R = lmul(s, 0, apply_d(ty, dinv2, lmul(s, 1, V, True)), True)
    worst = 0.0
    for c in range(3):
        r = np.abs(A @ V[c] - R[c]).max() / np.abs(abs(A) @ np.abs(V[c])).max()
        worst = max(worst, r)
    print("MEASURED probe %s %.2e" % (env or opts or "default", worst))
    assert worst <= 1e-12, worst
    s.close()


# ---- 5. blocks, reproducibility, launches ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random", "mbndry30_wzero"])
def test_blocks_bit_identical_to_columns(system):
    s = factored(*SYSTEMS[system]())
    for nrhs in range(1, 14):
        X = np.random.default_rng(nrhs).standard_normal((nrhs, s.dim))
        for trans in (0, 1):
            for device in (False, True):
                Y = lmul(s, trans, X, device)
                assert_bits(Y, lmul(s, trans, X, device), (nrhs, trans, device, "repeat"))
                for c in range(nrhs):
                    assert_bits(Y[c], lmul(s, trans, X[c:c + 1], device)[0], (nrhs, trans, device, c))
    s.close()


@pytest.mark.gpu
def test_large_blocks_and_in_place():
    s = factored(*LARGE())
    import torch
    X = np.random.default_rng(4).standard_normal((8, s.dim))
    for trans in (0, 1):
        Y = lmul(s, trans, X, True)
        assert_bits(Y, lmul(s, trans, X, True), trans)
        assert_bits(Y[5], lmul(s, trans, X[5:6], True)[0], trans)
        d = torch.tensor(X.ravel(), dtype=torch.float64, device="cuda")
        assert s.lmultiply_device(trans, d.data_ptr(), d.data_ptr(), 8) == SYMSOLVER_SUCCESS
        assert_bits(d.cpu().numpy().reshape(8, s.dim), Y, ("in place", trans))
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1", "3"])
def test_launch_counts(block, monkeypatch):
    """two launches per block of columns"""
    if block is not None:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*mbndry_kkt(70, sigma_spread=3.0, seed=5)[:4])
    width = 8 if block is None else int(block)
    for nrhs in (1, 8, 13):
        X = np.random.default_rng(nrhs).standard_normal((nrhs, s.dim))
        for trans in (0, 1):
            for device in (False, True):
                lmul(s, trans, X, device)
                info = s.info()
                assert info["launches_solve"] == 2 * -(-nrhs // width), (nrhs, trans, device, info["launches_solve"])
                assert info["ms_solve_gpu"] > 0.0
    s.close()


# ---- 6. alter_d -----------------------------------------------------------------------------------------------------
def all_jobs(s, B):
    return [run(s, job, B, device) for job in range(5) for device in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["hs071_0", "MBndryCntrl1_30", "mbndry30_wzero", "random"])
def test_alter_round_trip_and_refusals(system):
    s = factored(*SYSTEMS[system]())
    n = s.dim
    B = np.random.default_rng(2).standard_normal((2, n))
    before = all_jobs(s, B)
    var, ty, dinv2 = s.enquire_indef()
    assert s.alter_d(dinv2) == SYMSOLVER_SUCCESS, s.last_error()
    for a, b in zip(all_jobs(s, B), before):
        assert_bits(a, b, "round trip")
    # refused: nothing changes
    one = int(np.flatnonzero(ty != 2)[0])
    bad_off = dinv2.copy()
    bad_off[one, 1] = 0.5
    bad_nan = dinv2.copy()
    bad_nan[n // 2, 0] = np.nan
    bad_inf = dinv2.copy()
    bad_inf[-1, 1] = np.inf
    for bad in (bad_off, bad_nan, bad_inf):
        assert s.alter_d(bad) == SYMSOLVER_FATAL_ERROR and "refused" in s.last_error()
        for a, b in zip(all_jobs(s, B), before):
            assert_bits(a, b, "refused")
        assert_bits(s.enquire_indef()[2], dinv2, "refused: D")
    s.close()


def modulus(ty, dinv2):
    """D^-1 of |D|: |d| for 1x1 pivots, the eigen-modulus for 2x2 blocks (the inverse of |D| is the modulus of D^-1)"""
    m = dinv2.copy()
    m[ty == 1, 0] = np.abs(dinv2[ty == 1, 0])
    for p in np.flatnonzero(ty == 2):
        Bi = np.array([[dinv2[p, 0], dinv2[p, 1]], [dinv2[p, 1], dinv2[p + 1, 0]]])
        w, U = np.linalg.eigh(Bi)
        Mb = (U * np.abs(w)) @ U.T
        m[p, 0], m[p, 1], m[p + 1, 0] = Mb[0, 0], Mb[0, 1], Mb[1, 1]
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "mbndry30_wzero", "random"])
def test_alter_modulus_preconditioner_and_refactor(system):
    dim, irn, jcn, val = SYSTEMS[system]()
    s = factored(dim, irn, jcn, val)
    info0 = s.info()
    var, ty, dinv2 = s.enquire_indef()
    b = np.random.default_rng(6).standard_normal((1, dim))
    x0 = run(s, 0, b, True)
    m = modulus(ty, dinv2)
    assert s.alter_d(m) == SYMSOLVER_SUCCESS, s.last_error()
    assert_bits(s.enquire_indef()[2], m, "altered D")
    # L |D| L^T in numpy, from the factors themselves
    Lh = lmul(s, 0, np.eye(dim), False).T          # S^-1 P L
    Aabs = Lh @ d_blocks(ty, m) @ Lh.T
    assert np.linalg.eigvalsh(Aabs).min() > 0
    xr = np.linalg.solve(Aabs, b[0])
    x = run(s, 0, b, True)[0]
    err = np.abs(x - xr).max() / np.abs(xr).max()
    res = np.abs(Aabs @ x - b[0]).max() / (np.abs(Aabs).max() * np.abs(x).max() + np.abs(b).max())
    print("MEASURED modulus %s diff %.2e residual %.2e" % (system, err, res))
    assert err <= 1e-8 and res <= 1e-13, (err, res)
    assert s.info()["num_neg"] == info0["num_neg"] and s.NumberOfNegEVals() == info0["num_neg"]
    # the next factorisation computes D afresh
    assert s.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    assert_bits(s.enquire_indef()[2], dinv2, "refactor")
    assert_bits(run(s, 0, b, True), x0, "refactor: solve")
    s.close()


# ---- 7. refusals ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    x = np.ones(dim)
    d2 = np.ones((dim, 2))
    with pytest.raises(RuntimeError, match="no factors"):
        s.lmultiply(0, x)
    assert s.alter_d(d2) == SYMSOLVER_FATAL_ERROR and "no factors" in s.last_error()
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    for trans in (-1, 2):
        with pytest.raises(RuntimeError, match="trans"):
            s.lmultiply(trans, x)
        assert s.lmultiply_device(trans, 0, 0) == SYMSOLVER_FATAL_ERROR
    s.lmultiply(1, x)
    v0 = val.copy()
    r = int(irn[0])
    v0[(irn == r) | (jcn == r)] = 0.0
    s.GetValuesArrayPtr()[:] = v0
    assert s.factor(False, 0)[0] == SYMSOLVER_SINGULAR
    with pytest.raises(RuntimeError, match="no factors"):
        s.lmultiply(0, x)
    assert s.alter_d(d2) == SYMSOLVER_FATAL_ERROR and "no factors" in s.last_error()
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    L = s._L
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    for trans in (0, 1):
        with pytest.raises(RuntimeError, match="sharded"):
            s.lmultiply(trans, x)
    assert s.alter_d(d2) == SYMSOLVER_FATAL_ERROR and "sharded" in s.last_error()
    s.close()


# ---- 8. the HSL_MA97 shim -------------------------------------------------------------------------------------------
class Ma97:
    """the shim through ctypes on the lower-triangle CSC of a matrix, and a C ABI handle on the same triplets"""

    def __init__(self, lib_path, dim, irn, jcn, val):
        import scipy.sparse as sp
        Lo = sp.tril(to_scipy(dim, irn, jcn, val)).tocsc()
        Lo.sort_indices()
        self.ptr, self.row = Lo.indptr.astype(np.int32), Lo.indices.astype(np.int32)
        self.cv = Lo.data.astype(np.float64)
        cols = np.repeat(np.arange(dim), np.diff(self.ptr)).astype(np.int32)
        self.s = factored(dim, self.row + 1, cols + 1, self.cv, pivtol=0.01, pivtolmax=0.01)
        self.dim = dim
        self.lib = lib = C.CDLL(lib_path)
        self.ctrl, self.info = C.create_string_buffer(1024), C.create_string_buffer(1024)
        self.akeep, self.fkeep = C.c_void_p(), C.c_void_p()
        ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
        self.ip, self.dp = ip, dp
        lib.ma97_default_control_d(self.ctrl)
        lib.ma97_analyse_d(C.c_int(0), C.c_int(dim), self.ptr.ctypes.data_as(ip), self.row.ctypes.data_as(ip),
                           self.cv.ctypes.data_as(dp), C.byref(self.akeep), self.ctrl, self.info, None)
        assert self.flag() == 0
        self.scale = np.zeros(dim)
        lib.ma97_factor_d(C.c_int(4), self.ptr.ctypes.data_as(ip), self.row.ctypes.data_as(ip), self.cv.ctypes.data_as(dp),
                          C.byref(self.akeep), C.byref(self.fkeep), self.ctrl, self.info, self.scale.ctypes.data_as(dp))

    def flag(self):
        return C.cast(self.info, C.POINTER(C.c_int))[0]

    def keeps(self):
        return C.byref(self.akeep), C.byref(self.fkeep), self.ctrl, self.info

    def close(self):
        self.lib.ma97_finalise_d(C.byref(self.akeep), C.byref(self.fkeep))
        self.s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["hs071_0", "MBndryCntrl1_30", "mbndry30_wzero"])
def test_ma97_shim_lmultiply_and_alter(system, built_lib):
    m = Ma97(built_lib, *SYSTEMS[system]())
    assert m.flag() == 0
    dim, lib, dp = m.dim, m.lib, m.dp
    rng = np.random.default_rng(5)
    for trans in (0, 1):
        for k, ldx, ldy in ((1, dim, dim), (3, dim, dim), (3, dim + 7, dim + 2), (2, dim, dim + 5)):
            B = rng.standard_normal((k, dim))
            X = np.full((k, ldx), 42.0)
            X[:, :dim] = B
            Y = np.full((k, ldy), -3.0)
            lib.ma97_lmultiply_d(C.c_int(trans), C.c_int(k), X.ctypes.data_as(dp), C.c_int(ldx), Y.ctypes.data_as(dp),
                                 C.c_int(ldy), *m.keeps())
            assert m.flag() == 0, (trans, k, ldx, ldy)
            assert_bits(Y[:, :dim], lmul(m.s, trans, B, False), (trans, k, ldx, ldy))
            assert np.all(Y[:, dim:] == -3.0) and np.all(X[:, dim:] == 42.0)
    Y = np.full(dim, 7.0)
    lib.ma97_lmultiply_d(C.c_int(0), C.c_int(0), None, C.c_int(dim), Y.ctypes.data_as(dp), C.c_int(dim), *m.keeps())
    assert m.flag() == 0 and np.all(Y == 7.0)                                # k = 0: nothing
    lib.ma97_lmultiply_d(C.c_int(2), C.c_int(1), Y.ctypes.data_as(dp), C.c_int(dim), Y.ctypes.data_as(dp), C.c_int(dim),
                         *m.keeps())
    assert m.flag() < 0
    # enquire -> alter round trip: nothing changes
    d = np.zeros((dim, 2))
    lib.ma97_enquire_indef_d(C.byref(m.akeep), C.byref(m.fkeep), m.ctrl, m.info, None, d.ctypes.data_as(dp))
    assert m.flag() == 0
    B = rng.standard_normal((1, dim))
    x0 = run(m.s, 0, B, False)
    X = B.copy()
    lib.ma97_solve_d(C.c_int(0), C.c_int(1), X.ctypes.data_as(dp), C.c_int(dim), *m.keeps())
    lib.ma97_alter_d(d.ctypes.data_as(dp), *m.keeps())
    assert m.flag() == 0
    X2 = B.copy()
    lib.ma97_solve_d(C.c_int(0), C.c_int(1), X2.ctypes.data_as(dp), C.c_int(dim), *m.keeps())
    assert_bits(X2, X, "alter round trip")
    assert_bits(X, x0, "shim = C ABI")
    d2 = np.zeros((dim, 2))
    lib.ma97_enquire_indef_d(C.byref(m.akeep), C.byref(m.fkeep), m.ctrl, m.info, None, d2.ctypes.data_as(dp))
    assert_bits(d2, d, "enquire after alter")
    bad = d.copy()
    bad[0, 0] = np.nan
    lib.ma97_alter_d(bad.ctypes.data_as(dp), *m.keeps())
    assert m.flag() < 0
    # enquire_posdef is refused on an indefinite KKT matrix
    out = np.full(dim, 5.0)
    lib.ma97_enquire_posdef_d(*m.keeps(), out.ctypes.data_as(dp))
    assert m.flag() < 0 and np.all(out == 5.0)
    m.close()


@pytest.mark.gpu
def test_ma97_shim_enquire_posdef(built_lib):
    """SPD (shifted 2-D Laplacian with a random diagonal): d = sqrt(D) = the diagonal of numpy's Cholesky factor of the
    permuted, scaled matrix"""
    import scipy.sparse as sp
    g = 20
    T = sp.diags([-np.ones(g - 1), 2.0 * np.ones(g), -np.ones(g - 1)], [-1, 0, 1])
    A = (sp.kron(sp.eye(g), T) + sp.kron(T, sp.eye(g))).tocsr()
    A = A + sp.diags(np.random.default_rng(0).uniform(0.1, 10.0, g * g))
    C_ = sp.tril(A).tocoo()
    dim = g * g
    m = Ma97(built_lib, dim, (C_.row + 1).astype(np.int32), (C_.col + 1).astype(np.int32), C_.data)
    assert m.flag() == 0
    d = np.zeros(dim)
    m.lib.ma97_enquire_posdef_d(*m.keeps(), d.ctypes.data_as(m.dp))
    assert m.flag() == 0
    var, ty, dinv2 = m.s.enquire_indef()
    assert np.all(ty == 1)
    Ad = A.toarray()
    SAS = (m.scale[:, None] * Ad * m.scale[None, :])[np.ix_(var, var)]
    ref = np.diag(np.linalg.cholesky(SAS))
    assert np.abs(d - ref).max() <= 1e-12 * ref.max(), np.abs(d - ref).max()
    m.close()
