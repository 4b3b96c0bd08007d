"""Partial solves (b200ldlt_solve_partial / _device, jobs 1-4: L, D, L^T on their own) and factor inspection
(b200ldlt_enquire_indef, device_ptr "scale"), through the C ABI and the HSL_MA97 shim.

S A S = P L D L^T P^T; intermediate vectors are in pivot order.  job 1: L^-1 P^T S b, job 2: D^-1 b, job 3: S P L^-T b,
job 4: S P L^-T D^-1 b.  Job 3 . 2 . 1 and job 4 . 1 must reproduce the full solve bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt, random_kkt, to_scipy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
NEW_SYMBOLS = ["b200ldlt_solve_partial", "b200ldlt_solve_partial_device", "b200ldlt_enquire_indef",
               "ma97_enquire_indef_d"]


def golden_system(case):
    z = np.load(os.path.join(G, case + "_kkt.npz"))
    k = min(int(f[4:]) for f in z.files if f.startswith("val_"))
    return int(z["dim"]), z["irn"], z["jcn"], z["val_%d" % k]


SYSTEMS = {
    "hs071_0": lambda: golden_system("hs071_0"),
    "MBndryCntrl1_30": lambda: golden_system("MBndryCntrl1_30"),
    "MDistCntrl3a_25": lambda: golden_system("MDistCntrl3a_25"),
    "LukVlE1_1000": lambda: golden_system("LukVlE1_1000"),
    "random": lambda: random_kkt(400, 150, density=0.02, seed=8)[:4],
    "mbndry30_wzero": lambda: mbndry_kkt(30, w_zero=True)[:4],
}
LARGE = lambda: mbndry_kkt(400)[:4]   # noqa: E731


def factored(dim, irn, jcn, val, **opts):
    s = B200Ldlt(**opts)
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    st, _ = s.factor(False, 0)
    assert st == SYMSOLVER_SUCCESS, s.last_error()
    return s


def device_doubles(ptr, n):
    """n doubles at a device address of the library, copied to the host"""
    import torch

    class Cai:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (int(ptr), False), "strides": None,
                                   "version": 2}

    return torch.as_tensor(Cai(), device="cuda").cpu().numpy().copy()


def run(s, job, B, device):
    """job on the columns of B (nrhs x dim, row c = column c), host or device entry point"""
    nrhs, dim = B.shape
    if device:
        import torch
        X = torch.tensor(B.ravel(), dtype=torch.float64, device="cuda")
        assert s.solve_partial_device(job, X.data_ptr(), nrhs) == SYMSOLVER_SUCCESS, s.last_error()
        return X.cpu().numpy().reshape(nrhs, dim)
    X = B.ravel().copy()
    assert s.solve_partial(job, X, nrhs) == SYMSOLVER_SUCCESS, s.last_error()
    return X.reshape(nrhs, dim)


def assert_bits(a, b, tag=""):
    diff = np.flatnonzero(np.asarray(a).ravel().view(np.uint64) != np.asarray(b).ravel().view(np.uint64))
    assert diff.size == 0, (tag, diff.size, diff[:5])


def check_compose(s, B, device):
    x0 = B.copy()
    if device:
        x0 = run(s, 0, B, True)
    else:
        x0 = B.ravel().copy()
        assert s.solve(x0, B.shape[0]) == SYMSOLVER_SUCCESS
        x0 = x0.reshape(B.shape)
    y = run(s, 1, B, device)
    assert_bits(run(s, 3, run(s, 2, y, device), device), x0, "3.2.1")
    assert_bits(run(s, 4, y, device), x0, "4.1")


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


# ---- 1. bit-identity with the full solve ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("env", [
    {}, {"B200_SOLVE_DIRECT": "0"}, {"B200_SOLVE_DIRECT": "1"}, {"B200_SOLVE_DIRECT": "4"}, {"B200_SOLVE_NOPAIR": "1"},
    {"B200_SOLVE_BLOCK": "2"},
])
@pytest.mark.parametrize("system", sorted(SYSTEMS))
def test_parts_compose_to_solve_bitwise(system, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    s = factored(*SYSTEMS[system]())
    rng = np.random.default_rng(1)
    for nrhs in (1, 3):
        B = rng.standard_normal((nrhs, s.dim))
        check_compose(s, B, device=False)
        check_compose(s, B, device=True)
    s.close()


@pytest.mark.gpu
def test_parts_compose_to_solve_bitwise_large():
    s = factored(*LARGE())
    B = np.random.default_rng(2).standard_normal((2, s.dim))
    check_compose(s, B[:1], device=True)
    check_compose(s, B, device=True)
    check_compose(s, B[:1], device=False)
    s.close()


# ---- 2. adjoints ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(SYSTEMS) + ["mbndry400"])
def test_adjoint_identities(system):
    s = factored(*(LARGE() if system == "mbndry400" else SYSTEMS[system]()))
    rng = np.random.default_rng(3)
    for _ in range(2):
        u, v = rng.standard_normal((1, s.dim)), rng.standard_normal((1, s.dim))
        for ja, jb in ((1, 3), (2, 2)):
            a, b = run(s, ja, u, True)[0], run(s, jb, v, True)[0]
            lhs, rhs = v[0] @ a, b @ u[0]
            assert abs(lhs - rhs) <= 1e-12 * max(np.abs(v[0] * a).sum(), np.abs(b * u[0]).sum()), (ja, jb, lhs, rhs)
    s.close()


# ---- 3. reconstruction of A from the parts -------------------------------------------------------------------------
def d_blocks(ty, dinv2):
    """D (dense, pivot order) from the D^-1 entries of enquire_indef"""
    n = len(ty)
    Dm = np.zeros((n, n))
    p = 0
    while p < n:
        if ty[p] == 1:
            Dm[p, p] = 1.0 / dinv2[p, 0]
            p += 1
        else:
            assert ty[p] == 2 and ty[p + 1] == 3
            Bi = np.array([[dinv2[p, 0], dinv2[p, 1]], [dinv2[p, 1], dinv2[p + 1, 0]]])
            Dm[p:p + 2, p:p + 2] = np.linalg.inv(Bi)
            p += 2
    return Dm


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
    M = run(s, 1, np.eye(dim), False).T          # column j = job 1 (e_j): M = L^-1 P^T S
    Lh = np.linalg.inv(M)                        # = S^-1 P L
    var, ty, dinv2 = s.enquire_indef()
    Dm = d_blocks(ty, dinv2)
    err = np.abs(Lh @ Dm @ Lh.T - A).max() / np.abs(A).max()
    assert err <= 1e-12, err
    scale = device_doubles(s.device_ptr("scale"), dim)
    assert np.all(scale > 0) and np.all(np.frexp(scale)[0] == 0.5)    # powers of two
    T = (scale[:, None] * Lh)[var]               # = L, rows in pivot order
    assert np.abs(np.diag(T) - 1.0).max() <= 1e-12
    assert np.abs(np.triu(T, 1)).max() <= 1e-12
    s.close()


# ---- 4. D, inertia, pivot order ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(SYSTEMS))
def test_d_and_inertia(system):
    s = factored(*SYSTEMS[system]())
    n = s.dim
    var, ty, dinv2 = s.enquire_indef()
    assert np.array_equal(np.sort(var), np.arange(n))
    info = s.info()
    assert int((ty == 2).sum()) == int((ty == 3).sum()) == info["num_2x2"]
    assert np.all(ty[np.flatnonzero(ty == 2) + 1] == 3)
    assert np.all(dinv2[ty != 2, 1] == 0.0)
    neg, p = 0, 0
    while p < n:
        if ty[p] == 1:
            neg += dinv2[p, 0] < 0
            p += 1
        else:
            Bi = np.array([[dinv2[p, 0], dinv2[p, 1]], [dinv2[p, 1], dinv2[p + 1, 0]]])
            neg += int((np.linalg.eigvalsh(Bi) < 0).sum())
            p += 2
    assert neg == info["num_neg"] == s.NumberOfNegEVals()
    # job 2 on unit vectors returns exactly those entries
    cols = np.arange(n) if n <= 2000 else np.random.default_rng(0).choice(n, 1500, replace=False)
    E = np.zeros((len(cols), n))
    E[np.arange(len(cols)), cols] = 1.0
    Y = run(s, 2, E, True)
    for r, p in enumerate(cols):
        exp = np.zeros(n)
        exp[p] = dinv2[p, 0]
        if ty[p] == 2:
            exp[p + 1] = dinv2[p, 1]
        elif ty[p] == 3:
            exp[p - 1] = dinv2[p - 1, 1]
        assert np.array_equal(Y[r], exp), p   # exact (0 * a negative entry is -0.0, hence values, not bits)
    s.close()


# ---- 5. blocked columns and launch counts --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random", "mbndry30_wzero"])
def test_blocked_partial_bit_identical_to_columns(system):
    s = factored(*SYSTEMS[system]())
    for nrhs in range(2, 14):
        B = np.random.default_rng(nrhs).standard_normal((nrhs, s.dim))
        for job in (1, 2, 3, 4):
            for device in (False, True):
                X = run(s, job, B, device)
                for c in range(nrhs):
                    assert_bits(X[c], run(s, job, B[c:c + 1], device)[0], (nrhs, job, device, c))
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1", "3"])
def test_launch_counts(block, monkeypatch):
    """per block: job 0: 8, job 1, 3, 4: 5, job 2: 1 (default B200_SOLVE_DIRECT=2)"""
    if block is not None:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*mbndry_kkt(70, sigma_spread=3.0, seed=5)[:4])
    width = 8 if block is None else int(block)
    for nrhs in (1, 8):
        nblk = -(-nrhs // width)
        B = np.random.default_rng(nrhs).standard_normal((nrhs, s.dim))
        for job, per in ((0, 8), (1, 5), (2, 1), (3, 5), (4, 5)):
            for device in (False, True):
                run(s, job, B, device)
                info = s.info()
                assert info["launches_solve"] == per * nblk, (job, nrhs, device, info["launches_solve"])
                assert info["ms_solve_gpu"] > 0.0
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("direct", ["0", "1", "4"])
def test_launch_counts_follow_direct_levels(direct, monkeypatch):
    monkeypatch.setenv("B200_SOLVE_DIRECT", direct)
    s = factored(*mbndry_kkt(70, sigma_spread=3.0, seed=5)[:4])
    B = np.random.default_rng(0).standard_normal((1, s.dim))
    counts = {}
    for job in range(5):
        run(s, job, B, True)
        counts[job] = s.info()["launches_solve"]
    assert counts[2] == 1
    assert counts[1] == counts[3] == counts[4] and 2 * counts[1] - 2 == counts[0], counts
    s.close()


# ---- 6. handle state and refusals ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_state_interleaved_refactor_reanalysis_pivtol():
    dim, irn, jcn, val, nc = mbndry_kkt(40, sigma_spread=3.0, seed=3)
    s = factored(dim, irn, jcn, val)
    L = s._L
    L.b200ldlt_set_pivtol.argtypes = [C.c_void_p, C.c_double, C.c_double]

    def check(tag):
        for rep in range(2):
            for nrhs in (1, 5):
                B = np.random.default_rng(10 * rep + nrhs).standard_normal((nrhs, s.dim))
                check_compose(s, B, device=bool(rep))
                x = B[0].copy()
                assert s.solve(x, 1) == SYMSOLVER_SUCCESS, tag

    check("first")
    v2 = val.copy()
    v2[: len(v2) // 3] *= 1.25
    s.GetValuesArrayPtr()[:] = v2
    assert s.factor(True, nc) == (SYMSOLVER_SUCCESS, nc)
    check("new values")
    assert s.IncreaseQuality()
    assert s.refactor(True, nc) == (SYMSOLVER_SUCCESS, nc)
    check("increase_quality")
    assert L.b200ldlt_set_pivtol(s._h, 1e-6, 1e-4) == SYMSOLVER_SUCCESS
    assert s.refactor(True, nc) == (SYMSOLVER_SUCCESS, nc)
    check("set_pivtol")
    s.close()


@pytest.mark.gpu
def test_state_after_reanalysis_by_increase_quality():
    """lifted pivots make increase_quality schedule a re-analysis: the parts still compose to the solve afterwards"""
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    s = factored(n, irn, jcn, val)
    assert s.info()["num_forced"] > 0
    B = np.random.default_rng(4).standard_normal((3, n))
    check_compose(s, B, device=False)
    assert s.IncreaseQuality()
    assert s.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    check_compose(s, B, device=True)
    check_compose(s, B[:1], device=False)
    s.close()


@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    x = np.ones(dim)
    assert s.solve_partial(1, x) == SYMSOLVER_FATAL_ERROR and "no factors" in s.last_error()
    with pytest.raises(RuntimeError, match="no factors"):
        s.enquire_indef()
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    for job in (-1, 5):
        assert s.solve_partial(job, x) == SYMSOLVER_FATAL_ERROR and "job" in s.last_error()
        assert s.solve_partial_device(job, 0) == SYMSOLVER_FATAL_ERROR
    assert s.solve_partial(1, x) == SYMSOLVER_SUCCESS
    # a zero row: SINGULAR leaves no factors
    v0 = val.copy()
    r = int(irn[0])
    v0[(irn == r) | (jcn == r)] = 0.0
    s.GetValuesArrayPtr()[:] = v0
    assert s.factor(False, 0)[0] == SYMSOLVER_SINGULAR
    assert s.solve_partial(2, x) == SYMSOLVER_FATAL_ERROR and "no factors" in s.last_error()
    with pytest.raises(RuntimeError, match="no factors"):
        s.enquire_indef()
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    L = s._L
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    for job in (1, 2, 3, 4):
        assert s.solve_partial(job, x) == SYMSOLVER_FATAL_ERROR and "sharded" in s.last_error()
    s.close()


# ---- 7. the HSL_MA97 shim --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["hs071_0", "MBndryCntrl1_30", "mbndry30_wzero"])
def test_ma97_shim_partial_solves_and_enquire(system, built_lib):
    dim, irn, jcn, val = SYSTEMS[system]()
    A = to_scipy(dim, irn, jcn, val)
    Lo = __import__("scipy.sparse", fromlist=["tril"]).tril(A).tocsc()
    Lo.sort_indices()
    ptr, row, cv = Lo.indptr.astype(np.int32), Lo.indices.astype(np.int32), Lo.data.astype(np.float64)
    # the C ABI handle on exactly the triplets the shim builds (CSC order): the same analysis, the same bits
    cols = np.repeat(np.arange(dim), np.diff(ptr)).astype(np.int32)
    s = factored(dim, row + 1, cols + 1, cv, pivtol=0.01, pivtolmax=0.01)   # the shim's handle: control.u = 0.01
    lib = C.CDLL(built_lib)
    vp = C.c_void_p
    ctrl, info = C.create_string_buffer(1024), C.create_string_buffer(1024)
    flag = lambda: C.cast(info, C.POINTER(C.c_int))[0]   # noqa: E731
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    ptr_p, row_p, cv_p = ptr.ctypes.data_as(ip), row.ctypes.data_as(ip), cv.ctypes.data_as(dp)
    lib.ma97_default_control_d(ctrl)
    akeep, fkeep = vp(), vp()
    lib.ma97_analyse_d(C.c_int(0), C.c_int(dim), ptr_p, row_p, cv_p, C.byref(akeep), ctrl, info, None)
    assert flag() == 0
    scale = np.zeros(dim)
    lib.ma97_factor_d(C.c_int(4), ptr_p, row_p, cv_p, C.byref(akeep), C.byref(fkeep), ctrl, info, scale.ctypes.data_as(dp))
    assert flag() == 0
    assert_bits(scale, device_doubles(s.device_ptr("scale"), dim), "scale")
    assert np.all(scale > 0)
    rng = np.random.default_rng(5)
    for job in range(5):
        for nrhs, ldx in ((1, dim), (3, dim), (3, dim + 7)):
            B = rng.standard_normal((nrhs, dim))
            X = np.zeros((nrhs, ldx))
            X[:, :dim] = B
            X[:, dim:] = 42.0
            lib.ma97_solve_d(C.c_int(job), C.c_int(nrhs), X.ctypes.data_as(dp), C.c_int(ldx), C.byref(akeep),
                             C.byref(fkeep), ctrl, info)
            assert flag() == 0, (job, nrhs, ldx)
            assert_bits(X[:, :dim], run(s, job, B, False), (job, nrhs, ldx))
            assert np.all(X[:, dim:] == 42.0)
    var, ty, dinv2 = s.enquire_indef()
    piv = np.zeros(dim, np.int32)
    d = np.zeros((dim, 2))
    lib.ma97_enquire_indef_d(C.byref(akeep), C.byref(fkeep), ctrl, info, piv.ctypes.data_as(ip), d.ctypes.data_as(dp))
    assert flag() == 0
    pos = np.arange(1, dim + 1)
    exp = np.zeros(dim, np.int64)
    exp[var] = np.where(ty == 1, pos, -pos)
    assert np.array_equal(piv, exp)
    assert_bits(d, dinv2, "d")
    piv2, d2 = np.zeros(dim, np.int32), np.zeros((dim, 2))
    lib.ma97_enquire_indef_d(C.byref(akeep), C.byref(fkeep), ctrl, info, None, d2.ctypes.data_as(dp))
    assert flag() == 0
    assert_bits(d2, dinv2, "d only")
    lib.ma97_enquire_indef_d(C.byref(akeep), C.byref(fkeep), ctrl, info, piv2.ctypes.data_as(ip), None)
    assert flag() == 0 and np.array_equal(piv2, exp)
    lib.ma97_finalise_d(C.byref(akeep), C.byref(fkeep))
    s.close()
