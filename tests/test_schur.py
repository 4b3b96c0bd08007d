"""Partial factorisation with an explicit Schur complement (b200ldlt_set_schur, b200ldlt_schur_complement / _reduce /
_expand).  S = vars, E = the rest:  S_c = A_SS - A_SE A_EE^-1 A_ES,  reduce: y = b_S - A_SE A_EE^-1 b_E,  expand: x_S = xs,
x_E = A_EE^-1 (b_E - A_ES xs).

CPU: the analysis with a Schur set (S last, in the caller's order, one root supernode with no rows) and a numpy
emulation of the partial factorisation driven by the exported maps.  GPU: S_c, the inertia, reduce / expand and the
contracts of the calls against numpy / scipy."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SymbolicAnalysis, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt, random_kkt, to_scipy

from test_symbolic import _check_structure

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def schur_sets(dim, nc, seed):
    """Schur sets of primal variables, constraint rows and a mix, of m = 1, a few and n/3"""
    rng = np.random.default_rng(seed)
    nx = dim - nc
    prim = lambda m: rng.choice(nx, m, replace=False)               # noqa: E731
    cons = lambda m: nx + rng.choice(nc, min(m, nc), replace=False)  # noqa: E731
    out = [prim(1), cons(1), prim(5), cons(4)]
    third = dim // 3
    out.append(rng.permutation(np.concatenate([prim(third - third // 3), cons(third // 3)])))
    return [np.asarray(v, dtype=np.int64) for v in out]


def emulate_schur(S, dim, irn, jcn, val, m):
    """The partial factorisation in numpy, from the exported maps only: every supernode but the last one assembled and
    eliminated without pivoting (quasi-definite systems), then the last one (S) assembled and returned unfactored,
    position t = the t-th Schur variable (lower triangle mirrored)."""
    perm = S.get("perm")
    sn_start, rows_ptr, rel = S.get("sn_start"), S.get("rows_ptr"), S.get("rel")
    parent, uent_ptr, u_dst64, t2u = S.get("sn_parent"), S.get("uent_ptr"), S.get("u_dst64"), S.get("t2u")
    nsn = len(sn_start) - 1
    uval = np.zeros(len(u_dst64))
    np.add.at(uval, t2u, val)
    cbs = [None] * nsn
    children = [[] for _ in range(nsn)]
    for s in range(nsn):
        if parent[s] >= 0:
            children[parent[s]].append(s)
    for s in range(nsn):
        k = sn_start[s + 1] - sn_start[s]
        r = rows_ptr[s + 1] - rows_ptr[s]
        f = k + r
        P = np.zeros(f * k)
        P[u_dst64[uent_ptr[s]:uent_ptr[s + 1]]] = uval[uent_ptr[s]:uent_ptr[s + 1]]
        F = np.zeros((f, f))
        F[:, :k] = P.reshape((k, f)).T
        F = np.tril(F) + np.tril(F, -1).T
        for c in children[s]:
            rl = rel[rows_ptr[c]:rows_ptr[c + 1]]
            F[np.ix_(rl, rl)] += cbs[c]
        if s == nsn - 1:
            assert k == m and r == 0
            return F
        for j in range(k):
            lj = F[j + 1:, j] / F[j, j]
            F[j + 1:, j + 1:] -= np.outer(lj, F[j + 1:, j])
        cbs[s] = F[k:, k:].copy()
    raise AssertionError("no supernodes")


def dense_schur(A, vars):
    e = np.setdiff1d(np.arange(A.shape[0]), vars)
    Ass, Ase, Aee = A[np.ix_(vars, vars)], A[np.ix_(vars, e)], A[np.ix_(e, e)]
    return Ass - Ase @ np.linalg.solve(Aee, Ase.T), e


CPU_SYSTEMS = {
    "random": lambda: random_kkt(150, 60, density=0.05, seed=5, delta_c=1e-2),
    "mbndry6": lambda: mbndry_kkt(6, sigma_spread=1.0, delta_c=1e-2, seed=3),
    "mbndry17": lambda: mbndry_kkt(17, sigma_spread=1.0, delta_c=1e-2, seed=3),
    "dense": lambda: random_kkt(30, 12, density=0.2, seed=2, delta_c=1e-2),   # n <= 48: the single-front case
}


# ---- CPU: the analysis ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("system", sorted(CPU_SYSTEMS))
def test_schur_analysis_structure(built_lib, system):
    dim, irn, jcn, val, nc = CPU_SYSTEMS[system]()
    val0 = val.copy()
    val0[-nc:] = 0.0   # a zero (2,2) block: the pairing is active
    nx = dim - nc
    for vars in schur_sets(dim, nc, seed=dim):
        m = len(vars)
        S = SymbolicAnalysis(dim, irn, jcn, val0, schur=vars)
        _check_structure(S, dim)
        perm, sn_start, rows_ptr, parent = S.get("perm"), S.get("sn_start"), S.get("rows_ptr"), S.get("sn_parent")
        nsn = len(sn_start) - 1
        assert np.array_equal(perm[dim - m:], vars)                      # S last, in the caller's order
        assert sn_start[nsn - 1] == dim - m and rows_ptr[nsn] == rows_ptr[nsn - 1] and parent[nsn - 1] == -1
        # every pair (primal at p, its saddle row at p + 1, same supernode) lies in E: count the candidate positions
        sn_of = np.searchsorted(sn_start, np.arange(dim), side="right") - 1
        cand = [p for p in range(1, dim - m) if perm[p] >= nx and perm[p - 1] < nx and sn_of[p] == sn_of[p - 1]]
        assert S.stats()["n_pairs"] <= len(cand)
        # E supernodes below S have S as their parent exactly when a column of theirs has an S row
        for s in range(nsn - 1):
            rw = S.get("rows")[rows_ptr[s]:rows_ptr[s + 1]]
            if parent[s] == nsn - 1:
                assert len(rw) and rw[0] >= dim - m


@pytest.mark.parametrize("system", sorted(CPU_SYSTEMS))
def test_schur_analysis_empty_set_is_the_plain_analysis(built_lib, system):
    dim, irn, jcn, val, nc = CPU_SYSTEMS[system]()
    a, b = SymbolicAnalysis(dim, irn, jcn, val), SymbolicAnalysis(dim, irn, jcn, val, schur=[])
    for name in ("perm", "sn_start", "sn_parent", "rows_ptr", "rows", "rel", "L_off", "cb_off", "u_dst64", "uent_ptr",
                 "t2u", "sn_level", "level_ptr", "level_sn", "child_ptr", "child_idx"):
        assert np.array_equal(a.get(name), b.get(name)), name


def test_schur_analysis_refusals(built_lib):
    dim, irn, jcn, val, nc = CPU_SYSTEMS["mbndry6"]()
    for bad in ([dim], [-1], [3, 3], list(range(dim))):
        with pytest.raises(RuntimeError):
            SymbolicAnalysis(dim, irn, jcn, val, schur=bad)


@pytest.mark.parametrize("system", sorted(CPU_SYSTEMS))
def test_schur_emulation_matches_numpy(built_lib, system):
    dim, irn, jcn, val, nc = CPU_SYSTEMS[system]()
    val0 = val.copy()
    val0[-nc:] = 0.0
    A = to_scipy(dim, irn, jcn, val).toarray()
    for vars in schur_sets(dim, nc, seed=dim + 1):
        S = SymbolicAnalysis(dim, irn, jcn, val0, schur=vars)
        F = emulate_schur(S, dim, irn, jcn, val, len(vars))
        F = np.tril(F) + np.tril(F, -1).T
        ref, _ = dense_schur(A, vars)
        scale = max(np.abs(A[np.ix_(vars, vars)]).max(), np.abs(A[np.ix_(vars, vars)] - ref).max())
        assert np.abs(F - ref).max() <= 1e-12 * scale, (system, len(vars))


# ---- GPU --------------------------------------------------------------------------------------------------------------
def golden_system(case):
    z = np.load(os.path.join(ROOT, "tests", "golden", case + "_kkt.npz"))
    k = min(int(f[4:]) for f in z.files if f.startswith("val_"))
    return int(z["dim"]), z["irn"], z["jcn"], z["val_%d" % k]


GPU_SYSTEMS = {
    "hs071_0": lambda: golden_system("hs071_0"),
    "MBndryCntrl1_30": lambda: golden_system("MBndryCntrl1_30"),
    "MDistCntrl3a_25": lambda: golden_system("MDistCntrl3a_25"),
    "LukVlE1_1000": lambda: golden_system("LukVlE1_1000"),
    "random": lambda: random_kkt(400, 150, density=0.02, seed=8)[:4],
    "mbndry30_wzero": lambda: mbndry_kkt(30, w_zero=True)[:4],
    "random_300_100": lambda: random_kkt(300, 100, seed=3)[:4],
}
M_CLASSES = (1, 20, 64, 150, 300)   # the root in each solve class: <= 32, 33..96, 97..256, > 256

# B200_SCHUR_MEASURED=<file>: the discrepancies of every case are appended there (one JSON line each).  The tolerances
# rest on the largest measured on an H100 80GB HBM3 (700 W); the cases with A_EE of condition up to 1e10 set them, the
# well-conditioned ones stay near 1e-15:
#   S_c and y, relative to max(|A_SS|, |A_SE A_EE^-1 A_ES|) / max|y|: 3.7e-11 (100x);
#   16 columns of S_c at N = 400 against scipy, relative to max(|column|, 1): 1.6e-10 (25x) -> TOL_SC  = 4e-9
#   round-trip residual ||A x - b|| / (||A|| ||x|| + ||b||) (S_c solved by numpy): 1.2e-10 -> TOL_RES = 1e-8
#   x_E from the exact x_S against numpy's full solve, relative to max|x|: 4.9e-10     -> TOL_XE  = 5e-8
# The residual and x_E include the conditioning of S_c and A, which the reduce / expand calls do not control.
MEASURED = os.environ.get("B200_SCHUR_MEASURED")
TOL_SC = 4e-9
TOL_RES = 1e-8
TOL_XE = 5e-8


def record(**kw):
    if MEASURED:
        with open(MEASURED, "a") as f:
            f.write(json.dumps(kw) + "\n")


_DENSE = {}


def dense(system):
    if system not in _DENSE:
        dim, irn, jcn, val = GPU_SYSTEMS[system]()
        _DENSE[system] = (dim, irn, jcn, val, to_scipy(dim, irn, jcn, val).toarray())
    return _DENSE[system]


def pick_vars(A, m, seed):
    """m seeded Schur variables with a well-conditioned A_EE: the first of a few seeded draws from all variables that
    keeps cond(A_EE) < 1e10 (a KKT system loses it when S takes the primal neighbours of a constraint row left in E);
    else constraint rows (the zero-diagonal rows) first, then primal variables, in a seeded order"""
    dim = A.shape[0]
    ok = lambda v: np.linalg.cond(A[np.ix_(*(2 * [np.setdiff1d(np.arange(dim), v)]))]) < 1e10   # noqa: E731
    for t in range(8):
        vars = np.random.default_rng(seed + 1000 * t).choice(dim, m, replace=False)
        if ok(vars):
            return vars
    rng = np.random.default_rng(seed)
    zero = np.flatnonzero(np.abs(np.diag(A)) <= 1e-7 * np.abs(A).max(axis=1))
    rest = np.setdiff1d(np.arange(dim), zero)
    vars = np.concatenate([rng.permutation(zero), rng.permutation(rest)])[:m]
    assert ok(vars), "no well-conditioned A_EE found"
    return rng.permutation(vars)


def schur_handle(dim, irn, jcn, val, vars, **opts):
    s = B200Ldlt(**opts)
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    assert s.set_schur(vars) == SYMSOLVER_SUCCESS, s.last_error()
    st, neg = s.factor(False, 0)
    assert st == SYMSOLVER_SUCCESS, s.last_error()
    return s, neg


def cases():
    out = []
    for system in GPU_SYSTEMS:
        for m in M_CLASSES:
            out.append((system, m))
    return out


def rel_err(a, b, scale):
    return float(np.abs(a - b).max() / scale)


@pytest.mark.gpu
@pytest.mark.parametrize("system,m", cases())
def test_schur_complement_inertia_and_round_trip(system, m):
    dim, irn, jcn, val, A = dense(system)
    if m >= dim:
        pytest.skip("m >= n")
    vars = pick_vars(A, m, seed=m)
    s, neg = schur_handle(dim, irn, jcn, val, vars)
    info = s.info()
    assert info["num_forced"] == 0
    sc = s.schur_complement()
    assert np.array_equal(sc.view(np.uint64), sc.T.view(np.uint64))          # bit-symmetric
    ref, e = dense_schur(A, vars)
    Ass = A[np.ix_(vars, vars)]
    scale = max(np.abs(Ass).max(), np.abs(Ass - ref).max())
    err_sc = rel_err(sc, ref, scale)
    # inertia: A_EE from the factorisation, A = A_EE + S_c (Haynsworth)
    neg_ee = int((np.linalg.eigvalsh(A[np.ix_(e, e)]) < 0).sum())
    neg_sc = int((np.linalg.eigvalsh(sc) < 0).sum())
    neg_a = int((np.linalg.eigvalsh(A) < 0).sum())
    # round trip: reduce, dense solve with S_c, expand
    rng = np.random.default_rng(7)
    worst_res, worst_y, worst_xe = 0.0, 0.0, 0.0
    for nrhs in (1, 11):
        B = rng.standard_normal((dim, nrhs))
        Y = s.schur_reduce(B)
        Yr = B[vars] - A[np.ix_(vars, e)] @ np.linalg.solve(A[np.ix_(e, e)], B[e])
        worst_y = max(worst_y, rel_err(Y, Yr, max(np.abs(Yr).max(), 1.0)))
        XS = np.linalg.solve(sc, Y)
        X = s.schur_expand(B, XS)
        assert np.array_equal(X[vars], XS)
        R = A @ X - B
        res = np.abs(R).max(axis=0) / (np.abs(A).sum(axis=1).max() * np.abs(X).max(axis=0) + np.abs(B).max(axis=0))
        worst_res = max(worst_res, float(res.max()))
        # the exact x_S of a full solve reproduces x_E
        Xf = np.linalg.solve(A, B)
        Xe = s.schur_expand(B, Xf[vars])
        worst_xe = max(worst_xe, rel_err(Xe, Xf, np.abs(Xf).max()))
    record(test="schur", system=system, m=int(m), err_sc=err_sc, err_y=worst_y, res=worst_res, err_xe=worst_xe)
    assert neg == info["num_neg"] == neg_ee
    assert neg + neg_sc == neg_a
    assert err_sc <= TOL_SC, err_sc
    assert worst_y <= TOL_SC, worst_y
    assert worst_res <= TOL_RES, worst_res
    assert worst_xe <= TOL_XE, worst_xe
    s.close()


def device_run(fn, *arrays):
    import torch
    ts = [torch.tensor(np.asfortranarray(a).ravel(order="F"), dtype=torch.float64, device="cuda") for a in arrays]
    st = fn(*[t.data_ptr() for t in ts])
    return st, [t.cpu().numpy() for t in ts]


def full_size_handle(dim, irn, jcn, val, nc, **opts):
    """300 seeded Schur variables, 200 constraint rows and 100 primal variables: the first of a few seeded draws whose
    A_EE factorises without lifted pivots (pivots are not delayed into S, so a constraint row of E that loses its best
    primal partners to S can need one); else 300 constraint rows, which leave every primal variable in E"""
    nx = dim - nc
    s = B200Ldlt(**opts)
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    draws = [np.random.default_rng(400 + t) for t in range(4)]
    sets = [r.permutation(np.concatenate([nx + r.choice(nc, 200, replace=False), r.choice(nx, 100, replace=False)]))
            for r in draws] + [nx + np.random.default_rng(400).choice(nc, 300, replace=False)]
    for vars in sets:
        assert s.set_schur(vars) == SYMSOLVER_SUCCESS, s.last_error()
        assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS, s.last_error()
        if s.info()["num_forced"] == 0:
            record(test="full_size_set", constraint_rows=int((vars >= nx).sum()))
            return s, vars
    raise AssertionError("every Schur set needed lifted pivots")


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph,one_stream", [(0, False), (1, False), (1, True)])
def test_schur_full_size(use_graph, one_stream, monkeypatch):
    import scipy.sparse.linalg as sla
    if one_stream:
        monkeypatch.setenv("B200_ONE_STREAM", "1")
    dim, irn, jcn, val, nc = mbndry_kkt(400)
    s, vars = full_size_handle(dim, irn, jcn, val, nc, use_graph=use_graph)
    rng = np.random.default_rng(400)
    sc = s.schur_complement()
    A = to_scipy(dim, irn, jcn, val).tocsc()
    e = np.setdiff1d(np.arange(dim), vars)
    lu = sla.splu(A[e][:, e].tocsc())
    Ase = A[vars][:, e]
    cols = rng.choice(len(vars), 16, replace=False)
    worst = 0.0
    for j in cols:
        ej = np.zeros(len(vars))
        ej[j] = 1.0
        ref = A[vars][:, vars] @ ej - Ase @ lu.solve(np.asarray(A[e][:, vars] @ ej).ravel())
        worst = max(worst, float(np.abs(sc[:, j] - ref).max() / max(np.abs(ref).max(), 1.0)))
    B = rng.standard_normal((dim, 3))
    Y = s.schur_reduce(B)
    X = s.schur_expand(B, np.linalg.solve(sc, Y))
    res = float((np.abs(A @ X - B).max(axis=0) / (abs(A).sum(axis=1).max() * np.abs(X).max(axis=0) + np.abs(B).max(axis=0))).max())
    record(test="full_size", use_graph=use_graph, one_stream=one_stream, err_sc=worst, res=res,
           ms_factor=s.info()["ms_factor_gpu"], launches=s.info()["launches_factor"])
    assert worst <= TOL_SC, worst
    assert res <= TOL_RES, res
    s.close()


@pytest.mark.gpu
def test_schur_reproducible_host_device_blocked():
    dim, irn, jcn, val, A = dense("MBndryCntrl1_30")
    vars = pick_vars(A, 150, seed=3)
    s, _ = schur_handle(dim, irn, jcn, val, vars)
    sc1 = s.schur_complement()
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    sc2 = s.schur_complement()
    assert np.array_equal(sc1.view(np.uint64), sc2.view(np.uint64))
    st, (dsc,) = device_run(s.schur_complement_device, np.zeros((150, 150)))
    assert st == SYMSOLVER_SUCCESS
    assert np.array_equal(dsc.view(np.uint64), sc1.ravel(order="F").view(np.uint64))
    rng = np.random.default_rng(1)
    B = rng.standard_normal((dim, 13))
    XS = rng.standard_normal((150, 13))
    Y = s.schur_reduce(B)
    launches_block = s.info()["launches_solve"]
    X = s.schur_expand(B, XS)
    for c in (0, 5, 12):
        assert np.array_equal(s.schur_reduce(B[:, c]).view(np.uint64), Y[:, c].view(np.uint64))
        assert np.array_equal(s.schur_expand(B[:, c], XS[:, c]).view(np.uint64), X[:, c].view(np.uint64))
    assert s.info()["launches_solve"] == 9   # expand of one column: 5 + 2 D with D = 2
    s.schur_reduce(B[:, 0])
    assert s.info()["launches_solve"] == 5   # reduce: 3 + D
    assert launches_block == 2 * 5           # 13 columns: blocks of 8 and 5
    st, (_, dy) = device_run(lambda b, y: s.schur_reduce_device(b, y, 13), B, np.zeros((150, 13)))
    assert st == SYMSOLVER_SUCCESS and np.array_equal(dy.view(np.uint64), Y.ravel(order="F").view(np.uint64))
    st, (_, _, dx) = device_run(lambda b, xs, x: s.schur_expand_device(b, xs, x, 13), B, XS, np.zeros((dim, 13)))
    assert st == SYMSOLVER_SUCCESS and np.array_equal(dx.view(np.uint64), X.ravel(order="F").view(np.uint64))
    s.close()


@pytest.mark.gpu
def test_schur_contracts():
    dim, irn, jcn, val, A = dense("MBndryCntrl1_30")
    vars = pick_vars(A, 20, seed=5)
    s = B200Ldlt()
    L = s._L
    ip = lambda a: np.ascontiguousarray(a, dtype=np.int32).ctypes.data_as(C.POINTER(C.c_int))   # noqa: E731
    assert L.b200ldlt_set_schur(s._h, 2, ip([0, 1])) == SYMSOLVER_FATAL_ERROR and "analyse first" in s.last_error()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    for m, v, what in ((-1, [0], "m must be >= 0"), (dim, list(range(dim)), "m must be < n"), (2, None, "NULL vars"),
                       (2, [0, dim], "out of range"), (2, [-1, 0], "out of range"), (3, [4, 5, 4], "repeated")):
        assert L.b200ldlt_set_schur(s._h, m, None if v is None else ip(v)) == SYMSOLVER_FATAL_ERROR
        assert s.last_error().startswith("set_schur: ") and what in s.last_error(), s.last_error()
    # the refusals left the handle ordinary
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    with pytest.raises(RuntimeError, match="not in Schur mode"):
        s.schur_complement()
    assert s.set_schur(vars) == SYMSOLVER_SUCCESS
    with pytest.raises(RuntimeError, match="no factors"):
        s.schur_complement()
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    b = np.ones(dim)
    y = np.full(20, 7.0)
    assert L.b200ldlt_schur_reduce(s._h, -1, b.ctypes.data_as(C.POINTER(C.c_double)),
                                   y.ctypes.data_as(C.POINTER(C.c_double))) == SYMSOLVER_FATAL_ERROR
    assert "nrhs" in s.last_error()
    assert L.b200ldlt_schur_reduce(s._h, 1, None, y.ctypes.data_as(C.POINTER(C.c_double))) == SYMSOLVER_FATAL_ERROR
    assert L.b200ldlt_schur_expand(s._h, 1, b.ctypes.data_as(C.POINTER(C.c_double)), None,
                                   b.ctypes.data_as(C.POINTER(C.c_double))) == SYMSOLVER_FATAL_ERROR
    assert L.b200ldlt_schur_complement(s._h, None) == SYMSOLVER_FATAL_ERROR
    assert np.all(y == 7.0) and np.all(b == 1.0)
    assert L.b200ldlt_schur_reduce(s._h, 0, None, None) == SYMSOLVER_SUCCESS and s.info()["launches_solve"] == 0
    # every other call that reads the factors is refused in Schur mode
    x = np.ones(dim)
    assert s.solve(x) == SYMSOLVER_FATAL_ERROR and s.last_error() == "solve: Schur mode"
    assert s.solve_partial(1, x) == SYMSOLVER_FATAL_ERROR and s.last_error() == "solve_partial: Schur mode"
    for call in (lambda: s.lmultiply(0, x), lambda: s.sparse_fwd_solve([0], [1.0]), lambda: s.solve_fredholm(x, 0.0),
                 lambda: s.selected_inverse(), lambda: s.enquire_indef(), lambda: s.enquire_zero_pivots()):
        with pytest.raises(RuntimeError, match=": Schur mode$"):
            call()
    assert s.alter_d(np.zeros((dim, 2))) == SYMSOLVER_FATAL_ERROR and s.last_error() == "alter_d: Schur mode"
    import torch
    d = torch.ones(dim, dtype=torch.float64, device="cuda")
    assert s.solve_refine_device(d.data_ptr())[0] == SYMSOLVER_FATAL_ERROR
    assert s.last_error() == "solve_refine_device: Schur mode"
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_FATAL_ERROR
    # SINGULAR in Schur mode keeps nothing, whatever the keep mode
    assert s.set_singular_action(1) == SYMSOLVER_SUCCESS
    e = np.setdiff1d(np.arange(dim), vars)
    r = int(e[0]) + 1
    v0 = val.copy()
    v0[(irn == r) | (jcn == r)] = 0.0
    s.GetValuesArrayPtr()[:] = v0
    assert s.factor(False, 0)[0] == SYMSOLVER_SINGULAR
    with pytest.raises(RuntimeError, match="no factors"):
        s.schur_complement()
    assert s.set_singular_action(0) == SYMSOLVER_SUCCESS
    # the set persists through re-analyses (b200ldlt_analyse_now runs the analysis increase_quality schedules)
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    sc1 = s.schur_complement()
    assert s.analyse_now(val) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    assert np.array_equal(s.schur_complement().view(np.uint64), sc1.view(np.uint64))
    # set_schur(0): the handle is a fresh one again, bit for bit
    assert s.set_schur([]) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    f = B200Ldlt()
    assert f.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    f.GetValuesArrayPtr()[:] = val
    assert f.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    assert s.info()["launches_factor"] == f.info()["launches_factor"]
    for a, bb in zip(s.enquire_indef(), f.enquire_indef()):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(bb).view(np.uint8))
    B = np.random.default_rng(2).standard_normal((dim, 3))
    Xs, Xf = B.T.copy(), B.T.copy()
    assert s.solve(Xs.ravel(), 3) == SYMSOLVER_SUCCESS and f.solve(Xf.ravel(), 3) == SYMSOLVER_SUCCESS
    assert s.info()["launches_solve"] == f.info()["launches_solve"]
    assert np.array_equal(Xs.view(np.uint64), Xf.view(np.uint64))
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    with pytest.raises(RuntimeError):
        s.schur_complement()
    f.close()
    s.close()
