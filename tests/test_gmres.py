"""FGMRES preconditioned by the LDL^T factors (b200ldlt_solve_gmres / _device), on the factored matrix or on new values
of its pattern.

The header (include/b200ldlt.h) states every order of operations: the operator product, the fixed-grid dot products and
norms, CGS2, the host's Givens rotations and back substitution, and the update.  The numpy replay below calls the
library's single-column solve for x_0 and each z_j and reproduces every returned bit: x and every struct field."""
import ctypes as C
import math

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SUCCESS
from ipopt_b200.capi import Gmres
from ipopt_b200.kkt import to_scipy

from test_error_analysis import rows_of, warp_sums
from test_partial_solve import SYSTEMS, assert_bits, factored
from test_refine import EPS, block_columns, dd_residual, omegas, replay as refine_replay, rule, tridiag

NEW_SYMBOLS = ["b200ldlt_solve_gmres", "b200ldlt_solve_gmres_device"]
FIELDS = [k for k, _ in Gmres._fields_]
ALL = dict(SYSTEMS, tridiag=tridiag)
LANE = np.arange(32)
NAN = float("nan")


# ---- the header's orders, replayed in float64 numpy / Python floats (every operation rounds once, nothing is fused) ----
def gdot(a, b):
    """<a, b> over the fixed grid: P = min(ceil(n / 256), 264) CTAs of 256 threads, each thread its indices in order,
    a shuffle-xor tree per warp, the 8 warps in order, the CTAs' partials in order"""
    n = len(a)
    P = min(-(-n // 256), 264)
    T = 256 * P
    K = -(-n // T)
    p = np.zeros(K * T)
    p[:n] = a * b
    p = p.reshape(K, T)
    acc = np.zeros(T)
    for k in range(K):
        acc = acc + p[k]
    acc = acc.reshape(P, 8, 32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, :, LANE ^ o]
    w = acc[:, :, 0]
    t = w[:, 0].copy()
    for k in range(1, 8):
        t = t + w[:, k]
    r = 0.0
    for q in range(P):
        r = r + float(t[q])
    return r


def apply_op(rows, z):
    ptr, col, a = rows
    return warp_sums(ptr, a * z[col])


class Cycle:
    """the host side of one cycle: the Givens rotations, the stopping decision and the back substitution"""

    def __init__(self, beta, restart, inner_tol):
        self.beta, self.restart, self.inner_tol = beta, restart, inner_tol
        self.g, self.cs, self.sn, self.R = [beta], [], [], []
        self.m, self.iters = 0, 0
        self.on = math.isfinite(beta) and beta != 0.0

    def step(self, h, j):
        self.iters += 1
        h = list(h)
        for i in range(j):
            t = self.cs[i] * h[i] + self.sn[i] * h[i + 1]
            h[i + 1] = self.cs[i] * h[i + 1] - self.sn[i] * h[i]
            h[i] = t
        a, b = h[j], h[j + 1]
        rho = math.sqrt(a * a + b * b)
        if not (math.isfinite(rho) and rho != 0.0 and all(math.isfinite(v) for v in h[:j + 2])):
            self.on = False
            return
        self.cs.append(a / rho)
        self.sn.append(b / rho)
        self.R.append(h[:j] + [rho])
        self.g.append(-(self.sn[j] * self.g[j]))
        self.g[j] = self.cs[j] * self.g[j]
        self.m = j + 1
        self.on = not (b == 0.0 or abs(self.g[j + 1]) <= self.inner_tol * self.beta or self.m == self.restart)

    def y(self):
        y = [0.0] * self.m
        for i in range(self.m - 1, -1, -1):
            t = self.g[i]
            for l in range(i + 1, self.m):
                t = t - self.R[l][i] * y[l]
            y[i] = t / self.R[i][i]
        return y


def replay(s, rows, b, restart, max_cycles, tol, inner_tol):
    """FGMRES in numpy with the library's single-column solve for x_0 and each z_j: (x, dict of the struct's fields)"""
    def solve(v):
        y = np.array(v, np.float64)
        assert s.solve(y, 1) == SYMSOLVER_SUCCESS, s.last_error()
        return y
    xs, oms, iters = [solve(b)], [], 0
    while True:
        r, sv = dd_residual(rows, b, xs[-1])
        oms.append(omegas(rows, b, xs[-1], r, sv))
        try:
            out = rule(oms, max_cycles, tol)
            break
        except AssertionError:
            pass
        beta = math.sqrt(gdot(r, r))
        cy = Cycle(beta, restart, inner_tol)
        V, Z = [r / beta], []
        j = 0
        while cy.on:
            Z.append(solve(V[j]))
            w = apply_op(rows, Z[j])
            hs = []
            for _ in range(2):
                hp = [gdot(V[q], w) for q in range(j + 1)]
                for q in range(j + 1):
                    w = w - hp[q] * V[q]
                hs.append(hp)
            hn = math.sqrt(gdot(w, w))
            V.append(w / hn)
            cy.step([hs[0][q] + hs[1][q] for q in range(j + 1)] + [hn], j)
            j += 1
        iters += cy.iters
        d = np.zeros_like(b)
        for q, yq in enumerate(cy.y()):
            d = d + yq * Z[q]
        xs.append(xs[-1] + d)
    status, cycles, nres, o1, o2, first = out
    return xs[cycles], dict(omega_first=first, omega1=o1, omega2=o2, cycles=cycles, iters=iters, status=status,
                            nres=nres)


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


@pytest.mark.parametrize("n", [1, 255, 256, 257, 70000, 300001])
def test_fixed_grid_dot_is_accurate(n):
    rng = np.random.default_rng(n)
    a, b = rng.standard_normal(n), rng.standard_normal(n)
    exact = math.fsum((a * b).tolist())
    assert abs(gdot(a, b) - exact) <= 1e-13 * np.sum(np.abs(a * b))


def test_host_cycle_solves_the_least_squares_problem():
    """the replayed rotations and back substitution minimise || beta e_1 - H y || for a random Hessenberg matrix"""
    rng = np.random.default_rng(4)
    m = 7
    H = np.triu(rng.standard_normal((m + 1, m)), -1)
    cy = Cycle(2.5, m, 0.0)
    for j in range(m):
        cy.step(H[:j + 2, j], j)
    assert cy.m == m and not cy.on
    e = np.zeros(m + 1)
    e[0] = 2.5
    ref = np.linalg.lstsq(H, e, rcond=None)[0]
    assert np.allclose(cy.y(), ref, rtol=1e-12, atol=1e-12)
    assert math.isclose(abs(cy.g[m]), np.linalg.norm(e - H @ ref), rel_tol=1e-10)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def gmres(s, B, vals=None, device=False, **kw):
    """the library's FGMRES on the columns (rows of B): (X rows, dict of per-column arrays)"""
    if not device:
        X, d = s.solve_gmres(B.T, vals=vals, **kw)
        return np.ascontiguousarray(X.T), d
    import torch
    db = torch.tensor(np.ascontiguousarray(B).ravel(), dtype=torch.float64, device="cuda")
    dx = torch.zeros_like(db)
    dv = None if vals is None else torch.tensor(vals, dtype=torch.float64, device="cuda")
    st, d = s.solve_gmres_device(db.data_ptr(), dx.data_ptr(), B.shape[0], None if dv is None else dv.data_ptr(), **kw)
    assert st == SYMSOLVER_SUCCESS, s.last_error()
    assert_bits(db.cpu().numpy(), np.ascontiguousarray(B).ravel(), "b untouched")
    if dv is not None:
        assert_bits(dv.cpu().numpy(), vals, "vals untouched")
    return dx.cpu().numpy().reshape(B.shape), d


def perturbed(val, seed=3):
    return val * (1.0 + 1e-3 * np.random.default_rng(seed).uniform(-1.0, 1.0, len(val)))


KW = dict(restart=20, max_cycles=10, tol=EPS, inner_tol=1e-10)
SHORT = dict(restart=3, max_cycles=4, tol=EPS, inner_tol=0.0)   # cycles that end at the restart length


@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(ALL))
def test_bit_exact_replay(system):
    dim, irn, jcn, val = ALL[system]()
    s = factored(dim, irn, jcn, val)
    if system == "tridiag":
        assert s.info()["num_forced"] > 0
    B = np.random.default_rng(5).standard_normal((2, dim))
    for vals, kw in ((None, KW), (perturbed(val), KW), (perturbed(val), SHORT)):
        rows = rows_of(dim, irn, jcn, val if vals is None else vals)
        X, got = gmres(s, B, vals, **kw)
        for c in range(B.shape[0]):
            x_ref, ref = replay(s, rows, B[c], kw["restart"], kw["max_cycles"], kw["tol"], kw["inner_tol"])
            tag = (system, vals is None, kw["restart"], c)
            assert_bits(X[c], x_ref, tag + ("x",))
            assert_outcome(got, c, ref, tag)
        if vals is None:
            Xv, gv = gmres(s, B, np.array(val, np.float64), **kw)   # the factored values, passed: the same bits
            assert_bits(Xv, X, (system, "vals == factored values"))
            for c in range(B.shape[0]):
                assert_outcome(gv, c, {k: got[k][c] for k in FIELDS}, (system, c, "vals == factored values"))
    s.close()


def flipped(alpha, k=3, system="MBndryCntrl1_30"):
    """a handle on a system whose factorisation lifts no pivots (job 0 inverts A), with D^-1 multiplied by alpha at k
    1x1 pivots: M A is then similar to diag(alpha at k places, 1 elsewhere)"""
    dim, irn, jcn, val = SYSTEMS[system]()
    s = factored(dim, irn, jcn, val)
    assert s.info()["num_forced"] == 0
    _, ty, dinv = s.enquire_indef()
    piv = np.flatnonzero(ty == 1)
    pick = piv[np.linspace(0, len(piv) - 1, k).astype(int)]
    dinv[pick, 0] *= alpha
    assert s.alter_d(dinv) == SYMSOLVER_SUCCESS, s.last_error()
    return s, dim, irn, jcn, val


@pytest.mark.gpu
@pytest.mark.parametrize("alpha", [-1.0, 3.0])
def test_gmres_converges_where_refinement_fails(alpha):
    s, dim, irn, jcn, val = flipped(alpha)
    B = np.random.default_rng(7).standard_normal((3, dim))
    Xr, gr = s.solve_refined(B.T, 10, EPS)
    assert np.all(gr["status"] != 0), gr
    assert np.all(gr["omega1"] + gr["omega2"] > 1e6 * EPS), gr
    X, got = gmres(s, B, **KW)
    assert np.all(got["status"] == 0), got
    assert np.all(got["omega1"] + got["omega2"] <= EPS), got
    # I - M A has minimal polynomial of degree 2, so exact arithmetic needs at most 2 steps; from x_0 = M b the residual
    # even lies in the alpha-eigenspace of A M, and 1 step suffices (measured on an H100: 1 for every column)
    _, one = gmres(s, B, restart=20, max_cycles=1, tol=0.0, inner_tol=1e-10)
    assert np.all(one["iters"] <= 2), one["iters"]
    rows = rows_of(dim, irn, jcn, val)
    x_ref, ref = replay(s, rows, B[0], **KW)
    assert_bits(X[0], x_ref, "replay")
    assert_outcome(got, 0, ref, "replay")
    s.close()


@pytest.mark.gpu
def test_other_values_without_refactorisation():
    """A' = A + diag(delta) at k variables, delta_i = 4 / (A^-1)_ii: I - M A' has an eigenvalue near -4, so classical
    refinement with M diverges; FGMRES with M solves A' x = b to the accuracy its omega implies"""
    import scipy.sparse.linalg as sla
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = factored(dim, irn, jcn, val)
    diag = np.flatnonzero(irn == jcn)
    var = irn[diag] - 1
    cand = diag[np.linspace(0, len(diag) - 1, 40).astype(int)]
    ainv = []
    for t in cand:
        e = np.zeros(dim)
        e[irn[t] - 1] = 1.0
        assert s.solve(e, 1) == SYMSOLVER_SUCCESS
        ainv.append(e[irn[t] - 1])
    ainv = np.array(ainv)
    pick = cand[np.argsort(-np.abs(ainv))[:2]]
    v2 = val.copy()
    for t, a in zip(pick, ainv[np.argsort(-np.abs(ainv))[:2]]):
        first = diag[var == irn[t] - 1][0]
        v2[first] += 4.0 / a
    A2 = to_scipy(dim, irn, jcn, v2).tocsc()
    lu = sla.splu(A2)
    assert np.all(np.isfinite(lu.U.diagonal())) and np.min(np.abs(lu.U.diagonal())) > 0.0
    rows2 = rows_of(dim, irn, jcn, v2)
    B = np.random.default_rng(8).standard_normal((2, dim))
    X, got = gmres(s, B, v2, **KW)
    for c in range(2):
        _, rref = refine_replay(s, rows2, B[c], 10, EPS)
        assert rref["status"] != 0, rref
        assert got["status"][c] == 0, got
        om = got["omega1"][c] + got["omega2"][c]
        assert om <= EPS
        xs = lu.solve(B[c])
        kappa = np.linalg.cond(A2.toarray(), np.inf)
        err = np.abs(X[c] - xs).max() / np.abs(xs).max()
        assert err <= 10.0 * kappa * max(om, EPS), (err, kappa, om)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["tridiag", "flipped"])
def test_blocks_and_entry_points(system, monkeypatch):
    """every column bit-identical to the call on it alone, to the device entry point, to a repeated call and to
    B200_SOLVE_BLOCK=1; the 11 columns finish at different cycles"""
    def make():
        if system == "flipped":
            return flipped(-1.0)
        dim, irn, jcn, val = tridiag()
        return factored(dim, irn, jcn, val), dim, irn, jcn, val
    s, dim, irn, jcn, val = make()
    B = block_columns(dim)
    vals = perturbed(val) if system == "tridiag" else None
    for kw in (KW, SHORT):
        X, got = gmres(s, B, vals, **kw)
        assert got["status"][3] == 0 and got["cycles"][3] == 0 and not np.any(X[3])
        Xd, gd = gmres(s, B, vals, device=True, **kw)
        X2, g2 = gmres(s, B, vals, **kw)
        for c in range(B.shape[0]):
            Xc, gc = gmres(s, B[c:c + 1], vals, **kw)
            assert_bits(X[c], Xc[0], (kw["restart"], c, "alone"))
            for other, tag in ((gd, "device"), (g2, "repeat"), (gc, "alone")):
                assert_outcome(got, c, {k: np.asarray(other[k])[0 if tag == "alone" else c] for k in FIELDS},
                               (kw["restart"], c, tag))
        assert_bits(Xd, X, (kw["restart"], "device"))
        assert_bits(X2, X, (kw["restart"], "repeat"))
        assert len(set(got["nres"].tolist())) > 1, got["nres"]
    s.close()
    monkeypatch.setenv("B200_SOLVE_BLOCK", "1")
    s1 = make()[0]
    X1, g1 = gmres(s1, B, vals, **KW)
    s1.close()
    monkeypatch.delenv("B200_SOLVE_BLOCK")
    s = make()[0]
    X, got = gmres(s, B, vals, **KW)
    s.close()
    assert_bits(X1, X, "B200_SOLVE_BLOCK=1")
    for c in range(B.shape[0]):
        assert_outcome(got, c, {k: np.asarray(g1[k])[c] for k in FIELDS}, (c, "block 1"))


@pytest.mark.gpu
def test_plain_solve_and_no_side_effects():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = factored(dim, irn, jcn, val)
    B = np.random.default_rng(4).standard_normal((3, dim))
    X0 = B.copy()
    assert s.solve(X0.ravel(), 3) == SYMSOLVER_SUCCESS
    ea0 = s.error_analysis(B.T, X0.T, True)
    Xr0, r0 = s.solve_refined(B.T)
    X, got = gmres(s, B, max_cycles=0)
    assert_bits(X, X0, "max_cycles = 0")
    assert np.all(got["cycles"] == 0) and np.all(got["nres"] == 1) and np.all(got["iters"] == 0)
    gmres(s, B, perturbed(val), **KW)
    gmres(s, B, **KW)
    X1 = B.copy()
    assert s.solve(X1.ravel(), 3) == SYMSOLVER_SUCCESS
    assert_bits(X1, X0, "solve after")
    ea1 = s.error_analysis(B.T, X0.T, True)
    for k in ea0:
        assert_bits(np.asarray(ea0[k], np.float64), np.asarray(ea1[k], np.float64), ("error_analysis", k))
    Xr1, r1 = s.solve_refined(B.T)
    assert_bits(Xr1, Xr0, "solve_refined after")
    for k in r0:
        assert_bits(np.asarray(r0[k], np.float64), np.asarray(r1[k], np.float64), ("solve_refined", k))
    assert s.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    X2 = B.copy()
    assert s.solve(X2.ravel(), 3) == SYMSOLVER_SUCCESS
    assert_bits(X2, X0, "refactor after")
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1"])
def test_launch_counts(block, monkeypatch):
    """one column: 1 + L0 + 5 nres - 2 + (L0 + 6) iters; a block of columns that take at most one cycle:
    1 + L0 + 3 E + 2 (E - 1) + (L0 + 6) T, E the largest nres and T the most steps of a column"""
    if block is not None:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*tridiag())
    B = block_columns(2000)[:8]
    x = B[0].copy()
    assert s.solve(x, 1) == SYMSOLVER_SUCCESS
    L0 = s.info()["launches_solve"]

    def per_block(nres, iters):
        return L0 + 3 * nres + 2 * (nres - 1) + (L0 + 6) * iters
    for device in (False, True):
        _, got = gmres(s, B[:1], device=device, **KW)
        assert s.info()["launches_solve"] == 1 + per_block(got["nres"][0], got["iters"][0])
        assert s.info()["ms_solve_gpu"] > 0.0
        _, got = gmres(s, B, device=device, restart=20, max_cycles=1, tol=EPS, inner_tol=1e-10)
        want = 1 + (per_block(got["nres"].max(), got["iters"].max()) if block is None
                    else int(np.sum([per_block(e, t) for e, t in zip(got["nres"], got["iters"])])))
        assert s.info()["launches_solve"] == want, (s.info()["launches_solve"], want, got)
    s.close()


@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    L = s._L
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    b, x = np.ones(dim), np.full(dim, 42.0)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
    out = (Gmres * 2)()

    def refused(nrhs, pb, px, match, restart=20, max_cycles=10, tol=EPS, inner_tol=1e-10, device=False):
        for o in out:
            for k in FIELDS:
                setattr(o, k, 42)
        f = L.b200ldlt_solve_gmres_device if device else L.b200ldlt_solve_gmres
        assert f(s._h, nrhs, pb, px, None, restart, max_cycles, tol, inner_tol, out) == SYMSOLVER_FATAL_ERROR \
            and match in s.last_error(), s.last_error()
        assert all(getattr(o, k) == 42 for o in out for k in FIELDS)
        assert np.all(x == 42.0)

    refused(1, dp(b), dp(x), "no factors")
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    refused(-1, dp(b), dp(x), "nrhs")
    refused(1, dp(b), dp(x), "restart", restart=0)
    refused(1, dp(b), dp(x), "restart", restart=65)
    refused(1, dp(b), dp(x), "max_cycles", max_cycles=-1)
    refused(1, dp(b), dp(x), "tol", tol=-1.0)
    refused(1, dp(b), dp(x), "tol", tol=NAN)
    refused(1, dp(b), dp(x), "inner_tol", inner_tol=-1.0)
    refused(1, dp(b), dp(x), "inner_tol", inner_tol=NAN)
    refused(1, None, dp(x), "NULL")
    refused(1, dp(b), None, "NULL")
    refused(1, None, None, "NULL", device=True)
    refused(1, dp(x), dp(x), "x must not be b")
    assert L.b200ldlt_solve_gmres(s._h, 1, dp(b), dp(x), None, 20, 10, EPS, 1e-10, None) == SYMSOLVER_FATAL_ERROR
    assert np.all(x == 42.0)
    # nrhs = 0: success, nothing written, nothing launched
    for o in out:
        o.status = 42
    assert L.b200ldlt_solve_gmres(s._h, 0, None, None, None, 20, 10, EPS, 1e-10, out) == SYMSOLVER_SUCCESS
    assert out[0].status == 42 and s.info()["launches_solve"] == 0
    # Schur mode: the shared refusal
    assert s.set_schur(np.arange(dim - 5, dim)) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    refused(1, dp(b), dp(x), "solve_gmres: Schur mode")
    assert s.set_schur([]) == SYMSOLVER_SUCCESS
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    X, got = s.solve_gmres(b)
    assert got["status"][0] in (0, 1, 2)
    # sharded handle
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    refused(1, dp(b), dp(x), "sharded")
    s.close()
