"""Sparse forward solve (b200ldlt_sparse_fwd_solve / _device): job 1 (L^-1 P^T S b, pivot order) of a right-hand side
with few non-zeros, swept over the fronts its non-zeros reach, through the C ABI and the HSL_MA97 shim
(ma97_sparse_fwd_solve_d).

The reach of a pattern is the set of fronts on the elimination-tree paths from the fronts of its variables to the root;
the call returns the pivot positions of the reach (ascending) and job 1's vector there, which must equal job 1 of the
dense b as values, with job 1 exactly zero everywhere else."""
import ctypes as C
import functools

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt

from test_partial_solve import SYSTEMS, assert_bits, factored, run
from test_lmultiply_alter import Ma97, lmul

NEW_SYMBOLS = ["b200ldlt_sparse_fwd_solve", "b200ldlt_sparse_fwd_solve_device", "ma97_sparse_fwd_solve_d"]


@functools.lru_cache(maxsize=None)
def large():
    return mbndry_kkt(400)[:4]


ALL_SYSTEMS = dict(SYSTEMS, mbndry400=large)


def sfs(s, bindex, bvals, device):
    """(xindex, x) of the sparse forward solve, host or device entry point"""
    if device:
        import torch
        db = torch.tensor(np.asarray(bvals, np.float64), device="cuda")
        dx = torch.full((s.dim,), np.nan, dtype=torch.float64, device="cuda")
        xi = s.sparse_fwd_solve_device(bindex, db.data_ptr(), dx.data_ptr())
        return xi, dx[:len(xi)].cpu().numpy()
    return s.sparse_fwd_solve(bindex, bvals)


def dense_job1(s, bindex, bvals):
    B = np.zeros((1, s.dim))
    B[0, bindex] = bvals
    return run(s, 1, B, True)[0]


class Tree:
    """the elimination tree and the variable -> pivot position map of a factored handle, from the symbolic arrays and
    enquire_indef (independent of the library's own reach computation)"""

    def __init__(self, s):
        self.sn_start = s.symbolic("sn_start")
        self.sn_parent = s.symbolic("sn_parent")
        self.rows_ptr = s.symbolic("rows_ptr")
        self.level = s.symbolic("sn_level")
        var = s.enquire_indef()[0]
        self.pos = np.empty(s.dim, np.int64)
        self.pos[var] = np.arange(s.dim)
        self.nsn = len(self.sn_start) - 1
        self.k = np.diff(self.sn_start)
        self.f = self.k + np.diff(self.rows_ptr)
        self.children = [[] for _ in range(self.nsn)]
        for c, p in enumerate(self.sn_parent):
            if p >= 0:
                self.children[p].append(c)

    def front_of(self, v):
        return int(np.searchsorted(self.sn_start, self.pos[v], side="right") - 1)

    def reach(self, bindex):
        fronts = set()
        for v in bindex:
            f = self.front_of(v)
            while f >= 0 and f not in fronts:
                fronts.add(f)
                f = int(self.sn_parent[f])
        return sorted(fronts)

    def positions(self, fronts):
        return np.concatenate([np.arange(self.sn_start[f], self.sn_start[f + 1]) for f in fronts]).astype(np.int64)

    def direct(self, levels):
        """fronts the direct kernel solves with B200_SOLVE_DIRECT=levels: on the lowest levels, order <= 64, every child
        of the same kind (children precede parents)"""
        d = np.zeros(self.nsn, bool)
        for s_ in range(self.nsn):
            d[s_] = self.level[s_] < levels and self.f[s_] <= 64 and all(d[c] for c in self.children[s_])
        return d

    def leaf_var(self, var, which=0):
        leaves = [f for f in range(self.nsn) if not self.children[f]]
        return int(var[self.sn_start[leaves[which % len(leaves)]]])


def patterns(n, seed):
    rng = np.random.default_rng(seed)
    out = {"one": rng.choice(n, 1, replace=False), "five": rng.choice(n, min(5, n), replace=False),
           "fifty": rng.choice(n, min(50, n), replace=False), "tenth": rng.choice(n, max(1, n // 10), replace=False),
           "all": rng.permutation(n)}
    return {k: (v.astype(np.int32), rng.standard_normal(len(v))) for k, v in out.items()}


def check_against_job1(s, tree, bindex, bvals, tag):
    ref = dense_job1(s, bindex, bvals)
    exp = tree.positions(tree.reach(bindex))
    mask = np.ones(s.dim, bool)
    mask[exp] = False
    assert np.all(ref[mask] == 0.0), (tag, "job 1 non-zero outside the reach")
    first = None
    for device in (False, True):
        xi, x = sfs(s, bindex, bvals, device)
        assert np.array_equal(xi, exp), (tag, device, "pattern")
        assert np.array_equal(x, ref[xi]), (tag, device, np.flatnonzero(x != ref[xi])[:5])
        if first is None:
            first = x
        else:
            assert_bits(x, first, (tag, "host = device"))
        assert_bits(sfs(s, bindex, bvals, device)[1], x, (tag, device, "repeat"))


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


# ---- 1. + 2. equality with job 1, the pattern of the reach ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("env", [{}, {"B200_SOLVE_DIRECT": "0"}, {"B200_SOLVE_DIRECT": "1"}, {"B200_SOLVE_DIRECT": "4"},
                                 {"B200_SOLVE_NOPAIR": "1"}], ids=["default", "direct0", "direct1", "direct4", "nopair"])
@pytest.mark.parametrize("system", sorted(ALL_SYSTEMS))
def test_equals_job1_on_the_reach(system, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    s = factored(*ALL_SYSTEMS[system]())
    tree = Tree(s)
    for name, (bi, bv) in patterns(s.dim, 11).items():
        check_against_job1(s, tree, bi, bv, (system, name))
    var = s.enquire_indef()[0]
    leaf = np.array([tree.leaf_var(var)], np.int32)
    check_against_job1(s, tree, leaf, np.array([1.5]), (system, "leaf"))
    s.close()


# ---- 3. stale sweep state -----------------------------------------------------------------------------------------------
def stale_state_round(s, fresh, tree, tag):
    """a sparse call after each kind of solve gives the bits of the same call on a fresh handle of the same factors; full
    solves between sparse calls keep their bits"""
    n = s.dim
    rng = np.random.default_rng(21)
    var = s.enquire_indef()[0]
    a_idx = np.array([tree.leaf_var(var, 0)], np.int32)
    ra = set(tree.reach(a_idx))
    # the other pattern: the leaf whose reach shares the fewest fronts with a's (disjoint where the tree is a forest)
    leaves = [f for f in range(tree.nsn) if not tree.children[f]]
    cand = [int(var[tree.sn_start[f]]) for f in leaves[:: max(1, len(leaves) // 64)]]
    b_var = min(cand, key=lambda v: len(ra & set(tree.reach([v]))))
    b_idx = np.array([b_var], np.int32)
    pats = {"a": (a_idx, np.array([0.75])), "b": (b_idx, np.array([-2.0])),
            "fifty": (rng.choice(n, min(50, n), replace=False).astype(np.int32), rng.standard_normal(min(50, n)))}
    want = {k: [sfs(fresh, bi, bv, d) for d in (False, True)] for k, (bi, bv) in pats.items()}
    rhs = rng.standard_normal((8, n))
    x_full = rhs[0].copy()
    assert fresh.solve(x_full, 1) == SYMSOLVER_SUCCESS
    before = {
        "full solve": lambda: s.solve(rhs[0].copy(), 1),
        "job 1": lambda: run(s, 1, rhs[:1], True),
        "blocked nrhs=8": lambda: run(s, 0, rhs, True),
        "lmultiply": lambda: lmul(s, 0, rhs[:1], True),
        "sparse b": lambda: sfs(s, *pats["b"], True),
    }
    for what, op in before.items():
        for k, (bi, bv) in pats.items():
            if what == "sparse b" and k == "b":
                continue
            for d in (False, True):
                op()
                xi, x = sfs(s, bi, bv, d)
                assert np.array_equal(xi, want[k][d][0]), (tag, what, k, d)
                assert_bits(x, want[k][d][1], (tag, what, k, d))
                xs = rhs[0].copy()
                assert s.solve(xs, 1) == SYMSOLVER_SUCCESS
                assert_bits(xs, x_full, (tag, what, k, d, "full solve after"))


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random", "mbndry400"])
def test_stale_state_and_refactor(system):
    args = ALL_SYSTEMS[system]()
    s, fresh = factored(*args), factored(*args)
    stale_state_round(s, fresh, Tree(s), system)
    assert s.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    stale_state_round(s, fresh, Tree(s), (system, "refactor"))
    s.close()
    fresh.close()


@pytest.mark.gpu
def test_stale_state_after_reanalysis_by_increase_quality():
    """the lifted-pivot system of test_partial_solve: increase_quality schedules a re-analysis, which rebuilds the plan"""
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    s, fresh = factored(n, irn, jcn, val), factored(n, irn, jcn, val)
    assert s.info()["num_forced"] > 0
    stale_state_round(s, fresh, Tree(s), "before")
    for h in (s, fresh):
        assert h.IncreaseQuality()
        assert h.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    tree = Tree(s)
    stale_state_round(s, fresh, tree, "reanalysed")
    for name, (bi, bv) in patterns(n, 3).items():
        check_against_job1(s, tree, bi, bv, ("reanalysed", name))
    s.close()
    fresh.close()


# ---- 4. the use case: a block of A^-1 from sparse solves ------------------------------------------------------------------
def apply_dinv(ty, dinv2, y):
    z = dinv2[:, 0] * y
    two = np.flatnonzero(ty == 2)
    z[two] += dinv2[two, 1] * y[two + 1]
    z[two + 1] += dinv2[two, 1] * y[two]
    return z


# Measured on an H100 (H100 80GB HBM3), MBndryCntrl1 N=400, 12 variables (4 in leaf fronts, 4 mid-tree, 4 in the root):
# max |E - E_ref| / max |E_ref| = 3.9e-17 for the 12 x 12 block E built as y_i^T D^-1 y_j against the entries of full
# solves.  Both evaluate the same bilinear form through the same factors in a different order, so they differ by rounding
# only; the tolerance sits about 2.5e4 above the measurement (room for the rounding of other matrices and patterns),
# while a wrong entry of y (a missed front, a stale update vector) shows as an O(1) error.
BLOCK_TOL = 1e-12


@pytest.mark.gpu
def test_block_of_inverse_from_sparse_solves():
    s = factored(*large())
    tree = Tree(s)
    var, ty, dinv2 = s.enquire_indef()
    leaves = [f for f in range(tree.nsn) if not tree.children[f]]
    roots = [f for f in range(tree.nsn) if tree.sn_parent[f] < 0]
    half = int(tree.level.max()) // 2
    mids = sorted((f for f in range(tree.nsn) if tree.children[f]), key=lambda f: (abs(int(tree.level[f]) - half), f))[:4]
    fronts = leaves[:: max(1, len(leaves) // 4)][:4] + mids
    root = max(roots, key=lambda f: tree.k[f])   # (the tree may be a forest: the top separator has the most pivots)
    rk = int(tree.k[root])
    vars12 = [int(var[tree.sn_start[f]]) for f in fronts] + [int(var[tree.sn_start[root] + q * (rk - 1) // 3]) for q in range(4)]
    assert len(set(vars12)) == 12
    n = s.dim
    Y = np.zeros((12, n))
    for i, v in enumerate(vars12):
        xi, x = sfs(s, np.array([v], np.int32), np.array([1.0]), True)
        Y[i, xi] = x
    E = np.array([[Y[i] @ apply_dinv(ty, dinv2, Y[j]) for j in range(12)] for i in range(12)])
    E_ref = np.zeros((12, 12))
    for j, v in enumerate(vars12):
        e = np.zeros(n)
        e[v] = 1.0
        assert s.solve(e, 1) == SYMSOLVER_SUCCESS
        E_ref[:, j] = e[vars12]
    err = np.abs(E - E_ref).max() / np.abs(E_ref).max()
    print("MEASURED A^-1 block rel. error %.2e" % err)
    assert err <= BLOCK_TOL, err
    assert np.abs(E - E.T).max() <= BLOCK_TOL * np.abs(E).max()
    s.close()


# ---- 5. launch counts ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("direct", ["0", "2"])
def test_launch_counts(direct, monkeypatch):
    """2 + (direct levels holding a direct front of the reach) + (1 if the reach has a front above them)"""
    monkeypatch.setenv("B200_SOLVE_DIRECT", direct)
    s = factored(*mbndry_kkt(70, sigma_spread=3.0, seed=5)[:4])
    tree = Tree(s)
    dfront = tree.direct(int(direct))
    var = s.enquire_indef()[0]
    leaf = [f for f in range(tree.nsn) if not tree.children[f] and (dfront[f] or direct == "0")][0]
    pats = {"leaf": np.array([var[tree.sn_start[leaf]]], np.int32), "dense": np.arange(s.dim, dtype=np.int32)}
    for name, bi in pats.items():
        reach = tree.reach(bi)
        d = len({int(tree.level[f]) for f in reach if dfront[f]})
        t = int(any(not dfront[f] for f in reach))
        for device in (False, True):
            sfs(s, bi, np.ones(len(bi)), device)
            info = s.info()
            assert info["launches_solve"] == 2 + d + t, (name, device, info["launches_solve"], d, t)
            assert info["ms_solve_gpu"] > 0.0
    if direct == "2":
        assert len({int(tree.level[f]) for f in range(tree.nsn) if dfront[f]}) == 2   # the dense pattern: 5 launches
    xi, x = s.sparse_fwd_solve(np.zeros(0, np.int32), np.zeros(0))
    assert len(xi) == 0 and s.info()["launches_solve"] == 0
    s.close()


# ---- 6. refusals --------------------------------------------------------------------------------------------------------
def raw_call(s, nbi, bindex, bvals, device):
    """the C entry point on sentinel outputs; returns (status, nxi, xindex, x) with x read back"""
    L = s._L
    n = s.dim
    nxi = C.c_int(-7)
    xi = np.full(n, 99, np.int32)
    ip = xi.ctypes.data_as(C.POINTER(C.c_int))
    bp = None if bindex is None else np.ascontiguousarray(bindex, np.int32)
    bptr = None if bp is None else bp.ctypes.data_as(C.POINTER(C.c_int))
    if device:
        import torch
        db = torch.tensor(np.asarray(bvals, np.float64), device="cuda") if len(bvals) else torch.zeros(1, dtype=torch.float64, device="cuda")
        dx = torch.full((n,), 42.0, dtype=torch.float64, device="cuda")
        st = L.b200ldlt_sparse_fwd_solve_device(s._h, nbi, bptr, C.c_void_p(db.data_ptr()), C.byref(nxi), ip,
                                                C.c_void_p(dx.data_ptr()))
        return st, nxi.value, xi, dx.cpu().numpy()
    x = np.full(n, 42.0)
    bv = np.ascontiguousarray(bvals, np.float64)
    st = L.b200ldlt_sparse_fwd_solve(s._h, nbi, bptr, bv.ctypes.data_as(C.POINTER(C.c_double)), C.byref(nxi), ip,
                                     x.ctypes.data_as(C.POINTER(C.c_double)))
    return st, nxi.value, xi, x


def assert_refused(s, nbi, bindex, bvals, msg):
    for device in (False, True):
        st, nxi, xi, x = raw_call(s, nbi, bindex, bvals, device)
        assert st == SYMSOLVER_FATAL_ERROR and msg in s.last_error(), (msg, device, st, s.last_error())
        assert nxi == -7 and np.all(xi == 99) and np.all(x == 42.0), (msg, device)


@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    one = np.array([3], np.int32)
    assert_refused(s, 1, one, [1.0], "no factors")
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    assert_refused(s, -1, one, [1.0], "nbi")
    assert_refused(s, dim + 1, np.arange(dim + 1), np.ones(dim + 1), "nbi")
    assert_refused(s, 1, None, [1.0], "NULL")
    assert_refused(s, 2, np.array([0, -1]), [1.0, 2.0], "out of range")
    assert_refused(s, 2, np.array([dim, 0]), [1.0, 2.0], "out of range")
    assert_refused(s, 3, np.array([4, 9, 4]), [1.0, 2.0, 3.0], "twice")
    # the handle is intact after refusals
    tree = Tree(s)
    check_against_job1(s, tree, np.array([4, 9], np.int32), np.array([1.0, 2.0]), "after refusals")
    st, nxi, xi, x = raw_call(s, 0, None, [], False)
    assert st == SYMSOLVER_SUCCESS and nxi == 0
    v0 = val.copy()
    r = int(irn[0])
    v0[(irn == r) | (jcn == r)] = 0.0
    s.GetValuesArrayPtr()[:] = v0
    assert s.factor(False, 0)[0] == SYMSOLVER_SINGULAR
    assert_refused(s, 1, one, [1.0], "no factors")
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    L = s._L
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    assert_refused(s, 1, one, [1.0], "sharded")
    s.close()


# ---- 7. the HSL_MA97 shim -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["hs071_0", "MBndryCntrl1_30", "mbndry30_wzero"])
def test_ma97_shim_sparse_fwd_solve(system, built_lib):
    m = Ma97(built_lib, *SYSTEMS[system]())
    assert m.flag() == 0
    dim, lib, ip, dp = m.dim, m.lib, m.ip, m.dp
    f_arrays = C.cast(m.ctrl, C.POINTER(C.c_int))
    rng = np.random.default_rng(9)
    order = np.arange(1, dim + 1, dtype=np.int32)
    for nbi in (1, min(5, dim), dim):
        bi = rng.choice(dim, nbi, replace=False).astype(np.int32)
        bv = rng.standard_normal(nbi)
        xi_ref, x_ref = m.s.sparse_fwd_solve(bi, bv)
        dense = np.zeros(dim)
        dense[xi_ref] = x_ref
        b = np.full(dim, np.nan)      # entries outside bindex are not read
        b[bi] = bv
        for base in (0, 1):
            f_arrays[0] = base
            for with_order in (False, True):
                nxi = C.c_int(-1)
                xindex = np.full(dim, -5, np.int32)
                x = np.full(dim, 42.0)
                bidx = (bi + base).astype(np.int32)
                lib.ma97_sparse_fwd_solve_d(C.c_int(nbi), bidx.ctypes.data_as(ip), b.ctypes.data_as(dp),
                                            order.ctypes.data_as(ip) if with_order else None, C.byref(nxi),
                                            xindex.ctypes.data_as(ip), x.ctypes.data_as(dp), *m.keeps())
                assert m.flag() == 0, (nbi, base, with_order)
                assert nxi.value == len(xi_ref)
                assert np.array_equal(xindex[:nxi.value], xi_ref + base)
                assert_bits(x, dense, (nbi, base, with_order))
    f_arrays[0] = 0
    # refused: a repeated index; nothing written
    nxi = C.c_int(-1)
    x = np.full(dim, 42.0)
    xindex = np.full(dim, -5, np.int32)
    bad = np.array([0, 0], np.int32)
    b = np.ones(dim)
    lib.ma97_sparse_fwd_solve_d(C.c_int(2), bad.ctypes.data_as(ip), b.ctypes.data_as(dp), None, C.byref(nxi),
                                xindex.ctypes.data_as(ip), x.ctypes.data_as(dp), *m.keeps())
    assert m.flag() < 0 and nxi.value == -1 and np.all(x == 42.0) and np.all(xindex == -5)
    m.close()
