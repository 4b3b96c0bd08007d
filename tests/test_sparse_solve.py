"""Sparse solve (b200ldlt_sparse_solve / _device): chosen entries of x = A^-1 b for right-hand sides that share one
sparse pattern, the forward sweep pruned to the fronts b reaches and the backward sweep pruned to the fronts the
selection reaches.

Every returned entry must equal job 0 on the dense b as a value; with bindex and xsel both NULL the call is
b200ldlt_solve, bit for bit and launch for launch."""
import ctypes as C

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS

from test_fredholm import handle, zeroed
from test_lmultiply_alter import lmul
from test_partial_solve import SYSTEMS, assert_bits, factored, run
from test_sparse_fwd_solve import ALL_SYSTEMS, Tree, large, patterns, sfs

NEW_SYMBOLS = ["b200ldlt_sparse_solve", "b200ldlt_sparse_solve_device"]


def sps(s, bindex, B, xsel, device):
    """the nrhs x nxs entries of the sparse solve of the rows of B (nrhs x nbi), host or device entry point"""
    B = np.atleast_2d(np.asarray(B, np.float64))
    nrhs = B.shape[0]
    nxs = s.dim if xsel is None else len(xsel)
    if device:
        import torch
        db = torch.tensor(B.ravel(), device="cuda") if B.size else torch.zeros(1, dtype=torch.float64, device="cuda")
        dx = torch.full((max(nrhs * nxs, 1),), np.nan, dtype=torch.float64, device="cuda")
        st = s.sparse_solve_device(bindex, db.data_ptr(), xsel, dx.data_ptr(), nrhs)
        assert st == SYMSOLVER_SUCCESS, s.last_error()
        return dx[:nrhs * nxs].cpu().numpy().reshape(nrhs, nxs)
    return s.sparse_solve(bindex, B, xsel)


def dense_b(n, bindex, B):
    B = np.atleast_2d(B)
    if bindex is None:
        return B.copy()
    D = np.zeros((B.shape[0], n))
    D[:, bindex] = B
    return D


def lifted():
    """the tridiagonal with tiny diagonal entries: lifted pivots (num_forced > 0)"""
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    return n, irn, jcn, val


def root_var(s, tree):
    var = s.enquire_indef()[0]
    roots = [f for f in range(tree.nsn) if tree.sn_parent[f] < 0]
    root = max(roots, key=lambda f: tree.k[f])
    return int(var[tree.sn_start[root] + tree.k[root] // 2])


def selections(s, tree, seed):
    n = s.dim
    rng = np.random.default_rng(seed)
    var = s.enquire_indef()[0]
    rep = rng.choice(n, min(6, n), replace=False)
    rep = rng.permutation(np.concatenate([rep, rep[:3], rep[:1]]))
    out = {"one": rng.choice(n, 1, replace=False), "five": rng.choice(n, min(5, n), replace=False),
           "fifty": rng.choice(n, min(50, n), replace=False), "tenth": rng.choice(n, max(1, n // 10), replace=False),
           "leaf": np.array([tree.leaf_var(var, 1)]), "root": np.array([root_var(s, tree)]), "repeats": rep}
    sel = {k: v.astype(np.int32) for k, v in out.items()}
    sel["all"] = None
    return sel


def b_patterns(s, tree, seed):
    var = s.enquire_indef()[0]
    pats = dict(patterns(s.dim, seed))
    pats["leaf"] = (np.array([tree.leaf_var(var)], np.int32), np.array([1.5]))
    pats["dense"] = (None, np.random.default_rng(seed + 1).standard_normal(s.dim))
    return pats


def check_against_job0(s, bindex, bvals, sels, tag):
    ref = run(s, 0, dense_b(s.dim, bindex, bvals), True)[0]
    for name, xsel in sels.items():
        exp = ref if xsel is None else ref[xsel]
        first = None
        for device in (False, True):
            x = sps(s, bindex, bvals, xsel, device)[0]
            assert np.array_equal(x, exp), (tag, name, device, np.flatnonzero(x != exp)[:5])
            if first is None:
                first = x
            else:
                assert_bits(x, first, (tag, name, "host = device"))
            assert_bits(sps(s, bindex, bvals, xsel, device)[0], x, (tag, name, device, "repeat"))


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


# ---- 1. equality with job 0 -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("env", [{}, {"B200_SOLVE_DIRECT": "0"}, {"B200_SOLVE_DIRECT": "1"}, {"B200_SOLVE_DIRECT": "4"},
                                 {"B200_SOLVE_NOPAIR": "1"}], ids=["default", "direct0", "direct1", "direct4", "nopair"])
@pytest.mark.parametrize("system", sorted(ALL_SYSTEMS))
def test_equals_job0(system, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    s = factored(*ALL_SYSTEMS[system]())
    tree = Tree(s)
    sels = selections(s, tree, 5)
    for name, (bi, bv) in b_patterns(s, tree, 11).items():
        check_against_job0(s, bi, bv, sels, (system, name))
    s.close()


# ---- 2. both NULL is b200ldlt_solve ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random", "mbndry400"])
def test_dense_and_full_is_solve(system):
    s = factored(*ALL_SYSTEMS[system]())
    rng = np.random.default_rng(4)
    for nrhs in (1, 3):
        B = rng.standard_normal((nrhs, s.dim))
        for device in (False, True):
            ref = run(s, 0, B, device)
            ref_launches = s.info()["launches_solve"]
            if not device:
                x = B.ravel().copy()
                assert s.solve(x, nrhs) == SYMSOLVER_SUCCESS
                assert_bits(x, ref.ravel(), (system, nrhs, "solve = job 0"))
                ref_launches = s.info()["launches_solve"]
            x = sps(s, None, B, None, device)
            assert_bits(x, ref, (system, nrhs, device))
            assert s.info()["launches_solve"] == ref_launches, (system, nrhs, device)
    s.close()


# ---- 3. blocks ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block", ["1", "2", None])
def test_blocks_equal_single_columns(block, monkeypatch):
    if block is not None:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*SYSTEMS["MBndryCntrl1_30"]())
    tree = Tree(s)
    n = s.dim
    rng = np.random.default_rng(7)
    var = s.enquire_indef()[0]
    cases = {"sparse": (rng.choice(n, 7, replace=False).astype(np.int32), rng.choice(n, 9).astype(np.int32)),
             "leaf-root": (np.array([tree.leaf_var(var)], np.int32), np.array([root_var(s, tree)], np.int32)),
             "dense b": (None, rng.choice(n, 5).astype(np.int32)),
             "all x": (rng.choice(n, 3, replace=False).astype(np.int32), None)}
    for name, (bi, xs) in cases.items():
        nbi = n if bi is None else len(bi)
        for nrhs in (1, 3, 8, 11):
            B = rng.standard_normal((nrhs, nbi))
            ref = run(s, 0, dense_b(n, bi, B), True)
            exp = ref if xs is None else ref[:, xs]
            for device in (False, True):
                X = sps(s, bi, B, xs, device)
                assert np.array_equal(X, exp), (name, nrhs, device)
                for c in range(nrhs):
                    assert_bits(X[c], sps(s, bi, B[c], xs, device)[0], (name, nrhs, device, c))
    s.close()


def raw_call(s, nrhs, nbi, bindex, b, nxs, xsel, device, nout=16):
    """the C entry point on a NaN-filled x of nout doubles; returns (status, x read back)"""
    L = s._L
    ip = C.POINTER(C.c_int)
    bi = None if bindex is None else np.ascontiguousarray(bindex, np.int32)
    xs = None if xsel is None else np.ascontiguousarray(xsel, np.int32)
    pbi = None if bi is None else bi.ctypes.data_as(ip)
    pxs = None if xs is None else xs.ctypes.data_as(ip)
    if device:
        import torch
        db = None if b is None else torch.tensor(np.asarray(b, np.float64).ravel(), device="cuda")
        dx = torch.full((nout,), np.nan, dtype=torch.float64, device="cuda")
        st = L.b200ldlt_sparse_solve_device(s._h, nrhs, nbi, pbi, None if db is None else C.c_void_p(db.data_ptr()),
                                            nxs, pxs, C.c_void_p(dx.data_ptr()))
        return st, dx.cpu().numpy()
    x = np.full(nout, np.nan)
    bv = None if b is None else np.ascontiguousarray(b, np.float64).ravel()
    st = L.b200ldlt_sparse_solve(s._h, nrhs, nbi, pbi, None if bv is None else bv.ctypes.data_as(C.POINTER(C.c_double)),
                                 nxs, pxs, x.ctypes.data_as(C.POINTER(C.c_double)))
    return st, x


@pytest.mark.gpu
def test_no_columns():
    s = factored(*SYSTEMS["MBndryCntrl1_30"]())
    one = np.array([3], np.int32)
    for device in (False, True):
        for nrhs, nxs, xs in ((0, 1, one), (2, 0, np.zeros(0, np.int32))):
            sps(s, one, np.ones((1, 1)), one, device)
            st, x = raw_call(s, nrhs, 1, one, np.ones(max(nrhs, 1)), nxs, xs, device)
            assert st == SYMSOLVER_SUCCESS and np.all(np.isnan(x)), (nrhs, nxs, device)
            assert s.info()["launches_solve"] == 0 and s.info()["ms_solve_gpu"] == 0.0
    # a zero b (nbi = 0): zero entries
    x = sps(s, np.zeros(0, np.int32), np.zeros((2, 0)), one, False)
    assert np.array_equal(x, np.zeros((2, 1)))
    s.close()


# ---- 4. pruning and launch counts -------------------------------------------------------------------------------------
def run_set_launches(run_set, tree, dfront):
    """(d, t) of a run set: the levels that hold a direct front of it, 1 if it has a front above them"""
    return len({int(tree.level[f]) for f in run_set if dfront[f]}), int(any(not dfront[f] for f in run_set))


@pytest.mark.gpu
@pytest.mark.parametrize("direct", ["0", "2"])
def test_pruning_and_launch_counts(direct, monkeypatch):
    monkeypatch.setenv("B200_SOLVE_DIRECT", direct)
    s = factored(*large())
    tree = Tree(s)
    dfront = tree.direct(int(direct))
    var = s.enquire_indef()[0]
    n = s.dim
    rng = np.random.default_rng(3)
    L_off = s.symbolic("L_off")
    nnz = np.diff(L_off)
    leaf = np.array([tree.leaf_var(var, 0)], np.int32)
    other_leaf = np.array([tree.leaf_var(var, 7)], np.int32)
    pats = {"leaf": leaf, "ten": rng.choice(n, 10, replace=False).astype(np.int32), "dense": None}
    sels = {"leaf": other_leaf, "root": np.array([root_var(s, tree)], np.int32),
            "ten": rng.choice(n, 10).astype(np.int32), "all": None}
    full = list(range(tree.nsn))
    for pn, bi in pats.items():
        if bi is not None:
            s.sparse_fwd_solve(bi, np.ones(len(bi)))
            sparse_run = s.symbolic("sparse_run_set")
        nbi = n if bi is None else len(bi)
        for xn, xs in sels.items():
            for device in (False, True):
                sps(s, bi, np.ones(nbi), xs, device)
                launches = s.info()["launches_solve"]
                rf, rb = s.symbolic("sparse_solve_fwd_run_set"), s.symbolic("sparse_solve_bwd_run_set")
                assert list(rf) == (full if bi is None else list(sparse_run)), (pn, xn)
                if xs is None:
                    assert list(rb) == full
                else:
                    assert set(tree.reach(xs)) <= set(rb) and list(rb) == sorted(rb), (pn, xn)
                if bi is None and xs is None:
                    d = run_set_launches(full, tree, dfront)[0]
                    assert launches == 4 + 2 * d, (pn, xn, launches)
                else:
                    df, tf = run_set_launches(rf, tree, dfront)
                    db, tb = run_set_launches(rb, tree, dfront)
                    assert launches == 1 + df + tf + 1 + db + tb + 1, (pn, xn, device, launches, df, tf, db, tb)
                assert s.info()["ms_solve_gpu"] > 0.0
        # the sparse forward solve's and the inverse entries' run sets are left as they were
        if bi is not None:
            assert list(s.symbolic("sparse_run_set")) == list(sparse_run)
    sps(s, leaf, np.ones(1), other_leaf, True)
    share_f = nnz[s.symbolic("sparse_solve_fwd_run_set")].sum() / L_off[-1]
    share_b = nnz[s.symbolic("sparse_solve_bwd_run_set")].sum() / L_off[-1]
    print("MEASURED leaf -> leaf: R_f %.4f, R_b %.4f of nnz(L)" % (share_f, share_b))
    assert share_f < 0.15 and share_b < 0.15, (share_f, share_b)
    s.close()


# ---- 5. stale sweep state ---------------------------------------------------------------------------------------------
def stale_round(s, fresh, tree, tag):
    """a sparse solve after each kind of call gives the bits of the same call on a fresh handle; full solves after it
    keep their bits"""
    n = s.dim
    rng = np.random.default_rng(21)
    var = s.enquire_indef()[0]
    leaf_a, leaf_b = tree.leaf_var(var, 0), tree.leaf_var(var, 5)
    calls = {"leaf->leaf": (np.array([leaf_a], np.int32), np.array([[0.75]]), np.array([leaf_b], np.int32)),
             "fifty->root": (rng.choice(n, min(50, n), replace=False).astype(np.int32),
                             rng.standard_normal((2, min(50, n))), np.array([root_var(s, tree)], np.int32)),
             "leaf->all": (np.array([leaf_b], np.int32), np.array([[-2.0]]), None),
             "dense->five": (None, rng.standard_normal((1, n)), rng.choice(n, min(5, n)).astype(np.int32))}
    want = {k: [sps(fresh, bi, B, xs, d) for d in (False, True)] for k, (bi, B, xs) in calls.items()}
    rhs = rng.standard_normal((8, n))
    x_full = rhs[0].copy()
    assert fresh.solve(x_full, 1) == SYMSOLVER_SUCCESS
    before = {
        "full solve": lambda: s.solve(rhs[0].copy(), 1),
        "job 1": lambda: run(s, 1, rhs[:1], True),
        "job 3": lambda: run(s, 3, rhs[:1], True),
        "blocked nrhs=8": lambda: run(s, 0, rhs, True),
        "lmultiply": lambda: lmul(s, 0, rhs[:1], True),
        "sparse fwd": lambda: sfs(s, np.array([leaf_a], np.int32), np.array([1.0]), True),
        "inverse entries": lambda: s.inverse_entries(np.array([leaf_a, leaf_b]), np.array([leaf_b, leaf_b])),
    }
    for what, op in before.items():
        for k, (bi, B, xs) in calls.items():
            for d in (False, True):
                op()
                assert_bits(sps(s, bi, B, xs, d), want[k][d], (tag, what, k, d))
                xs_ = rhs[0].copy()
                assert s.solve(xs_, 1) == SYMSOLVER_SUCCESS
                assert_bits(xs_, x_full, (tag, what, k, d, "full solve after"))


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random", "mbndry400"])
def test_stale_state_and_refactor(system):
    args = ALL_SYSTEMS[system]()
    s, fresh = factored(*args), factored(*args)
    stale_round(s, fresh, Tree(s), system)
    for h in (s, fresh):
        assert h.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    stale_round(s, fresh, Tree(s), (system, "refactor"))
    s.close()
    fresh.close()


@pytest.mark.gpu
def test_stale_state_after_reanalysis_by_increase_quality():
    s, fresh = factored(*lifted()), factored(*lifted())
    assert s.info()["num_forced"] > 0
    stale_round(s, fresh, Tree(s), "before")
    for h in (s, fresh):
        assert h.IncreaseQuality()
        assert h.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    tree = Tree(s)
    stale_round(s, fresh, tree, "reanalysed")
    sels = selections(s, tree, 2)
    for name, (bi, bv) in b_patterns(s, tree, 3).items():
        check_against_job0(s, bi, bv, sels, ("reanalysed", name))
    s.close()
    fresh.close()


# ---- 6. other factor states: D^+, lifted pivots, altered D -------------------------------------------------------------
@pytest.mark.gpu
def test_other_factor_states():
    # kept singular factors: job 0 is the D^+ solve
    dim, irn, jcn, val, rows = zeroed("MBndryCntrl1_30", 2)
    s, st, _ = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR
    tree = Tree(s)
    sels = selections(s, tree, 8)
    sels["zero rows"] = np.asarray(rows, np.int32)
    for name, (bi, bv) in b_patterns(s, tree, 9).items():
        check_against_job0(s, bi, bv, sels, ("D+", name))
    s.close()
    # lifted pivots (num_forced > 0): the perturbed matrix
    s = factored(*lifted())
    assert s.info()["num_forced"] > 0
    tree = Tree(s)
    sels = selections(s, tree, 10)
    for name, (bi, bv) in b_patterns(s, tree, 12).items():
        check_against_job0(s, bi, bv, sels, ("lifted", name))
    s.close()
    # altered D
    s = factored(*SYSTEMS["MBndryCntrl1_30"]())
    x0 = sps(s, np.array([4, 9], np.int32), np.array([[1.0, 2.0]]), None, False)
    assert s.alter_d(2.0 * s.enquire_indef()[2]) == SYMSOLVER_SUCCESS
    tree = Tree(s)
    sels = selections(s, tree, 13)
    for name, (bi, bv) in b_patterns(s, tree, 14).items():
        check_against_job0(s, bi, bv, sels, ("altered D", name))
    assert not np.array_equal(sps(s, np.array([4, 9], np.int32), np.array([[1.0, 2.0]]), None, False), x0)
    s.close()


# ---- 7. refusals ------------------------------------------------------------------------------------------------------
def assert_refused(s, msg, nrhs, nbi, bindex, b, nxs, xsel):
    for device in (False, True):
        before = s.info()["launches_solve"]
        st, x = raw_call(s, nrhs, nbi, bindex, b, nxs, xsel, device)
        assert st == SYMSOLVER_FATAL_ERROR and "sparse_solve: " in s.last_error() and msg in s.last_error(), \
            (msg, device, st, s.last_error())
        assert np.all(np.isnan(x)), (msg, device)
        assert s.info()["launches_solve"] == before, (msg, device)


@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    one, two = np.array([3], np.int32), np.array([4, 9], np.int32)
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    assert_refused(s, "no factors", 1, 1, one, [1.0], 1, one)
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    assert_refused(s, "nrhs", -1, 1, one, [1.0], 1, one)
    assert_refused(s, "nbi", 1, -1, one, [1.0], 1, one)
    assert_refused(s, "nbi", 1, dim + 1, np.arange(dim + 1), np.ones(dim + 1), 1, one)
    assert_refused(s, "nxs", 1, 1, one, [1.0], -1, one)
    assert_refused(s, "NULL", 1, 1, one, None, 1, one)
    st, x = raw_call(s, 1, 1, one, [1.0], 1, one, False)
    assert st == SYMSOLVER_SUCCESS
    L = s._L
    for device in (False, True):   # a NULL x
        f = L.b200ldlt_sparse_solve_device if device else L.b200ldlt_sparse_solve
        bv = np.ones(1)
        st = f(s._h, 1, 1, one.ctypes.data_as(C.POINTER(C.c_int)), bv.ctypes.data_as(C.POINTER(C.c_double)), 1,
               one.ctypes.data_as(C.POINTER(C.c_int)), None)
        assert st == SYMSOLVER_FATAL_ERROR and "NULL" in s.last_error()
    assert_refused(s, "bindex", 1, 5, None, np.ones(5), 1, one)
    assert_refused(s, "xsel", 1, 1, one, [1.0], 5, None)
    assert_refused(s, "out of range", 1, 2, np.array([0, -1]), [1.0, 2.0], 1, one)
    assert_refused(s, "out of range", 1, 2, np.array([dim, 0]), [1.0, 2.0], 1, one)
    assert_refused(s, "out of range", 1, 1, one, [1.0], 2, np.array([0, dim]))
    assert_refused(s, "out of range", 1, 1, one, [1.0], 1, np.array([-1]))
    assert_refused(s, "twice", 1, 3, np.array([4, 9, 4]), [1.0, 2.0, 3.0], 1, one)
    # the handle is intact after refusals
    tree = Tree(s)
    check_against_job0(s, two, np.array([1.0, 2.0]), {"two": two, "all": None}, "after refusals")
    # no factors after a SINGULAR factorisation outside keep mode
    v0 = val.copy()
    r = int(irn[0])
    v0[(irn == r) | (jcn == r)] = 0.0
    s.GetValuesArrayPtr()[:] = v0
    assert s.factor(False, 0)[0] == SYMSOLVER_SINGULAR
    assert_refused(s, "no factors", 1, 1, one, [1.0], 1, one)
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    assert_refused(s, "sharded", 1, 1, one, [1.0], 1, one)
    s.close()
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    assert s.set_schur(np.array([0, 1, 2], np.int32)) == SYMSOLVER_SUCCESS, s.last_error()
    s.GetValuesArrayPtr()[:] = val
    s.factor(False, 0)
    assert_refused(s, "Schur mode", 1, 1, one, [1.0], 1, one)
    s.close()
