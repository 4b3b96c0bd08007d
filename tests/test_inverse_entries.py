"""Entries of A^-1 at chosen positions (b200ldlt_inverse_entries / _device): M_ij = y_i^T D^-1 y_j with
y_k = L^-1 P^T S e_k, swept by pruned forward sweeps of blocks of unit columns and reduced on the device in a pinned
order.  Checked against a float64 replay of that order on y from sparse_fwd_solve and D^-1 from enquire_indef (exact),
against job 0, numpy and selected inversion (to rounding), and for the bit properties the header promises."""
import ctypes as C
import functools

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt, to_scipy

from test_fredholm import handle, zeroed
from test_partial_solve import SYSTEMS, assert_bits, factored, run
from test_sparse_fwd_solve import BLOCK_TOL, Tree

NEW_SYMBOLS = ["b200ldlt_inverse_entries", "b200ldlt_inverse_entries_device"]
SELINV_TOL = 1e-11   # the selected-inversion tests' bound, relative to the column max-norm


@functools.lru_cache(maxsize=None)
def large():
    return mbndry_kkt(400)[:4]


ALL_SYSTEMS = dict(SYSTEMS, mbndry400=large)
ENVS = [{}, {"B200_SOLVE_DIRECT": "0"}, {"B200_SOLVE_DIRECT": "1"}, {"B200_SOLVE_DIRECT": "4"},
        {"B200_SOLVE_NOPAIR": "1"}, {"B200_SOLVE_BLOCK": "1"}, {"B200_SOLVE_BLOCK": "3"}]
ENV_IDS = ["default", "direct0", "direct1", "direct4", "nopair", "block1", "block3"]


def entries(s, irow, jcol, device):
    irow, jcol = np.asarray(irow, np.int32), np.asarray(jcol, np.int32)
    if device:
        import torch
        d = torch.full((max(len(irow), 1),), np.nan, dtype=torch.float64, device="cuda")
        assert s.inverse_entries_device(irow, jcol, d.data_ptr()) == SYMSOLVER_SUCCESS, s.last_error()
        return d[:len(irow)].cpu().numpy()
    return s.inverse_entries(irow, jcol)


def replay(s, irow, jcol):
    """the documented summation order in float64 on the host, on y from sparse_fwd_solve and D^-1 from enquire_indef"""
    _, ty, dinv2 = s.enquire_indef()
    ys = {}
    for k in set(map(int, irow)) | set(map(int, jcol)):
        ys[k] = s.sparse_fwd_solve(np.array([k], np.int32), np.array([1.0]))
    out = np.zeros(len(irow))
    for t, (i, j) in enumerate(zip(irow, jcol)):
        (pi, ya), (pj, yb) = ys[int(i)], ys[int(j)]
        m = len(np.intersect1d(pi, pj))
        assert np.array_equal(pi[len(pi) - m:], pj[len(pj) - m:]), "the common part is a suffix"
        p, a, b = pi[len(pi) - m:], ya[len(ya) - m:], yb[len(yb) - m:]
        lane = [0.0] * 32
        for o in range(m):
            q = int(p[o])
            if ty[q] == 1:
                term = float(dinv2[q, 0]) * (float(a[o]) * float(b[o]))
            elif ty[q] == 2:
                a1, a2, b1, b2 = float(a[o]), float(a[o + 1]), float(b[o]), float(b[o + 1])
                dd = float(dinv2[q, 0]) * (a1 * b1) + float(dinv2[q + 1, 0]) * (a2 * b2)
                term = dd + float(dinv2[q, 1]) * ((a1 * b2) + (a2 * b1))
            else:
                continue
            lane[o % 32] = lane[o % 32] + term
        for k in (16, 8, 4, 2, 1):
            lane = [lane[l] + lane[l ^ k] for l in range(32)]
        out[t] = lane[0]
    return out


def job0_block(s, idx):
    """M[idx, idx] from job 0 on the unit columns (blocked)"""
    X = np.zeros((len(idx), s.dim))
    X[np.arange(len(idx)), idx] = 1.0
    X = X.ravel()
    assert s.solve(X, len(idx)) == SYMSOLVER_SUCCESS, s.last_error()
    return X.reshape(len(idx), s.dim)[:, idx].T


def entry_sets(s, tree, seed):
    """one entry, random diagonals, a random 16 x 16 block (both triangles), leaf / mid-tree / root fronts, repeats"""
    n = s.dim
    rng = np.random.default_rng(seed)
    var = s.enquire_indef()[0]
    leaves = [f for f in range(tree.nsn) if not tree.children[f]]
    roots = [f for f in range(tree.nsn) if tree.sn_parent[f] < 0]
    root = max(roots, key=lambda f: tree.k[f])
    half = int(tree.level.max()) // 2
    mids = sorted((f for f in range(tree.nsn) if tree.children[f]), key=lambda f: (abs(int(tree.level[f]) - half), f))[:3]
    fr = leaves[:: max(1, len(leaves) // 3)][:3] + mids + [root]
    tv = np.unique([int(var[tree.sn_start[f]]) for f in fr] + [int(var[tree.sn_start[f + 1] - 1]) for f in fr])
    blk = rng.choice(n, min(16, n), replace=False)
    bi, bj = np.meshgrid(blk, blk, indexing="ij")
    d = rng.choice(n, min(20, n), replace=False)
    ti, tj = np.meshgrid(tv, tv, indexing="ij")
    rep = np.array([blk[0], blk[1], blk[0], blk[1], blk[0]]), np.array([blk[1], blk[0], blk[1], blk[1], blk[1]])
    return {"one": (d[:1], d[1:2] if n > 1 else d[:1]), "diag": (d, d), "block16": (bi.ravel(), bj.ravel()),
            "tree": (ti.ravel(), tj.ravel()), "repeats": rep}


def check_set(s, irow, jcol, tag, exact=True):
    v = entries(s, irow, jcol, False)
    if exact:
        assert np.array_equal(v, replay(s, irow, jcol)), (tag, "replay")
    assert_bits(entries(s, irow, jcol, True), v, (tag, "host = device"))
    assert_bits(entries(s, irow, jcol, False), v, (tag, "repeat call"))
    assert_bits(entries(s, jcol, irow, False), v, (tag, "(j, i) = (i, j)"))
    # against job 0 on the unit columns: 1e-12 of the block's max-norm
    idx = np.unique(np.concatenate([irow, jcol]))
    Mb = job0_block(s, idx)
    pos = {int(k): q for q, k in enumerate(idx)}
    ref = np.array([Mb[pos[int(i)], pos[int(j)]] for i, j in zip(irow, jcol)])
    scale = max(np.abs(Mb).max(), 1e-300)
    err = np.abs(v - ref).max() / scale
    assert err <= BLOCK_TOL, (tag, err)
    return v


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


# ---- 1. + 2. + 3. exact replay, job 0, bit properties ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("env", ENVS, ids=ENV_IDS)
@pytest.mark.parametrize("system", sorted(ALL_SYSTEMS))
def test_replay_and_job0(system, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    s = factored(*ALL_SYSTEMS[system]())
    tree = Tree(s)
    for name, (i, j) in entry_sets(s, tree, 5).items():
        v = check_set(s, i, j, (system, name))
        if name == "repeats":
            assert_bits(v[[0, 2, 4]], np.full(3, v[0]), (system, "repeat entries"))
            assert_bits(v[1], v[0], (system, "(j, i) in one call"))
        if name == "block16":
            # every entry equals the same entry requested alone, as a value
            for t in range(0, len(i), 37):
                assert entries(s, i[t:t + 1], j[t:t + 1], False)[0] == v[t], (system, t)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["hs071_0", "MBndryCntrl1_30", "random"])
def test_numpy_and_selected_inverse(system):
    dim, irn, jcn, val = ALL_SYSTEMS[system]()
    s = factored(dim, irn, jcn, val)
    Minv = np.linalg.inv(to_scipy(dim, irn, jcn, val).toarray())
    rng = np.random.default_rng(3)
    i, j = rng.integers(0, dim, 400), rng.integers(0, dim, 400)
    v = entries(s, i, j, True)
    cm = np.abs(Minv).max(axis=0)
    assert np.all(np.abs(v - Minv[i, j]) <= 1e-10 * cm[j]), system
    diag, vals = s.selected_inverse()
    pi, pj = irn - 1, jcn - 1
    v = entries(s, pi, pj, False)
    assert np.all(np.abs(v - vals) <= SELINV_TOL * cm[pj]), system
    d = entries(s, np.arange(dim), np.arange(dim), False)
    assert np.all(np.abs(d - diag) <= SELINV_TOL * cm), system
    s.close()


def two_components():
    """two copies of MBndryCntrl1_30 side by side (block diagonal): the elimination tree is a forest"""
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    return (2 * dim, np.concatenate([irn, irn + dim]).astype(np.int32), np.concatenate([jcn, jcn + dim]).astype(np.int32),
            np.concatenate([val, val]))


@pytest.mark.gpu
def test_forest_pairs_are_plus_zero():
    s = factored(*two_components())
    tree = Tree(s)
    var = s.enquire_indef()[0]
    roots = [f for f in range(tree.nsn) if tree.sn_parent[f] < 0]
    assert len(roots) > 1, "two components give two trees"

    def leaf_under(r):
        f = r
        while tree.children[f]:
            f = tree.children[f][0]
        return int(var[tree.sn_start[f]])

    a, b = int(var[tree.sn_start[roots[0]]]), int(var[tree.sn_start[roots[-1]]])
    la, lb = leaf_under(roots[0]), leaf_under(roots[-1])
    i, j = np.array([a, la, a, la]), np.array([b, lb, lb, b])
    for device in (False, True):
        assert_bits(entries(s, i, j, device), np.zeros(4), ("+0", device))
    assert job0_block(s, np.array([a, b]))[0, 1] == 0.0
    check_set(s, np.concatenate([i, [a, la]]), np.concatenate([j, [la, la]]), "forest")
    s.close()


@pytest.mark.gpu
def test_value_equal_across_block_widths(monkeypatch):
    args = large()
    rng = np.random.default_rng(17)
    n = args[0]
    blk = rng.choice(n, 32, replace=False)
    i, j = np.tril_indices(32)
    i, j = blk[i], blk[j]
    res = {}
    for w in ("8", "1", "3"):
        monkeypatch.setenv("B200_SOLVE_BLOCK", w)
        s = factored(*args)
        res[w] = entries(s, i, j, False)
        s.close()
    assert np.array_equal(res["8"], res["1"]) and np.array_equal(res["8"], res["3"])


# ---- 4. pruning and launch counts ---------------------------------------------------------------------------------------
def expected_launches(s, tree, dfront, irow, jcol, width):
    pos = tree.pos
    cols = sorted(set(map(int, irow)) | set(map(int, jcol)), key=lambda v: pos[v])
    if len(cols) == 1:
        width = 1
    total = 1
    for c0 in range(0, len(cols), width):
        reach = tree.reach(cols[c0:c0 + width])
        total += 2 + len({int(tree.level[f]) for f in reach if dfront[f]}) + int(any(not dfront[f] for f in reach))
    return total


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{}, {"B200_SOLVE_DIRECT": "0"}, {"B200_SOLVE_BLOCK": "1"}, {"B200_SOLVE_BLOCK": "3"}],
                         ids=["default", "direct0", "block1", "block3"])
def test_pruning_and_launch_counts(env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    s = factored(*large())
    tree = Tree(s)
    dfront = tree.direct(int(env.get("B200_SOLVE_DIRECT", "2")))
    width = int(env.get("B200_SOLVE_BLOCK", "8"))
    var = s.enquire_indef()[0]
    leaf = tree.leaf_var(var)
    s.sparse_fwd_solve(np.array([leaf], np.int32), np.array([1.0]))
    want = s.symbolic("sparse_run_set")
    other = np.array([tree.leaf_var(var, 5)], np.int32)
    s.sparse_fwd_solve(other, np.array([1.0]))
    run_before = s.symbolic("sparse_run_set")
    entries(s, [leaf], [leaf], False)
    assert np.array_equal(s.symbolic("inverse_run_set"), want)
    assert np.array_equal(s.symbolic("sparse_run_set"), run_before), "sparse_run_set untouched"
    assert len(want) < tree.nsn // 4, (len(want), tree.nsn)
    rng = np.random.default_rng(4)
    b12 = rng.choice(s.dim, 12, replace=False)
    ti, tj = np.tril_indices(12)
    sets = {"leaf": ([leaf], [leaf]), "ten": (rng.choice(s.dim, 10, replace=False),) * 2, "block": (b12[ti], b12[tj])}
    for name, (i, j) in sets.items():
        for device in (False, True):
            entries(s, i, j, device)
            info = s.info()
            assert info["launches_solve"] == expected_launches(s, tree, dfront, i, j, width), (name, device, info)
            assert info["ms_solve_gpu"] > 0.0
    v = s.inverse_entries(np.zeros(0, np.int32), np.zeros(0, np.int32))
    assert len(v) == 0 and s.info()["launches_solve"] == 0 and s.info()["ms_solve_gpu"] == 0.0
    s.close()


# ---- 5. other operators: D^+, lifted pivots, altered D ------------------------------------------------------------------
@pytest.mark.gpu
def test_other_operators():
    rng = np.random.default_rng(8)
    # kept singular factors (D^+)
    dim, irn, jcn, val, rows = zeroed("MBndryCntrl1_30", 2)
    s, st, _ = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR
    idx = np.concatenate([rows, rng.choice(dim, 10, replace=False)])
    i, j = np.meshgrid(idx, idx, indexing="ij")
    check_set(s, i.ravel(), j.ravel(), "D+")
    s.close()
    # lifted pivots, before and after the re-analysis by increase_quality
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    s = factored(n, irn, jcn, val)
    assert s.info()["num_forced"] > 0
    idx = rng.choice(n, 12, replace=False)
    i, j = np.meshgrid(idx, idx, indexing="ij")
    for stage in ("lifted", "reanalysed"):
        v = entries(s, i.ravel(), j.ravel(), False)
        assert np.array_equal(v, replay(s, i.ravel(), j.ravel())), stage
        Mb = job0_block(s, np.unique(idx))
        # (ill-conditioned: the same 1e-5 bound as the selected-inversion test of this matrix)
        srt = np.searchsorted(np.unique(idx), idx)
        assert np.abs(v.reshape(12, 12) - Mb[np.ix_(srt, srt)]).max() <= 1e-5 * np.abs(Mb).max(), stage
        if stage == "lifted":
            assert s.IncreaseQuality()
            assert s.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    s.close()
    # altered D
    s = factored(*SYSTEMS["MBndryCntrl1_30"]())
    dinv = s.enquire_indef()[2]
    assert s.alter_d(2.0 * dinv) == SYMSOLVER_SUCCESS
    idx = rng.choice(s.dim, 12, replace=False)
    i, j = np.meshgrid(idx, idx, indexing="ij")
    check_set(s, i.ravel(), j.ravel(), "altered D")
    s.close()


# ---- 6. nothing else changes ------------------------------------------------------------------------------------------
def others(s, rhs):
    out = [run(s, 0, rhs[:1], True), run(s, 1, rhs[:1], True), run(s, 0, rhs, True), run(s, 0, rhs, False)]
    bi = np.array([3, 17], np.int32)
    out += list(s.sparse_fwd_solve(bi, np.array([1.0, -2.0])))
    out.append(s.symbolic("sparse_run_set"))
    return out


def same_as_fresh(s, fresh, rhs, tag):
    for a, b in zip(others(s, rhs), others(fresh, rhs)):
        assert_bits(np.asarray(a, np.float64), np.asarray(b, np.float64), tag)


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "mbndry400"])
def test_no_side_effects(system):
    args = ALL_SYSTEMS[system]()
    s, fresh = factored(*args), factored(*args)
    rng = np.random.default_rng(2)
    rhs = rng.standard_normal((5, s.dim))
    i, j = rng.choice(s.dim, 40), rng.choice(s.dim, 40)
    s.sparse_fwd_solve(np.array([3, 17], np.int32), np.array([1.0, -2.0]))
    entries(s, i, j, False)
    entries(s, i, j, True)
    same_as_fresh(s, fresh, rhs, (system, "after"))
    for h in (s, fresh):
        assert h.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    entries(s, i, j, False)
    same_as_fresh(s, fresh, rhs, (system, "refactor"))
    s.close()
    fresh.close()


@pytest.mark.gpu
def test_no_side_effects_after_reanalysis():
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    s, fresh = factored(n, irn, jcn, val), factored(n, irn, jcn, val)
    rng = np.random.default_rng(6)
    rhs = rng.standard_normal((3, n))
    i, j = rng.choice(n, 30), rng.choice(n, 30)
    entries(s, i, j, False)
    for h in (s, fresh):
        assert h.IncreaseQuality()
        assert h.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    v = entries(s, i, j, False)
    assert np.array_equal(v, replay(s, i, j))
    same_as_fresh(s, fresh, rhs, "reanalysed")
    s.close()
    fresh.close()


# ---- 7. refusals ------------------------------------------------------------------------------------------------------
def raw(s, nent, irow, jcol, device):
    L = s._L
    ip = C.POINTER(C.c_int)
    ia = None if irow is None else np.ascontiguousarray(irow, np.int32)
    ja = None if jcol is None else np.ascontiguousarray(jcol, np.int32)
    pi = None if ia is None else ia.ctypes.data_as(ip)
    pj = None if ja is None else ja.ctypes.data_as(ip)
    if device:
        import torch
        d = torch.full((8,), 42.0, dtype=torch.float64, device="cuda")
        st = L.b200ldlt_inverse_entries_device(s._h, nent, pi, pj, C.c_void_p(d.data_ptr()))
        return st, d.cpu().numpy()
    v = np.full(8, 42.0)
    st = L.b200ldlt_inverse_entries(s._h, nent, pi, pj, v.ctypes.data_as(C.POINTER(C.c_double)))
    return st, v


def assert_refused(s, nent, irow, jcol, msg):
    for device in (False, True):
        before = s.info()["launches_solve"]
        st, v = raw(s, nent, irow, jcol, device)
        assert st == SYMSOLVER_FATAL_ERROR and msg in s.last_error(), (msg, device, st, s.last_error())
        assert np.all(v == 42.0), (msg, device)
        assert s.info()["launches_solve"] == before, (msg, device)


@pytest.mark.gpu
def test_refusals():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    one = np.array([3], np.int32)
    assert_refused(s, 1, one, one, "no factors")
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    entries(s, one, one, False)
    assert_refused(s, -1, one, one, "nent")
    assert_refused(s, 1, None, one, "NULL")
    assert_refused(s, 1, one, None, "NULL")
    assert_refused(s, 2, np.array([0, -1]), np.array([0, 0]), "out of range")
    assert_refused(s, 2, np.array([0, 1]), np.array([dim, 0]), "out of range")
    for device in (False, True):
        st, v = raw(s, 0, None, None, device)
        assert st == SYMSOLVER_SUCCESS and np.all(v == 42.0) and s.info()["launches_solve"] == 0
    check_set(s, np.array([4, 9]), np.array([9, 9]), "after refusals")
    L = s._L
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    assert_refused(s, 1, one, one, "sharded")
    s.close()
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    assert s.set_schur(np.array([0, 1, 2], np.int32)) == SYMSOLVER_SUCCESS, s.last_error()
    s.GetValuesArrayPtr()[:] = val
    s.factor(False, 0)
    assert_refused(s, 1, one, one, "Schur mode")
    s.close()
