"""Selected inversion (b200ldlt_selected_inverse / _device): the diagonal of M = S P L^-T D^-1 L^-1 P^T S (= A^-1 for a
non-singular factorisation) and M on the pattern of A, checked against job 0 on identity columns, numpy, and the exact
identities the recurrence guarantees."""
import ctypes as C

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt, random_kkt, to_scipy

from test_fredholm import dup_kkt, handle, zeroed
from test_partial_solve import LARGE, SYSTEMS, assert_bits, factored

NEW_SYMBOLS = ["b200ldlt_selected_inverse", "b200ldlt_selected_inverse_device"]
# |selected inverse - job 0| <= TOL * max-norm of the column of M, for every entry compared.  Largest discrepancies
# measured (H100): 5.5e-14 on 55 columns of mbndry_kkt(400), 6.4e-15 on kept singular factors, <= 3.5e-15 on the small
# systems and against numpy; TOL leaves a margin of about 180 over the largest.
TOL = 1e-11


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(built_lib)
    for n in NEW_SYMBOLS:
        assert hasattr(lib, n), n


def job0_columns(s, cols):
    """M[:, c] for c in cols by job 0 (blocked), one row per column"""
    X = np.zeros((len(cols), s.dim))
    X[np.arange(len(cols)), cols] = 1.0
    X = X.ravel()
    assert s.solve(X, len(cols)) == SYMSOLVER_SUCCESS, s.last_error()
    return X.reshape(len(cols), s.dim)


def worst(s, irn, jcn, diag, vals, cols, Mc):
    """max over the entries of the columns cols of |selinv - job 0| / max-norm of the column"""
    where = {c: q for q, c in enumerate(cols)}
    nrm = np.abs(Mc).max(axis=1)
    nrm[nrm == 0] = 1.0           # a zero column of M (D^+ at a zero pivot): absolute difference
    w = 0.0
    for q, c in enumerate(cols):
        w = max(w, abs(diag[c] - Mc[q, c]) / nrm[q])
    i, j = irn - 1, jcn - 1
    for t in range(len(irn)):
        for a, b in ((i[t], j[t]), (j[t], i[t])):
            if b in where:
                q = where[b]
                w = max(w, abs(vals[t] - Mc[q, a]) / nrm[q])
    return w


def selinv_device(s):
    import torch
    d = torch.zeros(s.dim, dtype=torch.float64, device="cuda")
    v = torch.zeros(s.nonzeros, dtype=torch.float64, device="cuda")
    assert s.selected_inverse_device(d.data_ptr(), v.data_ptr()) == SYMSOLVER_SUCCESS, s.last_error()
    return d.cpu().numpy(), v.cpu().numpy()


def check_identities(s, irn, jcn, diag, vals):
    i, j = irn - 1, jcn - 1
    on = i == j
    assert_bits(vals[on], diag[i[on]], "diag triplets")
    key = {}
    for t in range(len(irn)):
        k = (min(i[t], j[t]), max(i[t], j[t]))
        if k in key:
            assert_bits(vals[t:t + 1], vals[key[k]:key[k] + 1], "duplicate / symmetric")
        key[k] = t


# ---- against job 0 (and numpy) on the small systems ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", sorted(SYSTEMS))
def test_small_systems_against_job0(system):
    dim, irn, jcn, val = SYSTEMS[system]()
    s = factored(dim, irn, jcn, val)
    diag, vals = s.selected_inverse()
    cols = np.arange(dim)
    Mc = job0_columns(s, cols)
    w = worst(s, irn, jcn, diag, vals, cols, Mc)
    print("%s: n=%d max |selinv - job0| / column max-norm = %.3e" % (system, dim, w))
    assert w <= TOL, w
    check_identities(s, irn, jcn, diag, vals)
    s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_against_numpy_inverse(seed):
    dim, irn, jcn, val = random_kkt(300, 100, density=0.03, seed=seed)[:4]
    A = to_scipy(dim, irn, jcn, val).toarray()
    assert np.linalg.cond(A) < 1e8
    Ai = np.linalg.inv(A)
    s = factored(dim, irn, jcn, val)
    diag, vals = s.selected_inverse()
    nrm = np.abs(Ai).max(axis=0)
    w = max(np.max(np.abs(diag - np.diag(Ai)) / nrm),
            np.max(np.abs(vals - Ai[irn - 1, jcn - 1]) / nrm[jcn - 1]))
    print("random_kkt seed %d: max |selinv - inv(A)| / column max-norm = %.3e (cond %.1e)" % (seed, w, np.linalg.cond(A)))
    assert w <= TOL, w
    s.close()


# ---- full size: a front of every class ---------------------------------------------------------------------------------
def class_columns(s):
    """original variables of: the root front, a front in each order class, a leaf of level 0, plus random ones (>= 48)"""
    ss, rp = s.symbolic("sn_start"), s.symbolic("rows_ptr")
    perm, lev, par = s.symbolic("perm"), s.symbolic("sn_level"), s.symbolic("sn_parent")
    k, r = np.diff(ss), np.diff(rp)
    f = k + r
    picks = [int(np.flatnonzero(par < 0)[0])]
    for lo, hi in [(1, 32), (33, 64), (65, 96), (97, 256), (257, 1 << 30)]:
        c = np.flatnonzero((f >= lo) & (f <= hi) & (r > 0))
        assert c.size, (lo, hi)
        picks.append(int(c[c.size // 2]))
    picks.append(int(np.flatnonzero(lev == 0)[0]))
    cols = []
    for sn in picks:
        cols += [int(perm[ss[sn]]), int(perm[ss[sn + 1] - 1])]
    rng = np.random.default_rng(7)
    cols += list(rng.choice(s.dim, 48 - len(cols) + 8, replace=False))
    return np.unique(np.array(cols))


@pytest.mark.gpu
def test_full_size_against_job0():
    dim, irn, jcn, val = LARGE()
    s = factored(dim, irn, jcn, val)
    diag, vals = s.selected_inverse()
    cols = class_columns(s)
    assert cols.size >= 48
    Mc = job0_columns(s, cols)
    w = worst(s, irn, jcn, diag, vals, cols, Mc)
    print("mbndry_kkt(400): %d columns, max |selinv - job0| / column max-norm = %.3e" % (cols.size, w))
    assert w <= TOL, w
    check_identities(s, irn, jcn, diag, vals)
    d2, v2 = s.selected_inverse()
    assert_bits(d2, diag, "repeat diag")
    assert_bits(v2, vals, "repeat vals")
    dd, dv = selinv_device(s)
    assert_bits(dd, diag, "device diag")
    assert_bits(dv, vals, "device vals")
    s.close()


# ---- exact identities ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "LukVlE1_1000", "random"])
def test_bitwise_identities(system):
    dim, irn, jcn, val = SYSTEMS[system]()
    # every triplet given again in the other triangle, and the first ten twice more: values split so the sums agree
    irn2 = np.concatenate([irn, jcn, irn[:10]]).astype(np.int32)
    jcn2 = np.concatenate([jcn, irn, jcn[:10]]).astype(np.int32)
    val2 = np.concatenate([val * 0.5, val * 0.5, np.zeros(10)])
    s = factored(dim, irn2, jcn2, val2)
    diag, vals = s.selected_inverse()
    check_identities(s, irn2, jcn2, diag, vals)
    d2, v2 = s.selected_inverse()
    assert_bits(d2, diag)
    assert_bits(v2, vals)
    dd, dv = selinv_device(s)
    assert_bits(dd, diag)
    assert_bits(dv, vals)
    d3, _ = s.selected_inverse(pattern=False)
    _, v3 = s.selected_inverse(diag=False)
    assert_bits(d3, diag)
    assert_bits(v3, vals)
    s.close()


# Every term of the recurrence is linear in D^-1, so D^-1 -> 2 D^-1 doubles every output exactly -- away from overflow
# and subnormals.  Only outputs in the subnormal range (below the smallest normal double, before and after) are exempt:
# on LukVlE1_1000, whose chained Jacobian makes entries of M decay geometrically, 5 diagonal and 17 pattern entries are
# subnormal and differ (the diagonal ones between 0 and 1.7e-310, by 1 ulp; H100); every other output must be bit-exact.
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "LukVlE1_1000", "random"])
def test_alter_d_doubles_exactly(system):
    dim, irn, jcn, val = SYSTEMS[system]()
    s = factored(dim, irn, jcn, val)
    diag, vals = s.selected_inverse()
    var, ty, dinv = s.enquire_indef()
    assert s.alter_d(2.0 * dinv) == SYMSOLVER_SUCCESS
    d4, v4 = s.selected_inverse()
    tiny = np.finfo(np.float64).tiny
    for tag, got, want in (("diag", d4, 2.0 * diag), ("vals", v4, 2.0 * vals)):
        differ = got.view(np.uint64) != want.view(np.uint64)
        subnormal = (np.abs(got) < tiny) & (np.abs(want) < tiny)
        print("%s %s: %d outputs differ from the doubled ones, all subnormal: %s"
              % (system, tag, differ.sum(), bool(subnormal[differ].all())))
        assert not (differ & ~subnormal).any(), (tag, np.flatnonzero(differ & ~subnormal)[:5])
    s.close()


@pytest.mark.gpu
def test_two_handles_interleaved():
    """a handle with large fronts, then one with only small fronts, then the first again: the second plan must not take
    anything the first one's launches need"""
    big = factored(*LARGE())
    d0, v0 = big.selected_inverse()
    small = factored(*SYSTEMS["hs071_0"]())
    ds, vs = small.selected_inverse()
    d1, v1 = big.selected_inverse()
    assert_bits(d1, d0, "big diag")
    assert_bits(v1, v0, "big vals")
    assert_bits(small.selected_inverse()[0], ds, "small diag")
    big.close()
    small.close()


# ---- no side effects -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_no_side_effects():
    dim, irn, jcn, val = LARGE()
    b = np.random.default_rng(9).standard_normal(dim)
    s = factored(dim, irn, jcn, val)
    ref = factored(dim, irn, jcn, val)
    x0 = b.copy()
    assert s.solve(x0) == SYMSOLVER_SUCCESS
    s.selected_inverse()
    x1 = b.copy()
    assert s.solve(x1) == SYMSOLVER_SUCCESS
    assert_bits(x1, x0, "solve after the call")
    # refactor after the call (it reuses CB / W) == a handle that never called it
    assert s.refactor()[0] == SYMSOLVER_SUCCESS
    assert ref.refactor()[0] == SYMSOLVER_SUCCESS
    for a, c in zip(s.enquire_indef(), ref.enquire_indef()):
        assert_bits(a.astype(np.float64), c.astype(np.float64), "factors after refactor")
    x2, x3 = b.copy(), b.copy()
    assert s.solve(x2) == SYMSOLVER_SUCCESS and ref.solve(x3) == SYMSOLVER_SUCCESS
    assert_bits(x2, x3, "solve after refactor")
    s.close()
    ref.close()


@pytest.mark.gpu
def test_after_reanalysis_by_increase_quality():
    """a tridiagonal matrix with lifted pivots: increase_quality schedules a re-analysis, which rebuilds the plan"""
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    s = factored(n, irn, jcn, val)
    assert s.info()["num_forced"] > 0
    # the lifted pivots (D^-1 up to 1/1.5e-8) make M ill-conditioned both before and after the re-analysis: job 0 and
    # the recurrence agree to 2.0e-7 of the column max-norm before it (H100), so this checks the rebuilt plan against
    # job 0 at 1e-5, not at TOL; the other tests hold the accuracy
    cols = np.arange(0, n, 7)
    for stage in ("before", "reanalysed"):
        diag, vals = s.selected_inverse()
        w = worst(s, irn, jcn, diag, vals, cols, job0_columns(s, cols))
        print("lifted-pivot tridiagonal, %s: %.3e" % (stage, w))
        assert w <= 1e-5, (stage, w)
        check_identities(s, irn, jcn, diag, vals)
        if stage == "before":
            assert s.IncreaseQuality()
            assert s.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    s.close()


# ---- singular factors ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "random"])
def test_kept_singular_factors(system):
    dim, irn, jcn, val, rows = zeroed(system, 2)
    s, st, _ = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR
    diag, vals = s.selected_inverse()
    cols = np.arange(dim)
    w = worst(s, irn, jcn, diag, vals, cols, job0_columns(s, cols))
    print("%s, 2 zeroed rows (D^+): max |selinv - job0| / column max-norm = %.3e" % (system, w))
    assert w <= TOL, w
    s.close()


@pytest.mark.gpu
def test_lifted_zero_refused():
    seen = 0
    for (nx, nc, seed) in [(40, 12, 0), (120, 40, 1), (300, 100, 2)]:
        dim, irn, jcn, val, _ = dup_kkt(nx, nc, seed)
        for ordering in (0, 1):
            s, st, _ = handle(dim, irn, jcn, val, ordering=ordering)
            if "lifted zero" in s.last_error():
                seen += 1
                with pytest.raises(RuntimeError, match="no factors"):
                    s.selected_inverse()
            s.close()
    assert seen >= 1


# ---- launch count and refusals -------------------------------------------------------------------------------------
def expected_launches(s):
    ss, rp, lev = s.symbolic("sn_start"), s.symbolic("rows_ptr"), s.symbolic("sn_level")
    k, r = np.diff(ss), np.diff(rp)
    f = k + r
    n = 2
    for l in range(int(lev.max()) + 1):
        m = lev == l
        n += int((r[m] > 0).any()) + int((f[m] <= 96).any()) + int(((f[m] > 96) & (f[m] <= 256)).any())
        n += 2 * int(((f[m] > 96) & (r[m] > 0)).any()) + int((f[m] > 96).any())
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "LukVlE1_1000", "mbndry400"])
def test_launch_count(system):
    dim, irn, jcn, val = LARGE() if system == "mbndry400" else SYSTEMS[system]()
    s = factored(dim, irn, jcn, val)
    s.selected_inverse()
    assert s.info()["launches_solve"] == expected_launches(s)
    s.close()


@pytest.mark.gpu
def test_refusals():
    dp = C.POINTER(C.c_double)
    dim, irn, jcn, val, rows = zeroed("MBndryCntrl1_30", 1)
    s, st, _ = handle(dim, irn, jcn, val, keep=0)
    assert st == SYMSOLVER_SINGULAR
    L = s._L
    d, v = np.full(dim, 3.0), np.full(len(irn), 3.0)
    d0, v0 = d.copy(), v.copy()
    assert L.b200ldlt_selected_inverse(s._h, d.ctypes.data_as(dp), v.ctypes.data_as(dp)) == SYMSOLVER_FATAL_ERROR
    assert "no factors" in s.last_error()
    assert_bits(d, d0)
    assert_bits(v, v0)
    s.close()
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = factored(dim, irn, jcn, val)
    assert L.b200ldlt_selected_inverse(s._h, None, None) == SYMSOLVER_FATAL_ERROR
    assert "NULL" in s.last_error()
    assert s.selected_inverse_device(0, 0) == SYMSOLVER_FATAL_ERROR
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(s._h, 0, 1) == SYMSOLVER_SUCCESS
    d, v = np.full(dim, 3.0), np.full(len(irn), 3.0)
    d0, v0 = d.copy(), v.copy()
    assert L.b200ldlt_selected_inverse(s._h, d.ctypes.data_as(dp), v.ctypes.data_as(dp)) == SYMSOLVER_FATAL_ERROR
    assert "sharded" in s.last_error()
    assert_bits(d, d0)
    assert_bits(v, v0)
    s.close()
