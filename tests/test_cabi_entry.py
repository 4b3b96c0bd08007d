"""The rules the C ABI calls that read the factors share (include/b200ldlt.h, head of the partial-solves section): one
pinned staging for the host columns of solve, solve_partial, lmultiply and solve_fredholm, the empty-call rule, the
"<call>: " refusal messages, and the same launch count from both entry points."""
import ctypes as C

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt

from test_fredholm import fred, handle, zeroed
from test_lmultiply_alter import lmul
from test_partial_solve import SYSTEMS, assert_bits, factored, run

dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
M70 = lambda: mbndry_kkt(70, sigma_spread=3.0, seed=5)[:4]   # noqa: E731  (n = 10080: the staging copies run in chunks)


def kept_singular():
    """MBndryCntrl1_30 with two zeroed variables, factors kept: solve_fredholm takes its zero-pivot path"""
    dim, irn, jcn, val, rows = zeroed("MBndryCntrl1_30", 2)
    s, st, _ = handle(dim, irn, jcn, val)
    assert st == SYMSOLVER_SINGULAR and len(s.enquire_zero_pivots()) == 2
    return s


def counters(s):
    i = s.info()
    return i["launches_solve"], i["ms_solve_gpu"]


def call(s, kind, B, device, arg):
    """one call of `kind` on the columns of B (nrhs x dim); returns (outputs, launches_solve)"""
    if kind == "solve":
        if device:
            out = run(s, 0, B, True)
        else:
            out = B.ravel().copy()
            assert s.solve(out, B.shape[0]) == SYMSOLVER_SUCCESS, s.last_error()
        out = [out]
    elif kind == "partial":
        out = [run(s, arg, B, device)]
    elif kind == "lmultiply":
        out = [lmul(s, arg, B, device)]
    else:
        X, F, c = fred(s, B, 1e-10, device)
        out = [X, F, c.astype(np.float64)]
    launches, ms = counters(s)
    assert launches > 0 and ms > 0.0, (kind, device, launches, ms)
    return out, launches


# ---- 1. one staging for every host call ----------------------------------------------------------------------------
SEQUENCE = [("solve", 1, None), ("fredholm", 5, None), ("lmultiply", 9, 1), ("partial", 2, 3), ("solve", 12, None),
            ("fredholm", 1, None), ("lmultiply", 3, 0), ("partial", 7, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "1"])
@pytest.mark.parametrize("system", ["mbndry70", "kept_singular"])
def test_shared_staging_interleaved(system, block, monkeypatch):
    """host calls of all four staged kinds, widths growing and shrinking (Fredholm writes twice the columns it reads):
    every host result bit-equal to the device entry point on the same input, with the same launch count"""
    if block:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*M70()) if system == "mbndry70" else kept_singular()
    rng = np.random.default_rng(11)
    for rep in range(2):
        for kind, nrhs, arg in SEQUENCE:
            B = rng.standard_normal((nrhs, s.dim))
            host, lh = call(s, kind, B, False, arg)
            dev, ld = call(s, kind, B, True, arg)
            tag = (rep, kind, nrhs, arg)
            assert lh == ld, tag
            for a, b in zip(host, dev):
                assert_bits(a, b, tag)
    s.close()


# ---- 2. calls without columns ----------------------------------------------------------------------------------------
def device_array(values):
    import torch
    return torch.tensor(np.asarray(values, np.float64).ravel(), device="cuda")


@pytest.mark.gpu
def test_calls_without_columns():
    """after a call with columns, a call without: success, launches_solve = ms_solve_gpu = 0, outputs untouched"""
    s = factored(*SYSTEMS["MBndryCntrl1_30"]())
    L, h, n = s._L, s._h, s.dim
    B = np.random.default_rng(2).standard_normal((2, n))
    sentinel = np.full(2 * n, 42.0)
    xi_sentinel = np.full(n, 99, np.int32)
    one = np.array([7], np.int32)

    def empty(tag, fn):
        before = counters(s)
        assert before[0] > 0 and before[1] > 0.0, tag
        x, xi, cons, nxi = sentinel.copy(), xi_sentinel.copy(), np.full(1, -1, np.int32), C.c_int(-7)
        dx = device_array(sentinel)
        st = fn(x.ctypes.data_as(dp), C.c_void_p(dx.data_ptr()), xi.ctypes.data_as(ip), cons.ctypes.data_as(ip), nxi)
        assert st == SYMSOLVER_SUCCESS, (tag, s.last_error())
        assert counters(s) == (0, 0.0), (tag, counters(s))
        assert_bits(x, sentinel, tag)
        assert_bits(dx.cpu().numpy(), sentinel, tag)
        assert np.array_equal(xi, xi_sentinel) and cons[0] == -1, tag
        return nxi.value

    for nrhs in (0, -1):
        run(s, 0, B, False)
        empty(("solve", nrhs), lambda x, dx, xi, c, nxi: L.b200ldlt_solve(h, nrhs, x))
        run(s, 0, B, True)
        empty(("solve_device", nrhs), lambda x, dx, xi, c, nxi: L.b200ldlt_solve_device(h, nrhs, dx))
        for job in (1, 2, 3, 4):
            run(s, job, B, False)
            empty(("solve_partial", job, nrhs), lambda x, dx, xi, c, nxi: L.b200ldlt_solve_partial(h, job, nrhs, x))
            run(s, job, B, True)
            empty(("solve_partial_device", job, nrhs),
                  lambda x, dx, xi, c, nxi: L.b200ldlt_solve_partial_device(h, job, nrhs, dx))
        for trans in (0, 1):
            lmul(s, trans, B, False)
            empty(("lmultiply", trans, nrhs), lambda x, dx, xi, c, nxi: L.b200ldlt_lmultiply(h, trans, nrhs, x, x))
            lmul(s, trans, B, True)
            empty(("lmultiply_device", trans, nrhs),
                  lambda x, dx, xi, c, nxi: L.b200ldlt_lmultiply_device(h, trans, nrhs, dx, dx))
    fred(s, B, 0.0, False)
    empty("solve_fredholm", lambda x, dx, xi, c, nxi: L.b200ldlt_solve_fredholm(h, 0, 0.0, x, c))
    fred(s, B, 0.0, True)
    empty("solve_fredholm_device", lambda x, dx, xi, c, nxi: L.b200ldlt_solve_fredholm_device(h, 0, 0.0, dx, c))
    s.sparse_fwd_solve(one, [1.0])
    assert empty("sparse_fwd_solve", lambda x, dx, xi, c, nxi: L.b200ldlt_sparse_fwd_solve(
        h, 0, one.ctypes.data_as(ip), x, C.byref(nxi), xi, x)) == 0
    db, dxs = device_array([1.0]), device_array(sentinel)
    s.sparse_fwd_solve_device(one, db.data_ptr(), dxs.data_ptr())
    assert empty("sparse_fwd_solve_device", lambda x, dx, xi, c, nxi: L.b200ldlt_sparse_fwd_solve_device(
        h, 0, one.ctypes.data_as(ip), dx, C.byref(nxi), xi, dx)) == 0
    s.close()


# ---- 3. refusal messages -------------------------------------------------------------------------------------------
class Calls:
    """every call that reads the factors, on valid arguments of one column, by the name its messages start with"""

    def __init__(self, s):
        self.s, self.L, self.h, n = s, s._L, s._h, s.dim
        self.x, self.d2 = np.ones(2 * n), np.zeros((n, 2))
        self.dx = device_array(np.ones(2 * n))
        self.diag, self.vals = np.zeros(n), np.zeros(s.nonzeros)
        self.xi, self.cons, self.nzero = np.zeros(n, np.int32), np.zeros(1, np.int32), C.c_int(0)
        self.bi = np.array([3], np.int32)

    def all(self):
        L, h, x, dx = self.L, self.h, self.x.ctypes.data_as(dp), C.c_void_p(self.dx.data_ptr())
        xi, nxi, bi = self.xi.ctypes.data_as(ip), C.byref(C.c_int(0)), self.bi.ctypes.data_as(ip)
        return [
            ("solve", lambda: L.b200ldlt_solve(h, 1, x)),
            ("solve", lambda: L.b200ldlt_solve_device(h, 1, dx)),
            ("solve_partial", lambda: L.b200ldlt_solve_partial(h, 3, 1, x)),
            ("solve_partial", lambda: L.b200ldlt_solve_partial_device(h, 1, 1, dx)),
            ("enquire_indef", lambda: L.b200ldlt_enquire_indef(h, xi, None, self.d2.ctypes.data_as(dp))),
            ("lmultiply", lambda: L.b200ldlt_lmultiply(h, 0, 1, x, x)),
            ("lmultiply", lambda: L.b200ldlt_lmultiply_device(h, 1, 1, dx, dx)),
            ("sparse_fwd_solve", lambda: L.b200ldlt_sparse_fwd_solve(h, 1, bi, x, nxi, xi, x)),
            ("sparse_fwd_solve", lambda: L.b200ldlt_sparse_fwd_solve_device(h, 1, bi, dx, nxi, xi, dx)),
            ("alter_d", lambda: L.b200ldlt_alter_d(h, self.d2.ctypes.data_as(dp))),
            ("enquire_zero_pivots", lambda: L.b200ldlt_enquire_zero_pivots(h, C.byref(self.nzero), None)),
            ("solve_fredholm", lambda: L.b200ldlt_solve_fredholm(h, 1, 0.0, x, self.cons.ctypes.data_as(ip))),
            ("solve_fredholm", lambda: L.b200ldlt_solve_fredholm_device(h, 1, 0.0, dx, self.cons.ctypes.data_as(ip))),
            ("selected_inverse", lambda: L.b200ldlt_selected_inverse(h, self.diag.ctypes.data_as(dp),
                                                                      self.vals.ctypes.data_as(dp))),
            ("selected_inverse", lambda: L.b200ldlt_selected_inverse_device(h, dx, None)),
        ]


def refused(s, name, fn, reason):
    assert fn() == SYMSOLVER_FATAL_ERROR, name
    msg = s.last_error()
    assert msg.startswith(name + ": ") and reason in msg, (name, msg)


@pytest.mark.gpu
def test_refusal_messages():
    dim, irn, jcn, val = SYSTEMS["MBndryCntrl1_30"]()
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    calls = Calls(s)
    for name, fn in calls.all():
        refused(s, name, fn, "no factors (factorise first; a SINGULAR factorisation keeps them only in keep mode")
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    calls.d2[:] = s.enquire_indef()[2]
    ok = dict(calls.all())   # (the last call of each name)
    L, h, x = s._L, s._h, calls.x.ctypes.data_as(dp)
    bad = [
        ("solve_partial", lambda: L.b200ldlt_solve_partial(h, 5, 1, x), "job"),
        ("solve_partial", lambda: L.b200ldlt_solve_partial_device(h, -1, 1, None), "job"),
        ("lmultiply", lambda: L.b200ldlt_lmultiply(h, 2, 1, x, x), "trans"),
        ("lmultiply", lambda: L.b200ldlt_lmultiply_device(h, -1, 1, None, None), "trans"),
        ("sparse_fwd_solve", lambda: L.b200ldlt_sparse_fwd_solve(h, -1, None, None, None, None, None), "nbi"),
        ("sparse_fwd_solve", lambda: L.b200ldlt_sparse_fwd_solve_device(h, 1, None, None, None, None, None), "NULL"),
        ("alter_d", lambda: L.b200ldlt_alter_d(h, None), "no entries"),
        ("enquire_zero_pivots", lambda: L.b200ldlt_enquire_zero_pivots(h, None, None), "NULL"),
        ("solve_fredholm", lambda: L.b200ldlt_solve_fredholm(h, -1, 0.0, x, None), "nrhs"),
        ("solve_fredholm", lambda: L.b200ldlt_solve_fredholm_device(h, 1, -1.0, None, None), "tol"),
        ("selected_inverse", lambda: L.b200ldlt_selected_inverse(h, None, None), "NULL"),
        ("selected_inverse", lambda: L.b200ldlt_selected_inverse_device(h, None, None), "NULL"),
    ]
    for name, fn, reason in bad:
        refused(s, name, fn, reason)
        assert ok[name]() == SYMSOLVER_SUCCESS, (name, s.last_error())
    # a sharded handle: solve, enquire_indef and enquire_zero_pivots stay available
    L.b200ldlt_shard_setup.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.b200ldlt_shard_setup(h, 0, 1) == SYMSOLVER_SUCCESS
    for name, fn in calls.all():
        if name in ("solve", "enquire_indef", "enquire_zero_pivots"):
            assert fn() == SYMSOLVER_SUCCESS, (name, s.last_error())
        else:
            refused(s, name, fn, "not available on a sharded handle")
    assert calls.L.b200ldlt_solve_partial(h, 0, 1, x) == SYMSOLVER_SUCCESS   # job 0 is the solve
    s.close()


# ---- 4. the same launch count from both entry points -----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, "3"])
def test_host_and_device_launch_counts_agree(block, monkeypatch):
    if block:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    s = factored(*M70())
    rng = np.random.default_rng(4)
    for nrhs in (1, 5):
        B = rng.standard_normal((nrhs, s.dim))
        for kind, arg in [("solve", None), ("partial", 1), ("partial", 2), ("partial", 3), ("partial", 4),
                          ("lmultiply", 0), ("lmultiply", 1), ("fredholm", None)]:
            assert call(s, kind, B, False, arg)[1] == call(s, kind, B, True, arg)[1], (kind, arg, nrhs)
    import torch
    bi = rng.choice(s.dim, 20, replace=False).astype(np.int32)
    bv = rng.standard_normal(20)
    s.sparse_fwd_solve(bi, bv)
    host = counters(s)[0]
    db, dx = device_array(bv), torch.zeros(s.dim, dtype=torch.float64, device="cuda")
    s.sparse_fwd_solve_device(bi, db.data_ptr(), dx.data_ptr())
    assert counters(s)[0] == host > 0
    s.selected_inverse()
    host = counters(s)[0]
    d = torch.zeros(s.dim, dtype=torch.float64, device="cuda")
    assert s.selected_inverse_device(d.data_ptr(), 0) == SYMSOLVER_SUCCESS
    assert counters(s)[0] == host > 0
    s.close()
