"""Tensor-core Schur complement (wgmma int8 Ozaki split, ipopt_b200/csrc/schur_tc.cu) against the FP64 DFMA kernel and
against numpy, on a matrix whose elimination tree is two dense children under one dense root, so the contribution block
of a child IS the quantity under test:  CB = - A21 A11^-1 A12  (r x r, lower triangle)."""
import ctypes as C

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_SUCCESS
from ipopt_b200.sharded import _DevArr

pytestmark = pytest.mark.gpu


def arrow_matrix(kb, r, seed):
    """[[D1, 0, B1^T], [0, D2, B2^T], [B1, B2, D3]]: SPD, D1/D2 dense kb x kb, D3 dense r x r (lower triplets, 1-based)."""
    rng = np.random.default_rng(seed)
    n = 2 * kb + r
    A = np.zeros((n, n))
    for b in range(2):
        M = rng.standard_normal((kb, kb))
        A[b * kb:(b + 1) * kb, b * kb:(b + 1) * kb] = M @ M.T + kb * np.eye(kb)
        A[2 * kb:, b * kb:(b + 1) * kb] = rng.standard_normal((r, kb)) * np.exp(rng.uniform(-2, 2, (r, 1)))
    M = rng.standard_normal((r, r))
    A[2 * kb:, 2 * kb:] = M @ M.T + 50.0 * r * np.eye(r)
    A = np.tril(A) + np.tril(A, -1).T
    i, j = np.nonzero(np.tril(A))
    return n, A, (i + 1).astype(np.int32), (j + 1).astype(np.int32), A[i, j]


def factor_and_cb(n, irn, jcn, val, tc_min_r):
    import torch
    s = B200Ldlt(ordering=1, pair_saddle=0, scaling=0, tc_schur_min_r=tc_min_r)
    assert s.InitializeStructure(n, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, 0)
    assert st == SYMSOLVER_SUCCESS and neg == 0, s.info()
    L = s._L
    L.b200ldlt_device_ptr.restype = C.c_void_p
    L.b200ldlt_device_ptr.argtypes = [C.c_void_p, C.c_char_p]
    cb_off = s.symbolic("cb_off")
    sn_start, rows_ptr = s.symbolic("sn_start"), s.symbolic("rows_ptr")
    ptr = L.b200ldlt_device_ptr(s._h, b"CB")
    cb = torch.as_tensor(_DevArr(ptr, int(cb_off[-1]), "<f8"), device="cuda").cpu().numpy().copy()
    return s, cb, cb_off, sn_start, rows_ptr


@pytest.mark.parametrize("kb,r", [(96, 256), (300, 700), (130, 513)])
def test_tc_schur_matches_dfma_and_numpy(kb, r):
    n, A, irn, jcn, val = arrow_matrix(kb, r, seed=kb + r)
    s0, cb0, cb_off, sn_start, rows_ptr = factor_and_cb(n, irn, jcn, val, 0)       # FP64 DFMA tiles
    s1, cb1, _, _, _ = factor_and_cb(n, irn, jcn, val, 128)                        # tensor cores for r >= 128
    nsn = len(sn_start) - 1
    checked = 0
    for q in range(nsn):
        k = int(sn_start[q + 1] - sn_start[q]); rr = int(rows_ptr[q + 1] - rows_ptr[q])
        if rr < 128 or k < 32:
            continue
        c0 = cb0[cb_off[q]:cb_off[q] + rr * rr].reshape(rr, rr).T   # column-major r x r
        c1 = cb1[cb_off[q]:cb_off[q] + rr * rr].reshape(rr, rr).T
        lo = np.tril_indices(rr)
        cols = np.arange(sn_start[q], sn_start[q + 1])
        ref = -A[2 * kb:, cols] @ np.linalg.solve(A[np.ix_(cols, cols)], A[cols, 2 * kb:])
        scale = np.abs(ref).max()
        assert np.abs(c0[lo] - ref[lo]).max() <= 1e-11 * scale            # both are right ...
        assert np.abs(c1[lo] - ref[lo]).max() <= 1e-11 * scale
        assert np.abs(c1[lo] - c0[lo]).max() <= 1e-13 * scale, (q, np.abs(c1[lo] - c0[lo]).max() / scale)   # ... and agree to FP64 GEMM accuracy
        checked += 1
    assert checked >= 1   # (the second child may be amalgamated into the root)
    b = np.random.default_rng(0).standard_normal(n)
    x0, x1 = b.copy(), b.copy()
    s0.solve(x0); s1.solve(x1)
    xr = np.linalg.solve(A, b)
    assert np.linalg.norm(x1 - xr) <= 1e-10 * np.linalg.norm(xr) and np.linalg.norm(x0 - xr) <= 1e-10 * np.linalg.norm(xr)
    s0.close(); s1.close()


def test_tc_schur_full_size_equivalence():
    """MBndryCntrl1-shaped KKT, N=200: same inertia and solution with the Schur complements of the fronts with r >= 256 on
    the tensor cores."""
    from ipopt_b200.kkt import mbndry_kkt
    dim, irn, jcn, val, nc = mbndry_kkt(200, sigma_spread=3.0, seed=1)
    b = np.random.default_rng(1).standard_normal(dim)
    xs = []
    for tc in (0, 256):
        s = B200Ldlt(tc_schur_min_r=tc)
        s.InitializeStructure(dim, len(irn), irn, jcn)
        s.GetValuesArrayPtr()[:] = val
        st, neg = s.factor(True, nc)
        assert st == SYMSOLVER_SUCCESS and neg == nc
        x = b.copy(); s.solve(x); xs.append(x)
        r, xi, bi = s.residual(x, b)
        assert r <= 1e-9 * (xi * 4.0 + bi)
        s.close()
    assert np.linalg.norm(xs[0] - xs[1]) <= 1e-7 * np.linalg.norm(xs[0])
