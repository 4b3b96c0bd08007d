"""What the handle holds across a failed analysis: everything an analysis derives is replaced whole, so an analysis that
fails leaves none behind.  The next call that needs one runs it again, and the calls that read the factors find none."""
import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_FATAL_ERROR, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import mbndry_kkt


def handle(dim, irn, jcn, val):
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    return s


def solved(s, b):
    x = b.copy()
    assert s.solve(x) == SYMSOLVER_SUCCESS, s.last_error()
    return x


@pytest.mark.gpu
def test_failed_reanalysis_leaves_the_handle_unanalysed():
    """Schur mode on 70 000 of the 80 800 variables of MBndryCntrl1 N=200 asks for a root front of order >= 65536, which
    the analysis refuses after the handle has been analysed and factored once.  The first check after the failure is
    symbolic_array, which launches nothing: should a failed analysis ever be trusted again, the test stops there instead
    of launching kernels on the plans of a half-built one."""
    dim, irn, jcn, val, nc = mbndry_kkt(200)
    b = np.random.default_rng(1).standard_normal(dim)
    s = handle(dim, irn, jcn, val)
    assert s.factor(True, nc) == (SYMSOLVER_SUCCESS, nc), s.last_error()
    x0 = solved(s, b)

    assert s.set_schur(np.random.default_rng(2).choice(dim, 70000, replace=False)) == SYMSOLVER_SUCCESS
    assert s.factor(True, nc)[0] == SYMSOLVER_FATAL_ERROR
    assert "front too large" in s.last_error(), s.last_error()
    with pytest.raises(KeyError):             # no analysis to report, and running it again fails the same way
        s.symbolic("sn_start")
    assert s.factor(True, nc)[0] == SYMSOLVER_FATAL_ERROR
    assert "front too large" in s.last_error(), s.last_error()
    x = b.copy()
    assert s.solve(x) == SYMSOLVER_FATAL_ERROR
    assert "no factors" in s.last_error(), s.last_error()
    assert np.array_equal(x, b)

    assert s.set_schur([]) == SYMSOLVER_SUCCESS
    assert s.factor(True, nc) == (SYMSOLVER_SUCCESS, nc), s.last_error()
    assert np.array_equal(solved(s, b), x0)
    s.close()
    fresh = handle(dim, irn, jcn, val)
    assert fresh.factor(True, nc) == (SYMSOLVER_SUCCESS, nc), fresh.last_error()
    assert np.array_equal(solved(fresh, b), x0)
    fresh.close()
