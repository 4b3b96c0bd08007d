"""GPU parity of the b200vec kernels (SURVEY.md 8a rows V1-V9) against the REFERENCE's own classes: every case runs the
same inputs through Ipopt::DenseVector / ExpansionMatrix / GenTMatrix / SymTMatrix of the unmodified libipopt.so
(tests/driver/libvecref.so, built against the unmodified libipopt.so in oracle/_ref) and through the CUDA kernels.
Bars: representation (homogeneous flag + scalar) identical; element-wise results BIT-IDENTICAL for everything the
reference computes with its own loops; <= 1 ulp-level relative error where the reference delegates to BLAS (Axpy -> daxpy);
min/max-type reductions exact; sum-type reductions within n*eps*sum|terms| (different summation order)."""
import numpy as np
import pytest

import vecref_api as R

pytestmark = pytest.mark.gpu
SIZES = [0, 1, 37, 1000, 100003]
SCALARS = [0.0, 1.0, -1.0, 2.5]


@pytest.fixture(scope="module")
def ctx():
    if not R.available():
        pytest.skip("tests/driver/libvecref.so not built (needs the reference artefacts in oracle/_ref at build time)")
    from ipopt_b200.vec import VecContext
    c = VecContext()
    yield c
    c.close()


def dev(ctx, hv):
    from ipopt_b200.vec import DenseVector
    v = DenseVector(ctx, hv.n)
    if hv.h:
        v.Set(hv.s)
    else:
        v.SetValues(hv.d[: hv.n])
    return v


def mk(rng, n, kind, positive=False):
    """kind: 'd' dense, 'h' homogeneous, 'z' homogeneous zero, 'o' homogeneous one"""
    if kind == "d":
        v = rng.standard_normal(n) * np.exp(rng.uniform(-3, 3, n))
        if positive:
            v = np.abs(v) + 1e-3
        else:
            v[rng.random(n) < 0.05] = 0.0
        return R.HostVec(n, values=v)
    s = {"h": 1.75 if positive else -1.75, "z": 0.0, "o": 1.0}[kind]
    return R.HostVec(n, scalar=s)


def same_state(yd, yh, exact=True, rtol=0.0):
    if yh.n == 0:
        return    # dimension 0: nothing to compare (the reference host wrapper stores such vectors as homogeneous)
    assert yd.IsHomogeneous() == bool(yh.h)
    if yh.h:
        assert yd.Scalar() == yh.s or (np.isnan(yd.Scalar()) and np.isnan(yh.s))
        return
    got, ref = yd.ExpandedValues(), yh.expanded()
    if exact:
        assert np.array_equal(got, ref, equal_nan=True), np.abs(got - ref).max()
    else:
        assert np.all(np.abs(got - ref) <= rtol * np.maximum(np.abs(ref), 1e-300) + 1e-300)


@pytest.mark.parametrize("n", SIZES)
def test_v3_copy_scal_set_addscalar(ctx, n):
    rng = np.random.default_rng(n)
    for ky in "dh":
        for kx in "dh":
            y, x = mk(rng, n, ky), mk(rng, n, kx)
            yd, xd = dev(ctx, y), dev(ctx, x)
            R.op("copy", y, x1=x); yd.Copy(xd); same_state(yd, y)
            for a in SCALARS:
                R.op("scal", y, a=a); yd.Scal(a); same_state(yd, y)
                R.op("add_scalar", y, a=a); yd.AddScalar(a); same_state(yd, y)
            R.op("set", y, a=3.5); yd.Set(3.5); same_state(yd, y)


@pytest.mark.parametrize("n", SIZES)
def test_v1_axpy(ctx, n):
    rng = np.random.default_rng(100 + n)
    for ky in "dhz":
        for kx in "dhz":
            for a in SCALARS:
                y, x = mk(rng, n, ky), mk(rng, n, kx)
                yd, xd = dev(ctx, y), dev(ctx, x)
                R.op("axpy", y, x1=x, a=a); yd.Axpy(a, xd)
                # dense += dense goes through BLAS daxpy in the reference (FMA or not is the BLAS build's choice)
                blas = (ky == "d" and kx == "d")
                if n == 0:
                    continue
                if blas:
                    assert yd.IsHomogeneous() == bool(y.h)
                    got, ref = yd.ExpandedValues(), y.expanded()
                    assert np.all(np.abs(got - ref) <= 4e-16 * (np.abs(ref) + np.abs(a * x.expanded())))
                else:
                    same_state(yd, y)


@pytest.mark.parametrize("n", SIZES)
def test_v2_reductions(ctx, n):
    rng = np.random.default_rng(200 + n)
    for ky in "dh":
        y = mk(rng, n, ky)
        yd = dev(ctx, y)
        for name, meth in [("amax", "Amax"), ("max", "Max"), ("min", "Min")]:
            assert getattr(yd, meth)() == R.op(name, y), name                       # order-independent: exact
        ref_abs = np.abs(y.expanded()).sum() if n else 0.0
        for name, meth in [("asum", "Asum"), ("sum", "Sum")]:
            assert abs(getattr(yd, meth)() - R.op(name, y)) <= 4 * max(n, 1) * 2.3e-16 * max(ref_abs, 1e-300), name
        nr = R.op("nrm2", y)
        assert abs(yd.Nrm2() - nr) <= 1e-13 * max(nr, 1e-300)
        for kx in "dh":
            x = mk(rng, n, kx)
            xd = dev(ctx, x)
            ref = R.op("dot", y, x1=x)
            bound = 4 * max(n, 1) * 2.3e-16 * max(float(np.abs(y.expanded() * x.expanded()).sum()) if n else 0.0, 1e-300)
            assert abs(yd.Dot(xd) - ref) <= bound
        p = mk(rng, n, ky, positive=True)
        pd = dev(ctx, p)
        ref = R.op("sumlogs", p)
        assert abs(pd.SumLogs() - ref) <= 1e-13 * max(float(np.abs(np.log(p.expanded())).sum()) if n else 0.0, 1.0)
    # extreme magnitudes: the scaled path of Nrm2
    if n > 1:
        for scale in (1e-170, 1e170):
            y = R.HostVec(n, values=rng.standard_normal(n) * scale)
            nr = R.op("nrm2", y)
            assert abs(dev(ctx, y).Nrm2() - nr) <= 1e-13 * nr


@pytest.mark.parametrize("n", SIZES)
def test_v4_elementwise(ctx, n):
    rng = np.random.default_rng(300 + n)
    for ky in "dhz":
        for kx in "dho":
            for name, meth in [("ew_divide", "ElementWiseDivide"), ("ew_multiply", "ElementWiseMultiply"),
                               ("ew_select", "ElementWiseSelect"), ("ew_max", "ElementWiseMax"), ("ew_min", "ElementWiseMin")]:
                y, x = mk(rng, n, ky), mk(rng, n, kx, positive=(name == "ew_divide"))
                yd, xd = dev(ctx, y), dev(ctx, x)
                R.op(name, y, x1=x); getattr(yd, meth)(xd)
                same_state(yd, y)
        for name, meth in [("ew_reciprocal", "ElementWiseReciprocal"), ("ew_abs", "ElementWiseAbs"),
                           ("ew_sqrt", "ElementWiseSqrt"), ("ew_sgn", "ElementWiseSgn")]:
            y = mk(rng, n, ky, positive=(name in ("ew_reciprocal", "ew_sqrt") and ky != "z"))
            if ky == "z" and name == "ew_reciprocal":
                continue
            yd = dev(ctx, y)
            R.op(name, y); getattr(yd, meth)()
            same_state(yd, y)


@pytest.mark.parametrize("n", [0, 1, 37, 100003])
def test_v5_add_two_vectors(ctx, n):
    rng = np.random.default_rng(400 + n)
    for ky in "dh":
        for k1 in "dh":
            for k2 in "dh":
                for a in SCALARS:
                    for b in SCALARS:
                        for c in SCALARS:
                            y, v1, v2 = mk(rng, n, ky), mk(rng, n, k1), mk(rng, n, k2)
                            yd, d1, d2 = dev(ctx, y), dev(ctx, v1), dev(ctx, v2)
                            R.op("add_two_vectors", y, x1=v1, x2=v2, a=a, b=b, c=c)
                            yd.AddTwoVectors(a, d1, b, d2, c)
                            # the mixed homogeneous/dense cases are composed of Copy/Scal/Axpy in the reference -> BLAS daxpy
                            all_dense = (ky == "d" or c == 0.0) and (k1 == "d" or a == 0.0) and (k2 == "d" or b == 0.0)
                            if n == 0:
                                continue
                            if a == 0.0 and b == 1.0 and c == 1.0 and ky == "d" and k2 == "d":
                                # REFERENCE DEFECT, not reproduced: IpDenseVector.cpp:1027-1033 wraps the daxpy of this case
                                # in a `for i < Dim()` loop, so the reference computes y + Dim()*v2 (in Dim() roundings and
                                # O(n^2) time).  The kernel implements the documented operation y = v2 + y; see
                                # test_v5_reference_defect_documented.
                                continue
                            if all_dense and c == 1.0 and (a == 0.0 or b == 0.0) and not (a == 0.0 and b == 0.0):
                                # the reference delegates these to BLAS daxpy (IpDenseVector.cpp:965-1072): FMA or not is
                                # the BLAS build's choice -> one rounding of slack
                                got, ref = yd.ExpandedValues(), y.expanded()
                                mag = np.abs(ref) + np.abs(a * v1.expanded()) + np.abs(b * v2.expanded())
                                assert not yd.IsHomogeneous() and np.all(np.abs(got - ref) <= 2.3e-16 * mag)
                            elif all_dense or y.h:
                                same_state(yd, y)
                            else:
                                mag = np.abs(c * 1.0) + np.abs(a * v1.expanded()) + np.abs(b * v2.expanded()) + np.abs(y.expanded())
                                assert yd.IsHomogeneous() == bool(y.h)
                                assert np.all(np.abs(yd.ExpandedValues() - y.expanded()) <= 1e-15 * (mag + 1.0))


def test_v5_reference_defect_documented(ctx):
    """AddTwoVectors(0, v1, 1, v2, 1) on dense vectors: the reference (IpDenseVector.cpp:1027-1033) runs its daxpy inside a
    loop over Dim() and returns y + Dim()*v2; the kernel returns y + v2 (the documented semantics, IpVector.hpp AddTwoVectors:
    "y = a*v1 + b*v2 + c*y").  This test pins BOTH facts so the deviation is explicit."""
    n = 5
    y0, v2 = np.arange(1.0, n + 1), np.array([0.5, -1.0, 2.0, 0.25, 3.0])
    y = R.HostVec(n, values=y0.copy()); h2 = R.HostVec(n, values=v2); h1 = R.HostVec(n, values=np.zeros(n))
    R.op("add_two_vectors", y, x1=h1, x2=h2, a=0.0, b=1.0, c=1.0)
    assert np.array_equal(y.expanded(), y0 + n * v2)            # what the reference does
    yd = dev(ctx, R.HostVec(n, values=y0.copy()))
    yd.AddTwoVectors(0.0, dev(ctx, h1), 1.0, dev(ctx, h2), 1.0)
    assert np.array_equal(yd.ExpandedValues(), y0 + v2)         # what the kernel does


@pytest.mark.parametrize("n", SIZES)
def test_v6_frac_to_bound(ctx, n):
    rng = np.random.default_rng(500 + n)
    for kx in "dh":
        for kd in "dhz":
            for tau in (0.99, 0.5, 1.0):
                x, d = mk(rng, n, kx, positive=True), mk(rng, n, kd)
                if kd == "d":
                    d.d[: n] *= 50.0
                ref = R.op("frac_to_bound", x, x1=d, a=tau)
                assert dev(ctx, x).FracToBound(dev(ctx, d), tau) == ref   # a min-reduction of identically rounded terms: exact


@pytest.mark.parametrize("n", SIZES)
def test_v7_add_vector_quotient(ctx, n):
    rng = np.random.default_rng(600 + n)
    for ky in "dh":
        for kz in "dh":
            for ks in "dh":
                for a in SCALARS:
                    for c in SCALARS:
                        y, z, s = mk(rng, n, ky), mk(rng, n, kz), mk(rng, n, ks, positive=True)
                        yd, zd, sd = dev(ctx, y), dev(ctx, z), dev(ctx, s)
                        R.op("add_vector_quotient", y, x1=z, x2=s, a=a, c=c)
                        yd.AddVectorQuotient(a, zd, sd, c)
                        same_state(yd, y)


@pytest.mark.parametrize("nrows,ncols", [(10, 0), (10, 10), (1000, 317), (100003, 60007)])
def test_v8_expansion_matrix(ctx, nrows, ncols):
    from ipopt_b200.vec import ExpansionMatrix
    rng = np.random.default_rng(700 + nrows)
    pos = np.sort(rng.choice(nrows, ncols, replace=False)).astype(np.int32)
    P = ExpansionMatrix(ctx, nrows, ncols, pos)
    for alpha in SCALARS[1:] + [0.0]:
        for beta in (0.0, 1.0, -0.5):
            for kx in "dhz":
                for ky in "dh":
                    x, y = mk(rng, ncols, kx), mk(rng, nrows, ky)
                    xd, yd = dev(ctx, x), dev(ctx, y)
                    R.expansion(0, nrows, ncols, pos, alpha, beta, y, x1=x); P.MultVector(alpha, xd, beta, yd)
                    same_state(yd, y)
                    x, y = mk(rng, nrows, kx), mk(rng, ncols, ky)
                    xd, yd = dev(ctx, x), dev(ctx, y)
                    R.expansion(1, nrows, ncols, pos, alpha, beta, y, x1=x); P.TransMultVector(alpha, xd, beta, yd)
                    same_state(yd, y)
        for kz in "dhz":
            for kX in "dh":
                S, Z, X = mk(rng, ncols, "d", positive=True), mk(rng, ncols, kz), mk(rng, nrows, kX)
                Sd, Zd, Xd = dev(ctx, S), dev(ctx, Z), dev(ctx, X)
                R.expansion(2, nrows, ncols, pos, alpha, 0.0, X, x1=S, x2=Z); P.AddMSinvZ(alpha, Sd, Zd, Xd)
                same_state(Xd, X)
            for kr in "dh":
                S, Rv, Z, D = mk(rng, ncols, "d", positive=True), mk(rng, ncols, kr), mk(rng, ncols, kz), mk(rng, nrows, "d")
                X = mk(rng, ncols, "h")
                Sd, Rd, Zd, Dd, Xd = dev(ctx, S), dev(ctx, Rv), dev(ctx, Z), dev(ctx, D), dev(ctx, X)
                R.expansion(3, nrows, ncols, pos, alpha, 0.0, X, x1=S, x2=Rv, x3=Z, x4=D)
                P.SinvBlrmZMTdBr(alpha, Sd, Rd, Zd, Dd, Xd)
                same_state(Xd, X)


@pytest.mark.parametrize("nrows,ncols,nnz", [(5, 7, 0), (50, 40, 300), (20000, 30000, 150000)])
def test_v9_triplet_spmv(ctx, nrows, ncols, nnz):
    from ipopt_b200.vec import TripletMatrix
    rng = np.random.default_rng(800 + nnz)
    ir = rng.integers(1, nrows + 1, nnz).astype(np.int32)
    jc = rng.integers(1, ncols + 1, nnz).astype(np.int32)    # duplicates included: they are accumulated in triplet order
    val = rng.standard_normal(nnz)
    A = TripletMatrix(ctx, nrows, ncols, ir, jc, symmetric=False)
    A.SetValues(val)
    for trans in (False, True):
        nin, nout = (nrows, ncols) if trans else (ncols, nrows)
        for alpha in (1.0, -1.0, 0.7):
            for beta in (0.0, 1.0, -2.0):
                for kx in "dh":
                    for ky in "dh":
                        x, y = mk(rng, nin, kx), mk(rng, nout, ky)
                        xd, yd = dev(ctx, x), dev(ctx, y)
                        R.tmat(False, trans, nrows, ncols, ir, jc, val, alpha, beta, x, y)
                        (A.TransMultVector if trans else A.MultVector)(alpha, xd, beta, yd)
                        same_state(yd, y)     # bit-identical: same accumulation order as the reference's scalar loop
    A.close()
    # symmetric (lower-triangle triplets + some diagonal entries)
    n = nrows
    i2 = rng.integers(1, n + 1, nnz).astype(np.int32)
    j2 = rng.integers(1, n + 1, nnz).astype(np.int32)
    lo, hi = np.maximum(i2, j2), np.minimum(i2, j2)
    Sm = TripletMatrix(ctx, n, n, lo, hi, symmetric=True)
    Sm.SetValues(val)
    for alpha in (1.0, 0.3):
        for beta in (0.0, 1.0):
            for kx in "dh":
                x, y = mk(rng, n, kx), mk(rng, n, "d")
                xd, yd = dev(ctx, x), dev(ctx, y)
                R.tmat(True, False, n, n, lo, hi, val, alpha, beta, x, y)
                Sm.MultVector(alpha, xd, beta, yd)
                same_state(yd, y)
    Sm.close()
