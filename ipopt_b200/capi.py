"""ctypes mirror of the reference's solver plugin interface on top of the C ABI.

Method names, argument meaning and status codes follow
``Ipopt::SparseSymLinearSolverInterface`` (reference
src/Algorithm/LinearSolvers/IpSparseSymLinearSolverInterface.hpp:98-256) and
``ESymSolverStatus`` (IpSymLinearSolver.hpp:19-33) so the parity tests read like calls the
reference's ``TSymLinearSolver`` makes (IpTSymLinearSolver.cpp:159-312).
There is NO CPU fallback: constructing :class:`B200Ldlt` without a usable CUDA device raises.
"""
import ctypes as C
import os

import numpy as np

SYMSOLVER_SUCCESS, SYMSOLVER_SINGULAR, SYMSOLVER_WRONG_INERTIA, SYMSOLVER_CALL_AGAIN, SYMSOLVER_FATAL_ERROR = range(5)

_HERE = os.path.dirname(os.path.abspath(__file__))


def lib_path():
    return os.path.join(_HERE, "lib", "libb200ldlt.so")


class Options(C.Structure):
    _fields_ = [("device", C.c_int), ("stream", C.c_void_p), ("ordering", C.c_int), ("pair_saddle", C.c_int),
                ("leaf_k", C.c_int), ("relax_frac", C.c_double), ("scaling", C.c_int), ("pivtol", C.c_double),
                ("pivtolmax", C.c_double), ("tiny", C.c_double), ("smem_front_max", C.c_int),
                ("use_graph", C.c_int), ("verbose", C.c_int), ("tc_schur_min_r", C.c_int)]


class AugSys(C.Structure):
    _fields_ = [("n_x", C.c_int), ("n_s", C.c_int), ("n_c", C.c_int), ("n_d", C.c_int), ("nnz_w", C.c_int),
                ("nnz_jc", C.c_int), ("nnz_jd", C.c_int), ("W", C.c_void_p), ("W_factor", C.c_double),
                ("D_x", C.c_void_p), ("delta_x", C.c_double), ("D_s", C.c_void_p), ("delta_s", C.c_double),
                ("J_c", C.c_void_p), ("D_c", C.c_void_p), ("delta_c", C.c_double), ("J_d", C.c_void_p),
                ("D_d", C.c_void_p), ("delta_d", C.c_double)]


class Info(C.Structure):
    _fields_ = [("n", C.c_int), ("nnz_in", C.c_int64), ("nnz_unique", C.c_int64), ("nsupernodes", C.c_int),
                ("nlevels", C.c_int), ("max_front", C.c_int), ("max_pivots", C.c_int), ("n_saddle", C.c_int),
                ("n_pairs", C.c_int), ("nnz_L", C.c_int64), ("nnz_L_true", C.c_int64), ("L_bytes", C.c_int64),
                ("cb_bytes", C.c_int64), ("flops_panel", C.c_double), ("flops_schur", C.c_double),
                ("t_order_s", C.c_double), ("t_symbolic_s", C.c_double), ("num_neg", C.c_int),
                ("num_forced", C.c_int), ("num_tiny", C.c_int), ("num_growth", C.c_int), ("num_2x2", C.c_int),
                ("ms_factor_gpu", C.c_float), ("ms_solve_gpu", C.c_float), ("launches_factor", C.c_int),
                ("launches_solve", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Errors(C.Structure):
    """b200ldlt_errors: the error analysis of one column (see include/b200ldlt.h for the definitions)"""
    _fields_ = [("anorm", C.c_double), ("xnorm", C.c_double), ("rnorm", C.c_double), ("omega1", C.c_double),
                ("omega2", C.c_double), ("cond1", C.c_double), ("cond2", C.c_double), ("ferr", C.c_double),
                ("n_i2", C.c_int), ("nprod", C.c_int)]


class Refined(C.Structure):
    """b200ldlt_refined: the outcome of the refinement of one column (see include/b200ldlt.h)"""
    _fields_ = [("omega_first", C.c_double), ("omega1", C.c_double), ("omega2", C.c_double), ("steps", C.c_int),
                ("status", C.c_int), ("nres", C.c_int)]


class Gmres(C.Structure):
    """b200ldlt_gmres: the outcome of FGMRES on one column (see include/b200ldlt.h)"""
    _fields_ = [("omega_first", C.c_double), ("omega1", C.c_double), ("omega2", C.c_double), ("cycles", C.c_int),
                ("iters", C.c_int), ("status", C.c_int), ("nres", C.c_int)]


EXPORTED = ["b200ldlt_default_options", "b200ldlt_create", "b200ldlt_destroy", "b200ldlt_last_error",
            "b200ldlt_analyse", "b200ldlt_values_ptr", "b200ldlt_factor", "b200ldlt_factor_device",
            "b200ldlt_solve", "b200ldlt_solve_device", "b200ldlt_num_neg", "b200ldlt_increase_quality",
            "b200ldlt_refactor", "b200ldlt_get_info", "b200ldlt_symbolic_array", "b200ldlt_analyse_now",
            "b200ldlt_residual", "b200ldlt_set_pivtol",
            "b200ldlt_assemble_augsys_device", "b200ldlt_solve_refine_device",
            "b200ldlt_solve_partial", "b200ldlt_solve_partial_device", "b200ldlt_enquire_indef",
            "b200ldlt_lmultiply", "b200ldlt_lmultiply_device", "b200ldlt_alter_d",
            "b200ldlt_sparse_fwd_solve", "b200ldlt_sparse_fwd_solve_device", "b200ldlt_set_singular_action",
            "b200ldlt_enquire_zero_pivots", "b200ldlt_solve_fredholm", "b200ldlt_solve_fredholm_device",
            "b200ldlt_selected_inverse", "b200ldlt_selected_inverse_device", "b200ldlt_set_schur",
            "b200ldlt_schur_complement", "b200ldlt_schur_complement_device", "b200ldlt_schur_reduce",
            "b200ldlt_schur_reduce_device", "b200ldlt_schur_expand", "b200ldlt_schur_expand_device",
            "b200ldlt_error_analysis", "b200ldlt_error_analysis_device", "b200ldlt_condest",
            "b200ldlt_inverse_entries", "b200ldlt_inverse_entries_device", "b200ldlt_solve_refined",
            "b200ldlt_solve_refined_device", "b200ldlt_sparse_solve", "b200ldlt_sparse_solve_device",
            "b200ldlt_solve_gmres", "b200ldlt_solve_gmres_device"]

_lib = None


def load_library():
    """Load libb200ldlt.so (raises if it has not been built: run ``python __graft_entry__.py build``)."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise RuntimeError("libb200ldlt.so is not built (%s); run `make -C ipopt_b200/csrc`" % p)
    L = C.CDLL(p)
    vp, ip, dp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_double)
    L.b200ldlt_default_options.argtypes = [C.POINTER(Options)]
    L.b200ldlt_default_options.restype = None
    L.b200ldlt_create.argtypes = [C.POINTER(Options)]
    L.b200ldlt_create.restype = vp
    L.b200ldlt_destroy.argtypes = [vp]
    L.b200ldlt_destroy.restype = None
    L.b200ldlt_last_error.argtypes = [vp]
    L.b200ldlt_last_error.restype = C.c_char_p
    L.b200ldlt_analyse.argtypes = [vp, C.c_int, C.c_int, ip, ip]
    L.b200ldlt_values_ptr.argtypes = [vp]
    L.b200ldlt_values_ptr.restype = dp
    L.b200ldlt_factor.argtypes = [vp, C.c_int, C.c_int, ip]
    L.b200ldlt_factor_device.argtypes = [vp, vp, C.c_int, C.c_int, ip]
    L.b200ldlt_refactor.argtypes = [vp, C.c_int, C.c_int, ip]
    L.b200ldlt_assemble_augsys_device.argtypes = [vp, C.POINTER(AugSys)]
    L.b200ldlt_solve_refine_device.argtypes = [vp, vp, C.c_int, C.c_int, C.c_double, ip, dp]
    L.b200ldlt_device_ptr.argtypes = [vp, C.c_char_p]
    L.b200ldlt_device_ptr.restype = vp
    L.b200ldlt_solve.argtypes = [vp, C.c_int, dp]
    L.b200ldlt_solve_device.argtypes = [vp, C.c_int, vp]
    L.b200ldlt_solve_partial.argtypes = [vp, C.c_int, C.c_int, dp]
    L.b200ldlt_solve_partial_device.argtypes = [vp, C.c_int, C.c_int, vp]
    L.b200ldlt_enquire_indef.argtypes = [vp, ip, ip, dp]
    L.b200ldlt_lmultiply.argtypes = [vp, C.c_int, C.c_int, dp, dp]
    L.b200ldlt_lmultiply_device.argtypes = [vp, C.c_int, C.c_int, vp, vp]
    L.b200ldlt_alter_d.argtypes = [vp, dp]
    L.b200ldlt_sparse_fwd_solve.argtypes = [vp, C.c_int, ip, dp, ip, ip, dp]
    L.b200ldlt_sparse_fwd_solve_device.argtypes = [vp, C.c_int, ip, vp, ip, ip, vp]
    L.b200ldlt_sparse_solve.argtypes = [vp, C.c_int, C.c_int, ip, dp, C.c_int, ip, dp]
    L.b200ldlt_sparse_solve_device.argtypes = [vp, C.c_int, C.c_int, ip, vp, C.c_int, ip, vp]
    L.b200ldlt_set_singular_action.argtypes = [vp, C.c_int]
    L.b200ldlt_enquire_zero_pivots.argtypes = [vp, ip, ip]
    L.b200ldlt_solve_fredholm.argtypes = [vp, C.c_int, C.c_double, dp, ip]
    L.b200ldlt_solve_fredholm_device.argtypes = [vp, C.c_int, C.c_double, vp, ip]
    L.b200ldlt_selected_inverse.argtypes = [vp, dp, dp]
    L.b200ldlt_selected_inverse_device.argtypes = [vp, vp, vp]
    L.b200ldlt_inverse_entries.argtypes = [vp, C.c_int, ip, ip, dp]
    L.b200ldlt_inverse_entries_device.argtypes = [vp, C.c_int, ip, ip, vp]
    L.b200ldlt_set_schur.argtypes = [vp, C.c_int, ip]
    L.b200ldlt_schur_complement.argtypes = [vp, dp]
    L.b200ldlt_schur_complement_device.argtypes = [vp, vp]
    L.b200ldlt_schur_reduce.argtypes = [vp, C.c_int, dp, dp]
    L.b200ldlt_schur_reduce_device.argtypes = [vp, C.c_int, vp, vp]
    L.b200ldlt_schur_expand.argtypes = [vp, C.c_int, dp, dp, dp]
    L.b200ldlt_schur_expand_device.argtypes = [vp, C.c_int, vp, vp, vp]
    L.b200ldlt_error_analysis.argtypes = [vp, C.c_int, dp, dp, C.c_int, C.POINTER(Errors)]
    L.b200ldlt_error_analysis_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.POINTER(Errors)]
    L.b200ldlt_condest.argtypes = [vp, dp, dp, dp, ip]
    L.b200ldlt_solve_refined.argtypes = [vp, C.c_int, dp, dp, C.c_int, C.c_double, C.POINTER(Refined)]
    L.b200ldlt_solve_refined_device.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.c_double, C.POINTER(Refined)]
    L.b200ldlt_solve_gmres.argtypes = [vp, C.c_int, dp, dp, dp, C.c_int, C.c_int, C.c_double, C.c_double,
                                       C.POINTER(Gmres)]
    L.b200ldlt_solve_gmres_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, C.c_int, C.c_double, C.c_double,
                                              C.POINTER(Gmres)]
    L.b200ldlt_num_neg.argtypes = [vp]
    L.b200ldlt_increase_quality.argtypes = [vp]
    L.b200ldlt_get_info.argtypes = [vp, C.POINTER(Info)]
    L.b200ldlt_symbolic_array.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int64), C.c_int64]
    L.b200ldlt_symbolic_array.restype = C.c_int64
    L.b200ldlt_analyse_now.argtypes = [vp, dp]
    L.b200ldlt_residual.argtypes = [vp, dp, dp, dp, dp, dp]
    L.b200ldlt_symbolic_create.argtypes = [C.c_int, C.c_int, ip, ip, dp, C.c_int, C.c_int, C.c_int, C.c_double]
    L.b200ldlt_symbolic_create.restype = vp
    L.b200ldlt_symbolic_create_schur.argtypes = [C.c_int, C.c_int, ip, ip, dp, C.c_int, C.c_int, C.c_int, C.c_double,
                                                 C.c_int, ip]
    L.b200ldlt_symbolic_create_schur.restype = vp
    L.b200ldlt_symbolic_free.argtypes = [vp]
    L.b200ldlt_symbolic_free.restype = None
    L.b200ldlt_symbolic_get.argtypes = [vp, C.c_char_p, C.POINTER(C.c_longlong), C.c_longlong]
    L.b200ldlt_symbolic_get.restype = C.c_longlong
    L.b200ldlt_symbolic_shard.argtypes = [vp, C.c_int, C.POINTER(C.c_longlong), C.c_longlong]
    L.b200ldlt_symbolic_shard.restype = C.c_longlong
    _lib = L
    return L


def _iptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class SymbolicAnalysis:
    """Host-only symbolic analysis (ordering, elimination tree, supernodes, maps). No GPU needed."""
    STATS = ["n", "nsn", "nlevels", "max_front", "max_k", "n_saddle", "n_pairs", "nnzL", "nnzL_true", "cb_total",
             "flops_panel", "flops_schur", "ms_order", "ms_symbolic"]

    def __init__(self, dim, irn, jcn, vals=None, ordering=0, pair_saddle=1, leaf_k=0, relax_frac=-1.0, schur=None):
        """schur: the 0-based Schur variables, which become the last pivot positions in this order (one root
        supernode); None or empty: the ordinary analysis."""
        L = load_library()
        irn = np.ascontiguousarray(irn, dtype=np.int32)
        jcn = np.ascontiguousarray(jcn, dtype=np.int32)
        vp = None
        if vals is not None:
            vals = np.ascontiguousarray(vals, dtype=np.float64)
            vp = _dptr(vals)
        self._L = L
        sc = np.ascontiguousarray([] if schur is None else schur, dtype=np.int32)
        self._h = L.b200ldlt_symbolic_create_schur(int(dim), int(len(irn)), _iptr(irn), _iptr(jcn), vp, ordering,
                                                   pair_saddle, leaf_k, relax_frac, len(sc), _iptr(sc))
        if not self._h:
            raise RuntimeError("symbolic analysis failed")

    def get(self, name):
        n = self._L.b200ldlt_symbolic_get(self._h, name.encode(), None, 0)
        if n < 0:
            raise KeyError(name)
        out = np.zeros(max(n, 1), dtype=np.int64)
        self._L.b200ldlt_symbolic_get(self._h, name.encode(), out.ctypes.data_as(C.POINTER(C.c_longlong)), n)
        return out[:n]

    def stats(self):
        return dict(zip(self.STATS, self.get("stats").tolist()))

    def shard(self, world):
        """(owner per supernode [-1 = top part, factorised by rank 0], number of subtrees below the cut)."""
        nsn = len(self.get("sn_start")) - 1
        out = np.zeros(max(nsn, 1), dtype=np.int64)
        nsub = self._L.b200ldlt_symbolic_shard(self._h, int(world), out.ctypes.data_as(C.POINTER(C.c_longlong)), nsn)
        return out[:nsn], int(nsub)

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200ldlt_symbolic_free(self._h)
            self._h = None


class B200Ldlt:
    """Mirror of Ipopt::SparseSymLinearSolverInterface on top of the C ABI (GPU required)."""

    Triplet_Format = 0  # EMatrixFormat, IpSparseSymLinearSolverInterface.hpp:101-114

    def __init__(self, **opts):
        L = load_library()
        self._L = L
        o = Options()
        L.b200ldlt_default_options(C.byref(o))
        for k, v in opts.items():
            if not hasattr(o, k):
                raise TypeError("unknown option %s" % k)
            setattr(o, k, v)
        self.options = o
        self._h = L.b200ldlt_create(C.byref(o))
        if not self._h:
            raise RuntimeError("b200ldlt_create failed: no usable CUDA device (this backend has no CPU fallback)")
        self.dim = 0
        self.nonzeros = 0
        self._negevals = -1
        self._ia = self._ja = None
        self._sc_m = 0

    # -- the 8 virtuals -------------------------------------------------------------------------
    def InitializeStructure(self, dim, nonzeros, ia, ja):
        self._ia = np.ascontiguousarray(ia, dtype=np.int32)
        self._ja = np.ascontiguousarray(ja, dtype=np.int32)
        assert len(self._ia) == nonzeros and len(self._ja) == nonzeros
        self.dim, self.nonzeros = int(dim), int(nonzeros)
        self._sc_m = 0                   # (the analysis clears Schur mode)
        return self._L.b200ldlt_analyse(self._h, self.dim, self.nonzeros, _iptr(self._ia), _iptr(self._ja))

    def GetValuesArrayPtr(self):
        p = self._L.b200ldlt_values_ptr(self._h)
        return np.ctypeslib.as_array(p, shape=(max(self.nonzeros, 1),))[:self.nonzeros]

    def MultiSolve(self, new_matrix, ia, ja, nrhs, rhs_vals, check_NegEVals, numberOfNegEVals):
        """rhs_vals: float64 array of dim*nrhs (column-major), overwritten with the solution."""
        if new_matrix:
            neg = C.c_int(-1)
            st = self._L.b200ldlt_factor(self._h, int(bool(check_NegEVals)), int(numberOfNegEVals), C.byref(neg))
            self._negevals = neg.value
            if st != SYMSOLVER_SUCCESS:
                return st
        assert rhs_vals.dtype == np.float64 and rhs_vals.flags["C_CONTIGUOUS"] or rhs_vals.flags["F_CONTIGUOUS"]
        return self._L.b200ldlt_solve(self._h, int(nrhs), _dptr(rhs_vals))

    def NumberOfNegEVals(self):
        return self._L.b200ldlt_num_neg(self._h)

    def IncreaseQuality(self):
        return bool(self._L.b200ldlt_increase_quality(self._h))

    def ProvidesInertia(self):
        return True

    def MatrixFormat(self):
        return self.Triplet_Format

    # -- extras -----------------------------------------------------------------------------------
    def factor(self, check=False, expected=0):
        neg = C.c_int(-1)
        st = self._L.b200ldlt_factor(self._h, int(check), int(expected), C.byref(neg))
        return st, neg.value

    def factor_device(self, d_vals_ptr, check=False, expected=0):
        neg = C.c_int(-1)
        st = self._L.b200ldlt_factor_device(self._h, C.c_void_p(d_vals_ptr), int(check), int(expected), C.byref(neg))
        return st, neg.value

    def refactor(self, check=False, expected=0):
        neg = C.c_int(-1)
        st = self._L.b200ldlt_refactor(self._h, int(check), int(expected), C.byref(neg))
        return st, neg.value

    def solve(self, rhs, nrhs=1):
        return self._L.b200ldlt_solve(self._h, int(nrhs), _dptr(rhs))

    def solve_device(self, d_rhs_ptr, nrhs=1):
        return self._L.b200ldlt_solve_device(self._h, int(nrhs), C.c_void_p(d_rhs_ptr))

    def solve_partial(self, job, rhs, nrhs=1):
        """One part of the solve, in place on float64 rhs (dim*nrhs, column-major): job 0 = A^-1 b, 1 = L^-1 P^T S b,
        2 = D^-1 b, 3 = S P L^-T b, 4 = S P L^-T D^-1 b (intermediate vectors in pivot order, see b200ldlt.h)."""
        return self._L.b200ldlt_solve_partial(self._h, int(job), int(nrhs), _dptr(rhs))

    def solve_partial_device(self, job, d_rhs_ptr, nrhs=1):
        return self._L.b200ldlt_solve_partial_device(self._h, int(job), int(nrhs), C.c_void_p(d_rhs_ptr))

    def enquire_indef(self):
        """(pivot_var, pivot_type, dinv) per pivot position: the 0-based original variable, 1 / 2 / 3 (1x1 / first /
        second of a 2x2 pivot), and an (n, 2) array of the diagonal and off-diagonal entry of D^-1 (scaled matrix)."""
        n = self.dim
        var, ty, d = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros((n, 2), np.float64)
        if self._L.b200ldlt_enquire_indef(self._h, _iptr(var), _iptr(ty), _dptr(d)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return var, ty, d

    def lmultiply(self, trans, x, nrhs=1):
        """Multiply by the factors: trans 0: S^-1 P L x (pivot -> original order), trans 1: L^T P^T S^-1 x (original ->
        pivot order), x float64 dim*nrhs column-major.  Returns y (a new array); raises on a refusal."""
        x = np.ascontiguousarray(x, dtype=np.float64).ravel()
        y = np.empty_like(x)
        if self._L.b200ldlt_lmultiply(self._h, int(trans), int(nrhs), _dptr(x), _dptr(y)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return y

    def lmultiply_device(self, trans, d_x_ptr, d_y_ptr, nrhs=1):
        """The same on device addresses (d_y may be d_x); returns the status."""
        return self._L.b200ldlt_lmultiply_device(self._h, int(trans), int(nrhs), C.c_void_p(d_x_ptr), C.c_void_p(d_y_ptr))

    def alter_d(self, dinv):
        """Replace D^-1 by an (n, 2) array in the layout enquire_indef returns; returns the status (FATAL_ERROR and D
        unchanged for a non-finite entry or an off-diagonal entry where no 2x2 pivot opens)."""
        d = np.ascontiguousarray(dinv, dtype=np.float64)
        assert d.size == 2 * self.dim
        return self._L.b200ldlt_alter_d(self._h, _dptr(d))

    def sparse_fwd_solve(self, bindex, b):
        """Job 1 (L^-1 P^T S b, pivot order) of a sparse b: bindex the distinct 0-based variables where b is non-zero, b
        their values.  Returns (xindex, x): the pivot positions of the fronts b reaches, ascending, and job 1's vector
        there (zero everywhere else).  Raises on a refusal."""
        bi = np.ascontiguousarray(bindex, dtype=np.int32)
        bv = np.ascontiguousarray(b, dtype=np.float64)
        assert bv.shape == bi.shape
        nxi = C.c_int(0)
        xi, x = np.zeros(max(self.dim, 1), np.int32), np.zeros(max(self.dim, 1), np.float64)
        if self._L.b200ldlt_sparse_fwd_solve(self._h, len(bi), _iptr(bi), _dptr(bv), C.byref(nxi), _iptr(xi),
                                             _dptr(x)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return xi[:nxi.value].copy(), x[:nxi.value].copy()

    def sparse_fwd_solve_device(self, bindex, d_b_ptr, d_x_ptr):
        """The same with the values in device memory: d_b holds len(bindex) doubles, d_x receives the nxi values (room for
        dim doubles).  Returns xindex; raises on a refusal."""
        bi = np.ascontiguousarray(bindex, dtype=np.int32)
        nxi = C.c_int(0)
        xi = np.zeros(max(self.dim, 1), np.int32)
        if self._L.b200ldlt_sparse_fwd_solve_device(self._h, len(bi), _iptr(bi), C.c_void_p(d_b_ptr), C.byref(nxi),
                                                    _iptr(xi), C.c_void_p(d_x_ptr)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return xi[:nxi.value].copy()

    def sparse_solve(self, bindex, B, xsel):
        """Chosen entries of A^-1 b for sparse b's that share one pattern (b200ldlt_sparse_solve): B is nrhs x nbi (or a
        vector of nbi), row c the values of column c at the 0-based variables bindex; returns the nrhs x nxs entries of
        the solutions at the variables xsel (a vector for a vector B).  bindex = None: B is dense (nrhs x dim); xsel =
        None: every entry.  Raises on a refusal."""
        B = np.asarray(B, dtype=np.float64)
        one = B.ndim == 1
        nbi = self.dim if bindex is None else len(bindex)
        Bm = np.ascontiguousarray(B.reshape(1 if one else B.shape[0], nbi))
        nrhs = Bm.shape[0]
        bi = None if bindex is None else np.ascontiguousarray(bindex, dtype=np.int32)
        xs = None if xsel is None else np.ascontiguousarray(xsel, dtype=np.int32)
        nxs = self.dim if xs is None else len(xs)
        X = np.zeros((nrhs, nxs))
        if self._L.b200ldlt_sparse_solve(self._h, nrhs, nbi, None if bi is None else _iptr(bi), _dptr(Bm), nxs,
                                         None if xs is None else _iptr(xs), _dptr(X)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return X[0] if one else X

    def sparse_solve_device(self, bindex, d_b_ptr, xsel, d_x_ptr, nrhs=1):
        """The same with the values in device memory: d_b holds nrhs x nbi doubles (column c at c nbi), d_x receives
        nrhs x nxs (pointers as ints).  Returns the status."""
        bi = None if bindex is None else np.ascontiguousarray(bindex, dtype=np.int32)
        xs = None if xsel is None else np.ascontiguousarray(xsel, dtype=np.int32)
        nbi = self.dim if bi is None else len(bi)
        nxs = self.dim if xs is None else len(xs)
        return self._L.b200ldlt_sparse_solve_device(self._h, int(nrhs), nbi, None if bi is None else _iptr(bi),
                                                    C.c_void_p(d_b_ptr), nxs, None if xs is None else _iptr(xs),
                                                    C.c_void_p(d_x_ptr))

    def set_singular_action(self, keep):
        """keep = 1: a SINGULAR factorisation whose zero pivots are all rounding noise keeps its factors (D^+); 0 (the
        default): it keeps none.  Takes effect from the next factor call; returns the status."""
        return self._L.b200ldlt_set_singular_action(self._h, int(keep))

    def enquire_zero_pivots(self):
        """The pivot positions of the zero pivots of the kept factors, ascending.  Raises without factors."""
        nz = C.c_int(0)
        pos = np.zeros(max(self.dim, 1), np.int32)
        if self._L.b200ldlt_enquire_zero_pivots(self._h, C.byref(nz), _iptr(pos)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return pos[:nz.value].copy()

    def solve_fredholm(self, B, tol):
        """Fredholm alternative for the columns of B (dim or dim x nrhs): returns (X, F, consistent) with X the D^+
        solutions, F the null-space certificates (A F = 0, b^T f > 0 where inconsistent) and consistent a bool array.
        Raises on a refusal."""
        B = np.asarray(B, dtype=np.float64)
        one = B.ndim == 1
        Bm = B.reshape(self.dim, -1, order="F")
        nrhs = Bm.shape[1]
        x = np.zeros((self.dim, 2 * nrhs), order="F")
        x[:, :nrhs] = Bm
        cons = np.zeros(max(nrhs, 1), np.int32)
        if self._L.b200ldlt_solve_fredholm(self._h, nrhs, float(tol), _dptr(x), _iptr(cons)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        X, F, c = x[:, :nrhs].copy(), x[:, nrhs:].copy(), cons[:nrhs].astype(bool)
        return (X[:, 0], F[:, 0], c) if one else (X, F, c)

    def solve_fredholm_device(self, d_x_ptr, nrhs, tol):
        """The same on a device array of dim x 2 nrhs doubles (b's in the first nrhs columns; x and f on return).
        Returns (status, consistent)."""
        cons = np.zeros(max(int(nrhs), 1), np.int32)
        st = self._L.b200ldlt_solve_fredholm_device(self._h, int(nrhs), float(tol), C.c_void_p(d_x_ptr), _iptr(cons))
        return st, cons[:int(nrhs)].astype(bool)

    def selected_inverse(self, diag=True, pattern=True):
        """Entries of M = A^-1 (b200ldlt_selected_inverse): (diag, vals) -- diag[i] = M_ii (dim doubles, original order),
        vals[t] = M at triplet t of the analysed pattern (nonzeros doubles) -- each None when not asked for."""
        d = np.zeros(self.dim) if diag else None
        v = np.zeros(self.nonzeros) if pattern else None
        if self._L.b200ldlt_selected_inverse(self._h, None if d is None else _dptr(d),
                                             None if v is None else _dptr(v)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return d, v

    def selected_inverse_device(self, d_diag_ptr, d_vals_ptr):
        """The same into device arrays (pointers as ints, 0 = not wanted). Returns the status."""
        return self._L.b200ldlt_selected_inverse_device(self._h, C.c_void_p(d_diag_ptr or None),
                                                        C.c_void_p(d_vals_ptr or None))

    def inverse_entries(self, irow, jcol):
        """Entries of M = A^-1 at chosen positions (b200ldlt_inverse_entries): vals[t] = M(irow[t], jcol[t]) for 0-based
        original indices, as a numpy array.  Raises on a refusal."""
        i = np.ascontiguousarray(irow, dtype=np.int32)
        j = np.ascontiguousarray(jcol, dtype=np.int32)
        assert i.shape == j.shape and i.ndim == 1
        v = np.zeros(max(len(i), 1))
        if self._L.b200ldlt_inverse_entries(self._h, len(i), _iptr(i), _iptr(j), _dptr(v)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return v[:len(i)].copy()

    def inverse_entries_device(self, irow, jcol, d_vals_ptr):
        """The same into a device array of len(irow) doubles (pointer as an int).  Returns the status."""
        i = np.ascontiguousarray(irow, dtype=np.int32)
        j = np.ascontiguousarray(jcol, dtype=np.int32)
        assert i.shape == j.shape and i.ndim == 1
        return self._L.b200ldlt_inverse_entries_device(self._h, len(i), _iptr(i), _iptr(j), C.c_void_p(d_vals_ptr))

    def set_schur(self, vars):
        """Schur mode on the 0-based variables vars (empty: off).  Takes effect at the next factor call, which re-analyses
        with vars last and leaves their Schur complement.  Returns the status."""
        v = np.ascontiguousarray(vars, dtype=np.int32)
        st = self._L.b200ldlt_set_schur(self._h, len(v), _iptr(v) if len(v) else None)
        if st == SYMSOLVER_SUCCESS:
            self._sc_m = len(v)
        return st

    def schur_complement(self):
        """S_c = A_SS - A_SE A_EE^-1 A_ES (m x m, row / column i = vars[i]) of the last factorisation.  Raises on a
        refusal."""
        m = self._sc_m
        sc = np.zeros((m, m), order="F")
        if self._L.b200ldlt_schur_complement(self._h, _dptr(sc)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return sc

    def schur_complement_device(self, d_sc_ptr):
        """The same into a device array of m x m doubles.  Returns the status."""
        return self._L.b200ldlt_schur_complement_device(self._h, C.c_void_p(d_sc_ptr))

    def schur_reduce(self, B):
        """y = b_S - A_SE A_EE^-1 b_E for the columns of B (dim or dim x nrhs).  Raises on a refusal."""
        B = np.asarray(B, dtype=np.float64)
        Bm = np.asfortranarray(B.reshape(self.dim, -1, order="F"))
        nrhs, m = Bm.shape[1], self._sc_m
        y = np.zeros((m, nrhs), order="F")
        if self._L.b200ldlt_schur_reduce(self._h, nrhs, _dptr(Bm), _dptr(y)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return y[:, 0] if B.ndim == 1 else y

    def schur_reduce_device(self, d_b_ptr, d_y_ptr, nrhs=1):
        return self._L.b200ldlt_schur_reduce_device(self._h, int(nrhs), C.c_void_p(d_b_ptr), C.c_void_p(d_y_ptr))

    def schur_expand(self, B, XS):
        """x with x_S = xs and x_E = A_EE^-1 (b_E - A_ES xs) for the columns of B (dim [x nrhs]) and XS (m [x nrhs]).
        Raises on a refusal."""
        B = np.asarray(B, dtype=np.float64)
        Bm = np.asfortranarray(B.reshape(self.dim, -1, order="F"))
        nrhs, m = Bm.shape[1], self._sc_m
        Xs = np.asfortranarray(np.asarray(XS, dtype=np.float64).reshape(m, nrhs, order="F"))
        x = np.zeros((self.dim, nrhs), order="F")
        if self._L.b200ldlt_schur_expand(self._h, nrhs, _dptr(Bm), _dptr(Xs), _dptr(x)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return x[:, 0] if B.ndim == 1 else x

    def schur_expand_device(self, d_b_ptr, d_xs_ptr, d_x_ptr, nrhs=1):
        return self._L.b200ldlt_schur_expand_device(self._h, int(nrhs), C.c_void_p(d_b_ptr), C.c_void_p(d_xs_ptr),
                                                    C.c_void_p(d_x_ptr))

    @staticmethod
    def _errors_dict(out, one):
        d = {k: np.array([getattr(o, k) for o in out], dtype=np.int32 if t is C.c_int else np.float64)
             for k, t in Errors._fields_}
        return {k: v[0] for k, v in d.items()} if one else d

    def error_analysis(self, B, X, cond=True):
        """Componentwise error analysis of the solutions X of A X = B (dim or dim x nrhs; b200ldlt_error_analysis): a dict
        of per-column arrays (scalars for 1-D input) -- anorm, xnorm, rnorm, omega1, omega2, cond1, cond2, ferr, n_i2,
        nprod.  cond=False: the norms and backward errors only (cond1 = cond2 = ferr = -1).  Raises on a refusal."""
        B = np.asarray(B, dtype=np.float64)
        one = B.ndim == 1
        Bm = np.asfortranarray(B.reshape(self.dim, -1, order="F"))
        Xm = np.asfortranarray(np.asarray(X, dtype=np.float64).reshape(self.dim, -1, order="F"))
        assert Xm.shape == Bm.shape
        nrhs = Bm.shape[1]
        out = (Errors * max(nrhs, 1))()
        if self._L.b200ldlt_error_analysis(self._h, nrhs, _dptr(Bm), _dptr(Xm), int(bool(cond)), out) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return self._errors_dict(out[:nrhs], one)

    def error_analysis_device(self, d_b_ptr, d_x_ptr, nrhs=1, cond=True):
        """The same on device arrays of dim x nrhs doubles.  Returns (status, dict of per-column arrays)."""
        out = (Errors * max(int(nrhs), 1))()
        st = self._L.b200ldlt_error_analysis_device(self._h, int(nrhs), C.c_void_p(d_b_ptr), C.c_void_p(d_x_ptr),
                                                    int(cond), out)
        return st, self._errors_dict(out[:int(nrhs)], False)

    @staticmethod
    def _refined_dict(out):
        return {k: np.array([getattr(o, k) for o in out], dtype=np.int32 if t is C.c_int else np.float64)
                for k, t in Refined._fields_}

    def solve_refined(self, B, max_steps=10, tol=2.0 ** -52):
        """Solve A X = B (dim or dim x nrhs) with iterative refinement until the componentwise backward error is <= tol,
        stops improving or max_steps corrections are taken (b200ldlt_solve_refined).  Returns (X, dict of per-column
        arrays: omega_first, omega1, omega2, steps, status, nres).  Raises on a refusal."""
        B = np.asarray(B, dtype=np.float64)
        Bm = np.asfortranarray(B.reshape(self.dim, -1, order="F"))
        nrhs = Bm.shape[1]
        X = np.zeros_like(Bm, order="F")
        out = (Refined * max(nrhs, 1))()
        if self._L.b200ldlt_solve_refined(self._h, nrhs, _dptr(Bm), _dptr(X), int(max_steps), float(tol),
                                          out) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return X.reshape(B.shape, order="F"), self._refined_dict(out[:nrhs])

    def solve_refined_device(self, d_b_ptr, d_x_ptr, nrhs=1, max_steps=10, tol=2.0 ** -52):
        """The same on device arrays of dim x nrhs doubles (x written).  Returns (status, dict of per-column arrays)."""
        out = (Refined * max(int(nrhs), 1))()
        st = self._L.b200ldlt_solve_refined_device(self._h, int(nrhs), C.c_void_p(d_b_ptr), C.c_void_p(d_x_ptr),
                                                   int(max_steps), float(tol), out)
        return st, self._refined_dict(out[:int(nrhs)])

    # Defaults from tools/bench_gmres.py (DESIGN section 7 item 16): inner_tol 1e-10 was the fastest or tied on every
    # system measured -- 1e-6 made the shifted systems take a second cycle, 1e-14 added a step everywhere; restart 20 was
    # never reached there and bounds V and Z at 41 vectors per column of a block.
    @staticmethod
    def _gmres_dict(out):
        return {k: np.array([getattr(o, k) for o in out], dtype=np.int32 if t is C.c_int else np.float64)
                for k, t in Gmres._fields_}

    def solve_gmres(self, B, vals=None, restart=20, max_cycles=10, tol=2.0 ** -52, inner_tol=1e-10):
        """Solve A_op X = B (dim or dim x nrhs) by FGMRES preconditioned by the factors, stopped like solve_refined
        (b200ldlt_solve_gmres).  vals: the nonzeros values of A_op in triplet order (None: the factored matrix).
        Returns (X, dict of per-column arrays: omega_first, omega1, omega2, cycles, iters, status, nres).  Raises on a
        refusal."""
        B = np.asarray(B, dtype=np.float64)
        Bm = np.asfortranarray(B.reshape(self.dim, -1, order="F"))
        nrhs = Bm.shape[1]
        X = np.zeros_like(Bm, order="F")
        pv = None
        if vals is not None:
            vals = np.ascontiguousarray(vals, dtype=np.float64)
            pv = _dptr(vals)
        out = (Gmres * max(nrhs, 1))()
        if self._L.b200ldlt_solve_gmres(self._h, nrhs, _dptr(Bm), _dptr(X), pv, int(restart), int(max_cycles),
                                        float(tol), float(inner_tol), out) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return X.reshape(B.shape, order="F"), self._gmres_dict(out[:nrhs])

    def solve_gmres_device(self, d_b_ptr, d_x_ptr, nrhs=1, d_vals_ptr=None, restart=20, max_cycles=10,
                           tol=2.0 ** -52, inner_tol=1e-10):
        """The same on device arrays of dim x nrhs doubles (x written) and, if given, nonzeros device values.  Returns
        (status, dict of per-column arrays)."""
        out = (Gmres * max(int(nrhs), 1))()
        st = self._L.b200ldlt_solve_gmres_device(self._h, int(nrhs), C.c_void_p(d_b_ptr), C.c_void_p(d_x_ptr),
                                                 C.c_void_p(d_vals_ptr) if d_vals_ptr else None, int(restart),
                                                 int(max_cycles), float(tol), float(inner_tol), out)
        return st, self._gmres_dict(out[:int(nrhs)])

    def condest(self):
        """(kappa1, anorm1, ainv1, nprod): the 1-norm condition estimate ||A||_1 est||M||_1 (b200ldlt_condest).  Raises
        on a refusal."""
        k, a, m, p = C.c_double(), C.c_double(), C.c_double(), C.c_int()
        if self._L.b200ldlt_condest(self._h, C.byref(k), C.byref(a), C.byref(m), C.byref(p)) != SYMSOLVER_SUCCESS:
            raise RuntimeError(self.last_error())
        return k.value, a.value, m.value, p.value

    def device_ptr(self, name):
        """Device address of a named array of the handle (b200ldlt_device_ptr: "scale", "x", "cbv", ...), 0 if none."""
        return self._L.b200ldlt_device_ptr(self._h, name.encode()) or 0

    def assemble_augsys_device(self, n_x, n_s, n_c, nnz_w, nnz_jc, nnz_jd, W=0, W_factor=1.0, D_x=0, delta_x=0.0, D_s=0,
                               delta_s=0.0, J_c=0, D_c=0, delta_c=0.0, J_d=0, D_d=0, delta_d=0.0):
        """Device pointers (ints, 0 = absent) of the blocks of the augmented system -> the handle's device value array
        (b200ldlt_assemble_augsys_device); follow with refactor()."""
        a = AugSys(n_x, n_s, n_c, n_s, nnz_w, nnz_jc, nnz_jd, W or None, W_factor, D_x or None, delta_x, D_s or None, delta_s,
                   J_c or None, D_c or None, delta_c, J_d or None, D_d or None, delta_d)
        return self._L.b200ldlt_assemble_augsys_device(self._h, C.byref(a))

    def solve_refine_device(self, d_rhs_ptr, min_steps=1, max_steps=10, tol=1e-10):
        steps, ratio = C.c_int(0), C.c_double(0.0)
        st = self._L.b200ldlt_solve_refine_device(self._h, C.c_void_p(d_rhs_ptr), int(min_steps), int(max_steps), float(tol),
                                                  C.byref(steps), C.byref(ratio))
        return st, steps.value, ratio.value

    def analyse_now(self, vals=None):
        return self._L.b200ldlt_analyse_now(self._h, None if vals is None else _dptr(np.ascontiguousarray(vals)))

    def residual(self, x, b):
        r, xi, bi = C.c_double(), C.c_double(), C.c_double()
        st = self._L.b200ldlt_residual(self._h, _dptr(x), _dptr(b), C.byref(r), C.byref(xi), C.byref(bi))
        if st != 0:
            raise RuntimeError(self.last_error())
        return r.value, xi.value, bi.value

    def info(self):
        i = Info()
        self._L.b200ldlt_get_info(self._h, C.byref(i))
        return i.as_dict()

    def symbolic(self, name):
        n = self._L.b200ldlt_symbolic_array(self._h, name.encode(), None, 0)
        if n < 0:
            raise KeyError(name)
        out = np.zeros(max(n, 1), dtype=np.int64)
        self._L.b200ldlt_symbolic_array(self._h, name.encode(), out.ctypes.data_as(C.POINTER(C.c_int64)), n)
        return out[:n]

    def last_error(self):
        return self._L.b200ldlt_last_error(self._h).decode()

    def close(self):
        if getattr(self, "_h", None):
            self._L.b200ldlt_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()
