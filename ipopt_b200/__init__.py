"""ipopt_b200 -- H100-native KKT (symmetric indefinite LDL^T) backend for coin-or/Ipopt.

The product is the C-ABI shared library ``ipopt_b200/lib/libb200ldlt.so`` (see ``include/b200ldlt.h``);
this package holds its sources (``csrc/``), the Ipopt-side plugin (``plugin/``) and a thin ctypes
mirror of the reference's ``SparseSymLinearSolverInterface`` used by the tests and ``bench.py``.
"""
from .capi import (B200Ldlt, SymbolicAnalysis, lib_path, load_library, SYMSOLVER_SUCCESS, SYMSOLVER_SINGULAR,
                   SYMSOLVER_WRONG_INERTIA, SYMSOLVER_CALL_AGAIN, SYMSOLVER_FATAL_ERROR)

__all__ = ["B200Ldlt", "SymbolicAnalysis", "lib_path", "load_library", "SYMSOLVER_SUCCESS", "SYMSOLVER_SINGULAR",
           "SYMSOLVER_WRONG_INERTIA", "SYMSOLVER_CALL_AGAIN", "SYMSOLVER_FATAL_ERROR"]
