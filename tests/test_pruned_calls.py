"""The three calls that run pruned sweeps -- b200ldlt_sparse_fwd_solve, b200ldlt_inverse_entries and
b200ldlt_sparse_solve -- share one per-analysis plan (per-front indices, marks, last run sets) and one list staging that
grows to the largest call.  Interleaved on one handle through both entry points, with sizes that grow and shrink, every
call must give the bits and launch count of the same call on a fresh handle, and leave the other calls' run sets as they
were; the same after a re-analysis of the handle."""
import numpy as np
import pytest

from ipopt_b200 import SYMSOLVER_SUCCESS

from test_partial_solve import assert_bits, factored
from test_sparse_fwd_solve import ALL_SYSTEMS, sfs
from test_inverse_entries import entries
from test_sparse_solve import sps

RUN_SETS = ("sparse_run_set", "inverse_run_set", "sparse_solve_fwd_run_set", "sparse_solve_bwd_run_set")
OWN = {"sfs": {"sparse_run_set"}, "inv": {"inverse_run_set"},
       "sps": {"sparse_solve_fwd_run_set", "sparse_solve_bwd_run_set"}}


def sequence(n, seed):
    """(kind, arguments) of calls whose sizes grow and shrink, so the shared staging grows partway through"""
    rng = np.random.default_rng(seed)

    def pick(k):
        return np.sort(rng.choice(n, min(k, n), replace=False)).astype(np.int32)

    blk = pick(24)
    bi, bj = np.meshgrid(blk, blk, indexing="ij")
    b50, b3 = pick(50), pick(3)
    return [
        ("sfs", (pick(1), rng.standard_normal(1))),
        ("inv", (pick(1), pick(1))),
        ("sps", (b3, rng.standard_normal((1, 3)), pick(2))),
        ("inv", (bi.ravel(), bj.ravel())),
        ("sfs", (b50, rng.standard_normal(len(b50)))),
        ("sps", (b50, rng.standard_normal((13, len(b50))), pick(n // 4))),
        ("sfs", (b3, rng.standard_normal(3))),
        ("sps", (None, rng.standard_normal((2, n)), pick(5))),
        ("inv", (blk[:3], blk[3:6])),
        ("sps", (b3, rng.standard_normal((1, 3)), None)),
        ("sps", (pick(n // 2), rng.standard_normal((3, min(n // 2, n))), pick(n // 2))),
        ("sfs", (pick(n // 3), rng.standard_normal(min(n // 3, n)))),
        ("inv", (pick(1), pick(1))),
        ("sps", (None, rng.standard_normal((1, n)), None)),
    ]


def call(s, kind, args, device):
    if kind == "sfs":
        return list(sfs(s, args[0], args[1], device))
    if kind == "inv":
        return [entries(s, args[0], args[1], device)]
    return [sps(s, args[0], args[1], args[2], device)]


def run_sets(s):
    return {name: s.symbolic(name) for name in RUN_SETS}


def check_sequence(s, args, seed, tag):
    for q, (kind, a) in enumerate(sequence(s.dim, seed)):
        for device in (False, True):
            before = run_sets(s)
            got = call(s, kind, a, device)
            launches = s.info()["launches_solve"]
            after = run_sets(s)
            fresh = factored(*args)
            want = call(fresh, kind, a, device)
            assert launches == fresh.info()["launches_solve"], (tag, q, kind, device)
            for x, y in zip(got, want):
                assert_bits(np.asarray(x, np.float64), np.asarray(y, np.float64), (tag, q, kind, device))
            fresh_sets = run_sets(fresh)
            fresh.close()
            for name in RUN_SETS:
                if name in OWN[kind]:
                    assert np.array_equal(after[name], fresh_sets[name]), (tag, q, kind, device, name)
                else:
                    assert np.array_equal(after[name], before[name]), (tag, q, kind, device, name, "touched")


@pytest.mark.gpu
@pytest.mark.parametrize("system", ["MBndryCntrl1_30", "mbndry400"])
def test_interleaved_calls_share_plan_and_staging(system):
    args = ALL_SYSTEMS[system]()
    s = factored(*args)
    check_sequence(s, args, 5, system)
    # a re-analysis replaces the plan: no run sets until the next calls, then the same sequence again
    dim, irn, jcn, val = args
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS, s.last_error()
    for name, v in run_sets(s).items():
        assert len(v) == 0, (system, name)
    check_sequence(s, args, 6, (system, "reanalysed"))
    s.close()
