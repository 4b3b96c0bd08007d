"""Blocked multi-right-hand-side solves (b200ldlt_solve / b200ldlt_solve_device with nrhs > 1, solve_multi.cu): every
column of a blocked solve is bit-identical to a single-column solve of that column, under every solve switch, across
state changes of the handle, and through the reference's IP loop in L-BFGS mode (the caller that solves several columns
per call)."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_SUCCESS
from ipopt_b200.kkt import lukvle1_kkt, mbndry_kkt, random_kkt, to_scipy
from oracle_api import OracleLdlt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
DRIVER = os.path.join(ROOT, "tests", "driver", "ipopt_driver")
NRHS = (2, 3, 5, 6, 8, 9, 13)


def golden_system(case):
    z = np.load(os.path.join(G, case + "_kkt.npz"))
    k = min(int(f[4:]) for f in z.files if f.startswith("val_"))
    return int(z["dim"]), z["irn"], z["jcn"], z["val_%d" % k], int(z["neg_%d" % k])


SYSTEMS = {
    "mbndry70": lambda: mbndry_kkt(70, sigma_spread=3.0, seed=5),
    "lukvle1_2000": lambda: lukvle1_kkt(2000, sigma_spread=2.0, seed=6),
    "random": lambda: random_kkt(400, 150, density=0.02, seed=8),
    "golden_MBndryCntrl1_30": lambda: golden_system("MBndryCntrl1_30"),
}


def factored(dim, irn, jcn, val, nc):
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, nc)
    assert st == SYMSOLVER_SUCCESS and neg == nc, s.info()
    return s


def rhs_block(dim, nrhs, seed):
    return np.random.default_rng(seed).standard_normal((nrhs, dim))   # column c = row c: column-major dim x nrhs


def assert_blocked_equals_columns(s, B, device):
    """solve(nrhs) against nrhs separate solve(1) calls, compared as raw 64-bit patterns."""
    nrhs, dim = B.shape
    if device:
        import torch
        X = torch.tensor(B.ravel(), dtype=torch.float64, device="cuda")
        assert s.solve_device(X.data_ptr(), nrhs) == SYMSOLVER_SUCCESS
        X = X.cpu().numpy()
        cols = []
        for c in range(nrhs):
            x = torch.tensor(B[c], dtype=torch.float64, device="cuda")
            assert s.solve_device(x.data_ptr(), 1) == SYMSOLVER_SUCCESS
            cols.append(x.cpu().numpy())
    else:
        X = B.ravel().copy()
        assert s.solve(X, nrhs) == SYMSOLVER_SUCCESS
        cols = []
        for c in range(nrhs):
            x = B[c].copy()
            assert s.solve(x, 1) == SYMSOLVER_SUCCESS
            cols.append(x)
    X = X.reshape(nrhs, dim)
    for c in range(nrhs):
        diff = np.flatnonzero(X[c].view(np.uint64) != cols[c].view(np.uint64))
        assert diff.size == 0, (nrhs, c, diff.size, diff[:5])


@pytest.mark.parametrize("env", [
    {}, {"B200_SOLVE_DIRECT": "0"}, {"B200_SOLVE_DIRECT": "1"}, {"B200_SOLVE_DIRECT": "4"}, {"B200_SOLVE_NOPAIR": "1"},
    {"B200_SOLVE_BLOCK": "2"}, {"B200_SOLVE_BLOCK": "4"},
])
@pytest.mark.parametrize("system", sorted(SYSTEMS))
def test_blocked_solve_bit_identical_to_single_column(system, env, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dim, irn, jcn, val, nc = SYSTEMS[system]()
    s = factored(dim, irn, jcn, val, nc)
    for nrhs in NRHS:
        B = rhs_block(dim, nrhs, nrhs)
        assert_blocked_equals_columns(s, B, device=False)
        assert_blocked_equals_columns(s, B, device=True)
    s.close()


@pytest.mark.parametrize("block", [None, "1"])
def test_blocked_path_runs(block, monkeypatch):
    """nrhs = 8 in one block pays the launches of one single-column solve; B200_SOLVE_BLOCK=1 restores the column loop."""
    if block is not None:
        monkeypatch.setenv("B200_SOLVE_BLOCK", block)
    dim, irn, jcn, val, nc = mbndry_kkt(70, sigma_spread=3.0, seed=5)
    s = factored(dim, irn, jcn, val, nc)
    x = rhs_block(dim, 1, 0).ravel()
    assert s.solve(x, 1) == SYMSOLVER_SUCCESS
    one = s.info()["launches_solve"]
    X = rhs_block(dim, 8, 1).ravel()
    assert s.solve(X, 8) == SYMSOLVER_SUCCESS
    eight = s.info()["launches_solve"]
    if block is None:
        assert one > 0 and eight == one, (one, eight)
    else:
        assert eight == 8 * one, (one, eight)
    s.close()


def test_state_across_interleaving_refactor_and_reanalysis():
    dim, irn, jcn, val, nc = mbndry_kkt(40, sigma_spread=3.0, seed=3)
    s = factored(dim, irn, jcn, val, nc)

    def check(tag):
        for rep in range(2):                 # flags are epoch-stamped, not cleared: twice each, interleaved
            for nrhs in (5, 1, 8, 2):
                B = rhs_block(s.dim, nrhs, 100 + nrhs + rep)
                if nrhs == 1:
                    x = B.ravel().copy()
                    assert s.solve(x, 1) == SYMSOLVER_SUCCESS, tag
                else:
                    assert_blocked_equals_columns(s, B, device=bool(rep))

    check("first")
    v2 = val.copy()
    v2[: len(v2) // 3] *= 1.25
    s.GetValuesArrayPtr()[:] = v2
    assert s.factor(True, nc) == (SYMSOLVER_SUCCESS, nc)
    check("new values")
    assert s.IncreaseQuality()                  # (no lifted pivots here: raises the pivot threshold)
    assert s.refactor(True, nc) == (SYMSOLVER_SUCCESS, nc)
    check("increase_quality")
    assert s.analyse_now(v2) == SYMSOLVER_SUCCESS
    assert s.refactor(True, nc) == (SYMSOLVER_SUCCESS, nc)
    check("analyse_now")
    dim3, irn3, jcn3, val3, nc3 = lukvle1_kkt(900, sigma_spread=2.0, seed=9)
    assert s.InitializeStructure(dim3, len(irn3), irn3, jcn3) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val3
    assert s.factor(True, nc3) == (SYMSOLVER_SUCCESS, nc3)
    check("new pattern")
    s.close()


def test_state_after_reanalysis_by_increase_quality(capfd):
    """A tridiagonal matrix with tiny diagonal entries makes the factorisation lift pivots, so increase_quality schedules a
    re-analysis on the current values: the next factorisation re-runs it and the blocked state is rebuilt for the new plan."""
    n = 2000
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    s = B200Ldlt(verbose=1)
    assert s.InitializeStructure(n, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == SYMSOLVER_SUCCESS
    assert s.info()["num_forced"] > 0
    for nrhs in (6, 3):
        assert_blocked_equals_columns(s, rhs_block(n, nrhs, nrhs), device=False)
    capfd.readouterr()
    assert s.IncreaseQuality()
    assert s.refactor(False, 0)[0] == SYMSOLVER_SUCCESS
    for nrhs in (6, 3):
        assert_blocked_equals_columns(s, rhs_block(n, nrhs, 10 + nrhs), device=True)
    err = capfd.readouterr().err
    assert "[b200ldlt] analyse:" in err and "[b200ldlt] blocked solve:" in err, err[-2000:]
    s.close()


@pytest.mark.parametrize("gen,arg,kw", [
    (mbndry_kkt, 60, dict(sigma_spread=2.0, seed=2)), (lukvle1_kkt, 3000, dict(sigma_spread=2.0, seed=3)),
])
def test_blocked_solve_vs_oracle(gen, arg, kw):
    dim, irn, jcn, val, nc = gen(arg, **kw)
    nrhs = 9
    B = rhs_block(dim, nrhs, 4)
    o = OracleLdlt()
    o.InitializeStructure(dim, len(irn), irn, jcn)
    o.GetValuesArrayPtr()[:] = val
    assert o.factor(False, 0)[0] == 0
    XO = B.ravel().copy()
    o.solve(XO, nrhs)
    o.close()
    s = factored(dim, irn, jcn, val, nc)
    X = B.ravel().copy()
    assert s.solve(X, nrhs) == SYMSOLVER_SUCCESS
    s.close()
    A = to_scipy(dim, irn, jcn, val)
    aA = abs(A).max()
    for c in range(nrhs):
        x, xo, b = X[c * dim:(c + 1) * dim], XO[c * dim:(c + 1) * dim], B[c]
        res = np.abs(A @ x - b).max() / (aA * np.abs(x).max() + np.abs(b).max())
        res_o = np.abs(A @ xo - b).max() / (aA * np.abs(xo).max() + np.abs(b).max())
        assert res < 1e-12, (c, res)
        assert np.linalg.norm(x - xo) <= max(1e-8, 1e3 * res_o) * np.linalg.norm(xo), c


def _driver(problem, N, tmp_path, tag, env_extra):
    if not os.path.exists(DRIVER):
        pytest.skip("tests/driver/ipopt_driver not built (needs the reference artefacts in oracle/_ref at build time)")
    js, fin = str(tmp_path / (tag + ".json")), str(tmp_path / (tag + ".bin"))
    env = dict(os.environ, OMP_NUM_THREADS=str(min(16, os.cpu_count() or 1)), **env_extra)
    cmd = [DRIVER, "--backend", "b200", "--problem", problem, "--N", str(N), "--print-level", "0", "--json", js,
           "--final", fin, "--opt", "hessian_approximation=limited-memory"]
    p = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=1500)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    with open(fin, "rb") as f:
        raw = f.read()
    n, m = struct.unpack("ii", raw[:8])
    obj, = struct.unpack("d", raw[8:16])
    vec = np.frombuffer(raw[16:], dtype=np.float64)
    return json.load(open(js)), raw, dict(obj=obj, x=vec[:n], z_L=vec[n:2 * n], z_U=vec[2 * n:3 * n], lam=vec[3 * n:3 * n + m])


@pytest.mark.parametrize("problem,N,tag", [
    ("MDistCntrl3a", 20, "MDistCntrl3a_20_limitedmemory"), ("LukVlE1", 200, "LukVlE1_200_limitedmemory"),
])
def test_ip_loop_lbfgs_blocked_equals_column_loop(problem, N, tag, tmp_path):
    """L-BFGS mode solves up to 2 x limited_memory_max_history columns per MultiSolve: the blocked solve and the column loop
    give the same run, byte for byte, and both match the reference run."""
    runs = [_driver(problem, N, tmp_path, name, env) for name, env in (("blocked", {}), ("loop", {"B200_SOLVE_BLOCK": "1"}))]
    (sa, ra, fa), (sb, rb, fb) = runs
    assert sa["n_rhs"] > sa["n_solve"]            # the run did solve several columns per call
    for key in ("status", "iterations", "n_factor", "n_solve", "n_rhs", "n_wrong_inertia"):
        assert sa[key] == sb[key], key
    assert ra == rb
    gold = np.load(os.path.join(G, tag + "_final.npz"))
    for summ, fin in ((sa, fa), (sb, fb)):
        assert summ["status"] == 0
        assert summ["iterations"] == int(gold["iterations"])
        assert summ["n_factor"] == int(gold["n_factor"]) and summ["n_wrong_inertia"] == int(gold["n_wrong_inertia"])
        assert abs(summ["n_solve"] - int(gold["n_solve"])) <= 4 and abs(summ["n_rhs"] - int(gold["n_rhs"])) <= 12
        assert abs(fin["obj"] - float(gold["obj"])) <= 1e-10 * max(abs(float(gold["obj"])), 1e-12)
        for key in ("x", "lam", "z_L", "z_U"):
            ref = gold[key]
            scale = max(np.abs(ref).max(), 1e-300)
            assert np.abs(fin[key] - ref).max() <= 1e-8 * scale, key
