"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle, the golden fixtures
captured at the reference's SparseSymLinearSolverInterface boundary, and size-independent properties at
BASELINE.json's full sizes.  Tolerances (floating point): solutions within 1e-8 relative of the oracle's
(north_star: "<= 1e-8 relative"), inertia exact, residuals at rounding level."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from ipopt_b200 import B200Ldlt, SYMSOLVER_SINGULAR, SYMSOLVER_SUCCESS, SYMSOLVER_WRONG_INERTIA
from ipopt_b200.kkt import lukvle1_kkt, mbndry_kkt, random_kkt, to_scipy
from oracle_api import OracleLdlt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
DRIVER = os.path.join(ROOT, "tests", "driver", "ipopt_driver")
RTOL = 1e-8
# raw (unrefined) GPU-vs-golden solution differences of the KKT snapshots: bound per case (measured values are printed by
# test_golden_kkt_snapshots with -s; the late-iteration systems have condition numbers ~1e12-1e16)
RAW_BOUND = {"hs071_0": 1e-5, "LukVlE1_1000": 1e-5, "MBndryCntrl1_30": 1e-5, "MDistCntrl3a_25": 1e-5}
raw_seen = {}


def gpu_solver(dim, irn, jcn, **kw):
    s = B200Ldlt(**kw)
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
    return s


def oracle_solution(dim, irn, jcn, val, b):
    o = OracleLdlt()
    o.InitializeStructure(dim, len(irn), irn, jcn)
    o.GetValuesArrayPtr()[:] = val
    st, neg = o.factor(False, 0)
    assert st == 0
    x = b.copy()
    o.solve(x, len(b) // dim)
    return x, neg


def scaled_residual(dim, irn, jcn, val, x, b):
    A = to_scipy(dim, irn, jcn, val)
    r = A @ x - b
    return np.abs(r).max() / (abs(A).max() * np.abs(x).max() + np.abs(b).max())


@pytest.mark.parametrize("case", ["hs071_0", "LukVlE1_1000", "MBndryCntrl1_30", "MDistCntrl3a_25"])
def test_golden_kkt_snapshots(case):
    z = np.load(os.path.join(G, case + "_kkt.npz"))
    ks = sorted(int(k[4:]) for k in z.files if k.startswith("val_"))
    dim, irn, jcn = int(z["dim"]), z["irn"], z["jcn"]
    s = gpu_solver(dim, irn, jcn)
    for k in ks:
        s.GetValuesArrayPtr()[:] = z["val_%d" % k]
        rhs = z["rhs_%d" % k].copy()
        nrhs = len(rhs) // dim
        st = s.MultiSolve(True, irn, jcn, nrhs, rhs, True, int(z["neg_%d" % k]))
        assert st == SYMSOLVER_SUCCESS, (case, k, s.info())
        assert s.NumberOfNegEVals() == int(z["neg_%d" % k])
        ref = z["sol_%d" % k]
        b0 = z["rhs_%d" % k]
        assert scaled_residual(dim, irn, jcn, z["val_%d" % k], rhs[:dim], b0[:dim]) < 1e-13
        # Late-iteration KKT systems are very ill-conditioned (Sigma spans ~18 orders of magnitude), so two
        # backward-stable solvers differ by cond*eps in the RAW solution: that difference is bounded per snapshot below.
        # The quantity the reference's caller consumes is the solution after iterative refinement (PDFullSpaceSolver
        # refines every solve, IpPDFullSpaceSolver.cpp:256-346): compare after ONE refinement step in which EACH solver
        # corrects its OWN solution -- the golden one with the CPU oracle, the GPU one with the GPU solver.
        A = to_scipy(dim, irn, jcn, z["val_%d" % k])
        o = OracleLdlt()
        o.InitializeStructure(dim, len(irn), irn, jcn)
        o.GetValuesArrayPtr()[:] = z["val_%d" % k]
        assert o.factor(False, 0)[0] == 0
        def refine(x, solve):
            out = x.copy()
            for c in range(nrhs):
                r = b0[c * dim:(c + 1) * dim] - A @ x[c * dim:(c + 1) * dim]
                assert solve(r) == SYMSOLVER_SUCCESS
                out[c * dim:(c + 1) * dim] += r
            return out
        xg, xo = refine(rhs, s.solve), refine(ref, lambda r: o.solve(r, 1))
        o.close()
        assert np.linalg.norm(xg - xo) <= RTOL * np.linalg.norm(xo), (case, k)
        raw = np.linalg.norm(rhs - ref) / np.linalg.norm(ref)
        raw_seen[(case, k)] = raw
        assert raw <= RAW_BOUND[case], (case, k, raw)   # raw (unrefined) solutions: conditioning-limited, bound per case
    s.close()


@pytest.mark.parametrize("gen,arg,kw", [
    (mbndry_kkt, 12, dict(sigma_spread=4.0, seed=1)), (mbndry_kkt, 60, dict(sigma_spread=2.0, seed=2)),
    (mbndry_kkt, 40, dict(w_zero=True)), (lukvle1_kkt, 3000, dict(sigma_spread=2.0, seed=3)),
    (lukvle1_kkt, 500, dict(w_zero=True)), (mbndry_kkt, 25, dict(sigma_spread=2.0, delta_c=1e-8, delta_x=1e-4, seed=4)),
])
def test_synthetic_vs_oracle(gen, arg, kw):
    dim, irn, jcn, val, nc = gen(arg, **kw)
    b = np.random.default_rng(7).standard_normal(dim)
    xo, nego = oracle_solution(dim, irn, jcn, val, b)
    s = gpu_solver(dim, irn, jcn)
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, nego)
    assert st == SYMSOLVER_SUCCESS and neg == nego, s.info()
    x = b.copy()
    assert s.solve(x) == SYMSOLVER_SUCCESS
    assert scaled_residual(dim, irn, jcn, val, x, b) < 1e-12
    # the forward error is conditioning-limited for both solvers: compare through the residual-corrected bound
    assert np.linalg.norm(x - xo) <= max(RTOL, 1e3 * scaled_residual(dim, irn, jcn, val, xo, b)) * np.linalg.norm(xo)
    s.close()


@pytest.mark.parametrize("env", [
    {}, {"B200_SOLVE_DIRECT": "0"}, {"B200_SOLVE_DIRECT": "1"}, {"B200_SOLVE_DIRECT": "4"}, {"B200_SOLVE_NOPAIR": "1"},
    {"B200_NO_WARP2": "1"}, {"B200_NO_PDL": "1"}, {"B200_CB_AT_END": "1"}, {"B200_ONE_STREAM": "1"},
])
def test_kernel_variants_agree_with_oracle(env, monkeypatch):
    """Every A/B switch of the factor / solve pipelines (read once at b200ldlt_create: DESIGN.md section 2) selects another
    set of kernels for the same mathematics: bottom levels inside the subtrees vs by the direct kernel, one vs two subtrees
    per CTA, fronts 33..64 in registers vs shared memory, with / without programmatic dependent launch, Schur complement per
    panel vs per level, one vs five streams.  All of them must reproduce the oracle."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for gen, arg, kw in ((mbndry_kkt, 70, dict(sigma_spread=3.0, seed=5)), (lukvle1_kkt, 2000, dict(sigma_spread=2.0, seed=6))):
        dim, irn, jcn, val, nc = gen(arg, **kw)
        b = np.random.default_rng(11).standard_normal(dim)
        xo, nego = oracle_solution(dim, irn, jcn, val, b)
        s = gpu_solver(dim, irn, jcn)
        s.GetValuesArrayPtr()[:] = val
        st, neg = s.factor(True, nego)
        assert st == SYMSOLVER_SUCCESS and neg == nego, (env, s.info())
        for _ in range(2):          # (twice: the solve flags are epoch-stamped, not cleared)
            x = b.copy()
            assert s.solve(x) == SYMSOLVER_SUCCESS
            assert scaled_residual(dim, irn, jcn, val, x, b) < 1e-12, env
            assert np.linalg.norm(x - xo) <= max(RTOL, 1e3 * scaled_residual(dim, irn, jcn, val, xo, b)) * np.linalg.norm(xo), env
        s.close()


@pytest.mark.parametrize("seed", range(4))
def test_random_saddle_point_inertia_and_solution(seed):
    dim, irn, jcn, val, nc = random_kkt(150 + 40 * seed, 60 + 10 * seed, density=0.03, seed=seed)
    A = to_scipy(dim, irn, jcn, val).toarray()
    ev = np.linalg.eigvalsh(A)
    s = gpu_solver(dim, irn, jcn)
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, int((ev < 0).sum()))
    assert st == SYMSOLVER_SUCCESS and neg == int((ev < 0).sum())
    b = np.random.default_rng(seed).standard_normal(dim)
    x = b.copy()
    s.solve(x)
    xr = np.linalg.solve(A, b)
    assert np.linalg.norm(x - xr) <= RTOL * np.linalg.norm(xr)
    s.close()


def test_edge_cases_dim1_diagonal_duplicates_multirhs():
    # dim 1
    s = gpu_solver(1, np.array([1], np.int32), np.array([1], np.int32))
    s.GetValuesArrayPtr()[:] = [-4.0]
    st, neg = s.factor(True, 1)
    assert (st, neg) == (SYMSOLVER_SUCCESS, 1)
    x = np.array([2.0])
    s.solve(x)
    assert x[0] == -0.5
    s.close()
    # diagonal matrix given twice (duplicates are summed), entries in both triangles, 3 right-hand sides
    n = 50
    d = np.linspace(-3, 5, n)
    d[np.abs(d) < 0.2] = 1.0
    irn = np.concatenate([np.arange(1, n + 1), np.arange(1, n + 1), [1, 7]]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n + 1), [7, 1]]).astype(np.int32)
    val = np.concatenate([0.25 * d, 0.75 * d, [0.1, 0.2]])
    A = to_scipy(n, irn, jcn, val).toarray()
    assert abs(A[0, 6] - 0.3) < 1e-15
    s = gpu_solver(n, irn, jcn)
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, int((np.linalg.eigvalsh(A) < 0).sum()))
    assert st == SYMSOLVER_SUCCESS
    B = np.random.default_rng(0).standard_normal((3, n))   # 3 columns stored contiguously (column-major dim x 3)
    X = B.copy().ravel()
    assert s.MultiSolve(False, irn, jcn, 3, X, False, 0) == SYMSOLVER_SUCCESS
    for c in range(3):
        assert np.allclose(A @ X[c * n:(c + 1) * n], B[c], atol=1e-12)
    s.close()


def test_status_codes_singular_wrong_inertia_and_quality():
    dim, irn, jcn, val, nc = random_kkt(30, 10, density=0.1, seed=6)
    s = gpu_solver(dim, irn, jcn)
    s.GetValuesArrayPtr()[:] = val
    rhs = np.ones(dim)
    # wrong inertia: reported WITHOUT solving, negevals still set (caller reads it: IpPDFullSpaceSolver.cpp:541)
    st = s.MultiSolve(True, irn, jcn, 1, rhs, True, nc + 1)
    assert st == SYMSOLVER_WRONG_INERTIA and s.NumberOfNegEVals() == nc and np.all(rhs == 1.0)
    # IncreaseQuality raises the threshold up to the cap and then reports false; refactor reuses device values
    n_up = 0
    while s.IncreaseQuality():
        n_up += 1
    assert 1 <= n_up <= 8
    st, neg = s.refactor(True, nc)
    assert st == SYMSOLVER_SUCCESS and neg == nc
    x = rhs.copy()
    s.solve(x)
    assert scaled_residual(dim, irn, jcn, val, x, rhs) < 1e-13
    s.close()
    # exactly singular (two identical constraint rows)
    A = to_scipy(dim, irn, jcn, val).toarray()
    A[32, :] = A[31, :]
    A[:, 32] = A[:, 31]
    A[31, 31] = A[32, 32] = A[31, 32] = A[32, 31] = 0.0
    i, j = np.nonzero(np.tril(A))
    s = gpu_solver(dim, (i + 1).astype(np.int32), (j + 1).astype(np.int32))
    s.GetValuesArrayPtr()[:] = A[i, j]
    st, neg = s.factor(True, nc)
    assert st == SYMSOLVER_SINGULAR
    s.close()


def test_new_structure_on_same_handle_and_value_updates():
    s = B200Ldlt()
    for N in (8, 15):
        dim, irn, jcn, val, nc = mbndry_kkt(N, sigma_spread=1.0, seed=N)
        assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
        for rep in range(3):
            v = val.copy()
            v[:len(v) // 3] *= (1.0 + 0.1 * rep)
            s.GetValuesArrayPtr()[:] = v
            st, neg = s.factor(True, nc)
            assert st == SYMSOLVER_SUCCESS and neg == nc
            b = np.arange(1.0, dim + 1)
            x = b.copy()
            s.solve(x)
            assert scaled_residual(dim, irn, jcn, v, x, b) < 1e-13
    s.close()


@pytest.mark.parametrize("N", [400])
def test_full_size_properties_mbndry(N):
    """BASELINE.json config MBndryCntrl1 N=400 (KKT dim 321 600): inertia, residual, linearity, determinism."""
    dim, irn, jcn, val, nc = mbndry_kkt(N, sigma_spread=6.0, seed=11)
    assert dim == 321600 and len(irn) == 1283200
    s = gpu_solver(dim, irn, jcn)
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, nc)
    assert st == SYMSOLVER_SUCCESS and neg == nc == 160000
    rng = np.random.default_rng(5)
    b1, b2 = rng.standard_normal(dim), rng.standard_normal(dim)
    x1, x2, x12 = b1.copy(), b2.copy(), (b1 + 2.0 * b2)
    s.solve(x1); s.solve(x2); s.solve(x12)
    r, xi, bi = s.residual(x1, b1)
    assert r <= 1e-10 * (xi * 4.0 + bi)
    assert np.linalg.norm(x12 - (x1 + 2.0 * x2)) <= 1e-9 * np.linalg.norm(x12)   # linearity of the solve
    y = b1.copy()
    s.factor(True, nc)
    s.solve(y)
    assert np.array_equal(y, x1)   # bit-reproducible (no atomics on the data path)
    s.close()


def test_full_size_lukvle1():
    dim, irn, jcn, val, nc = lukvle1_kkt(50000, sigma_spread=3.0, seed=2)
    assert dim == 99998 and len(irn) == 349991
    b = np.random.default_rng(1).standard_normal(dim)
    xo, nego = oracle_solution(dim, irn, jcn, val, b)
    s = gpu_solver(dim, irn, jcn)
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, nego)
    assert st == SYMSOLVER_SUCCESS and neg == nego
    x = b.copy()
    s.solve(x)
    assert scaled_residual(dim, irn, jcn, val, x, b) < 1e-12
    assert np.linalg.norm(x - xo) <= max(RTOL, 1e3 * scaled_residual(dim, irn, jcn, val, xo, b)) * np.linalg.norm(xo)
    s.close()


# ---- end-to-end through the reference's own IP loop (driver binary built against oracle/_ref) -------
def _run_driver(backend, problem, N, tmp_path, opts=None, extra=()):
    if not os.path.exists(DRIVER):
        pytest.skip("tests/driver/ipopt_driver not built (needs the reference artefacts in oracle/_ref at build time)")
    js, fin = str(tmp_path / "r.json"), str(tmp_path / "f.bin")
    env = dict(os.environ, OMP_NUM_THREADS=str(min(16, os.cpu_count() or 1)),
               B200_HSLLIB=os.path.join(ROOT, "ipopt_b200", "lib", "libb200ldlt.so"))
    cmd = [DRIVER, "--backend", backend, "--problem", problem, "--N", str(N), "--print-level", "0", "--json", js, "--final", fin]
    for k, v in (opts or {}).items():
        cmd += ["--opt", "%s=%s" % (k, v)]
    cmd += list(extra)
    p = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=1500)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    with open(fin, "rb") as f:
        n, m = struct.unpack("ii", f.read(8))
        obj, = struct.unpack("d", f.read(8))
        vec = np.frombuffer(f.read(), dtype=np.float64)
    return json.load(open(js)), dict(obj=obj, x=vec[:n], z_L=vec[n:2 * n], z_U=vec[2 * n:3 * n], lam=vec[3 * n:3 * n + m])


@pytest.mark.parametrize("problem,N", [("hs071", 0), ("LukVlE1", 1000), ("MBndryCntrl1", 30), ("MDistCntrl3a", 25)])
def test_ip_loop_parity_small(problem, N, tmp_path):
    summ, fin = _run_driver("b200", problem, N, tmp_path)
    gold = np.load(os.path.join(G, "%s_%d_final.npz" % (problem, N)))
    assert summ["status"] == 0
    assert summ["iterations"] == int(gold["iterations"])          # north_star: same count +-1; we require equal here
    assert summ["n_factor"] == int(gold["n_factor"]) and summ["n_solve"] == int(gold["n_solve"])
    assert abs(fin["obj"] - float(gold["obj"])) <= 1e-10 * abs(float(gold["obj"]))
    for key in ("x", "lam", "z_L", "z_U"):
        ref = gold[key]
        scale = max(np.abs(ref).max(), 1e-300)
        assert np.abs(fin[key] - ref).max() <= RTOL * scale, key


def _control_tol(problem, N):
    """Dual-iterate tolerances from the committed oracle-vs-oracle control (tests/golden/runs/control_dual_spread.json,
    made by tests/golden/make_goldens_r2.py control): the SAME CPU oracle with another nested-dissection seed ends, through
    the reference's IP loop, this far from itself.  north_star's 1e-8 holds for x everywhere and for lambda / z wherever the
    control does not show a larger solver-to-solver spread; where it does (the multipliers of the Mittelmann boundary-control
    problems are only determined to tol/sigma_min(J) by the reference's termination test, and z = mu/slack of an active bound
    amplifies the 1e-10 agreement of x by 1/slack), the bar is 4x the control's own spread."""
    ctl = json.load(open(os.path.join(G, "runs", "control_dual_spread.json")))
    tol = {"x": RTOL, "lam": RTOL, "z_L": RTOL, "z_U": RTOL}
    for r in ctl["runs"]:
        if r["problem"] == problem and r["N"] == N:
            for key in ("lam", "z_L", "z_U"):
                tol[key] = max(tol[key], 4.0 * r["spread"][key])
    return tol


def _rel_diff(fg, fo_sample, stride=1):
    zscale = max(float(fo_sample["z_L_absmax"]), float(fo_sample["z_U_absmax"]), 1e-300)
    rel = {}
    for key in ("x", "lam", "z_L", "z_U"):
        scale = zscale if key.startswith("z_") else max(float(fo_sample[key + "_absmax"]), 1e-300)
        rel[key] = float(np.abs(fg[key][::stride] - fo_sample[key]).max() / scale)
    return rel


@pytest.mark.parametrize("problem,N", [("LukVlE1", 50000), ("MBndryCntrl1", 400)])
def test_ip_loop_parity_full_size(problem, N, tmp_path):
    """GPU backend vs the CPU oracle, both driving the reference's unmodified IP loop on this box."""
    sg, fg = _run_driver("b200", problem, N, tmp_path)
    gold = json.load(open(os.path.join(G, "runs", "oracle_%s_%d.json" % (problem, N))))
    assert sg["status"] == 0 and sg["n_singular"] == 0
    assert abs(sg["iterations"] - gold["iterations"]) <= 1
    assert abs(sg["objective"] - gold["objective"]) <= 1e-8 * abs(gold["objective"])
    so, fo = _run_driver("oracle", problem, N, tmp_path)
    assert so["iterations"] == gold["iterations"]
    tol = _control_tol(problem, N)
    sample = {k: fo[k] for k in ("x", "lam", "z_L", "z_U")}
    sample.update({k + "_absmax": np.abs(fo[k]).max() if len(fo[k]) else 0.0 for k in ("x", "lam", "z_L", "z_U")})
    rel = _rel_diff(fg, sample)
    print("final-iterate max-norm relative differences GPU vs oracle:", rel, "tolerances:", tol)
    for key in ("x", "lam", "z_L", "z_U"):
        assert rel[key] <= tol[key], (key, rel, tol)


@pytest.mark.parametrize("problem,N", [("MDistCntrl3a", 600), ("MBndryCntrl1", 800)])
def test_ip_loop_parity_baseline_configs_4_and_5(problem, N, tmp_path):
    """BASELINE.json configs 4 (MDistCntrl3a N=600, KKT dim 1 080 000) and 5 (MBndryCntrl1 N=800, dim 1 283 200) on one GPU
    through the reference's IP loop, against the committed oracle run (iteration count, objective, every 97th entry of the
    final x / lambda / z: tests/golden/<case>_final_sample.npz made by make_goldens_r2.py full)."""
    sg, fg = _run_driver("b200", problem, N, tmp_path)
    gold = json.load(open(os.path.join(G, "runs", "oracle_%s_%d.json" % (problem, N))))
    samp = np.load(os.path.join(G, "%s_%d_final_sample.npz" % (problem, N)))
    assert sg["status"] == 0 and sg["n_singular"] == 0
    assert abs(sg["iterations"] - gold["iterations"]) <= 1
    assert sg["n_wrong_inertia"] == gold["n_wrong_inertia"]
    assert abs(sg["objective"] - gold["objective"]) <= 1e-8 * abs(gold["objective"])
    tol = _control_tol(problem, N)
    rel = _rel_diff(fg, samp, stride=int(samp["stride"]))
    print("final-iterate max-norm relative differences GPU vs oracle (sampled):", rel, "tolerances:", tol,
          "factor ms/call %.2f solve ms/call %.2f" % (1e3 * sg["t_factor_s"] / max(sg["n_factor"] - 1, 1), 1e3 * sg["t_solve_s"] / max(sg["n_solve"], 1)))
    for key in ("x", "lam", "z_L", "z_U"):
        assert rel[key] <= tol[key], (key, rel, tol)


@pytest.mark.parametrize("problem,N,opts,tag", [
    ("LukVlE2", 1000, {}, "LukVlE2_1000"),                                   # 10 inertia corrections (WRONG_INERTIA returns)
    ("LukVlE5", 1000, {}, "LukVlE5_1000"),                                   # 12 inertia corrections
    ("MBndryCntrl1", 20, {"start_with_resto": "yes"}, "MBndryCntrl1_20_yes"),       # restoration phase (AugRestoSystemSolver)
    ("LukVlI1", 200, {"start_with_resto": "yes"}, "LukVlI1_200_yes"),
    ("MDistCntrl3a", 20, {"hessian_approximation": "limited-memory"}, "MDistCntrl3a_20_limitedmemory"),   # L-BFGS: multi-rhs solves
    ("LukVlE1", 200, {"hessian_approximation": "limited-memory"}, "LukVlE1_200_limitedmemory"),
])
def test_ip_loop_parity_inertia_restoration_lbfgs(problem, N, opts, tag, tmp_path):
    """The callers around the path that the benchmark problems do not reach with default options: inertia correction
    (IpPDFullSpaceSolver.cpp:541-591), the restoration phase (IpAugRestoSystemSolver.cpp:260) and the low-rank L-BFGS
    wrapper with nrhs > 1 (IpLowRankAugSystemSolver.cpp:182,487).  Same counts and iterates as the oracle run."""
    summ, fin = _run_driver("b200", problem, N, tmp_path, opts)
    gold = np.load(os.path.join(G, tag + "_final.npz"))
    assert summ["status"] == 0
    assert summ["iterations"] == int(gold["iterations"])
    # same factorisations and inertia corrections; the number of back-solves may differ by a refinement step or two (the
    # reference's PDFullSpaceSolver adds a step when the residual ratio sits at its threshold, IpPDFullSpaceSolver.cpp:256-346)
    assert summ["n_factor"] == int(gold["n_factor"]) and summ["n_wrong_inertia"] == int(gold["n_wrong_inertia"])
    assert abs(summ["n_solve"] - int(gold["n_solve"])) <= 4 and abs(summ["n_rhs"] - int(gold["n_rhs"])) <= 12
    assert abs(fin["obj"] - float(gold["obj"])) <= 1e-10 * max(abs(float(gold["obj"])), 1e-12)
    for key in ("x", "lam", "z_L", "z_U"):
        ref = gold[key]
        scale = max(np.abs(ref).max(), 1e-300)
        assert np.abs(fin[key] - ref).max() <= RTOL * scale, key


@pytest.mark.parametrize("problem,N", [("hs071", 0), ("MBndryCntrl1", 30), ("MDistCntrl3a", 25), ("LukVlE1", 1000)])
def test_ma97_shim_through_stock_ipopt(problem, N, tmp_path):
    """SURVEY.md 8b' / 8f-3: the UNMODIFIED reference code path  linear_solver=ma97 + hsllib=libb200ldlt.so  -- Ipopt's own
    Ma97SolverInterface (IpMa97SolverInterface.cpp:303-314) dlopen()s the library and drives the GPU backend through the
    seven ma97_*_d entry points of ipopt_b200/csrc/hsl_shim.cpp; no custom hook, no plugin.  Same iterates as the oracle
    run behind the custom-solver hook."""
    summ, fin = _run_driver("ma97", problem, N, tmp_path)
    gold = np.load(os.path.join(G, "%s_%d_final.npz" % (problem, N)))
    assert summ["status"] == 0 and summ["backend"].startswith("ma97-shim")
    assert abs(summ["iterations"] - int(gold["iterations"])) <= 1
    assert abs(fin["obj"] - float(gold["obj"])) <= 1e-9 * max(abs(float(gold["obj"])), 1e-12)
    for key in ("x", "lam", "z_L", "z_U"):
        ref = gold[key]
        scale = max(np.abs(ref).max(), 1e-300)
        assert np.abs(fin[key] - ref).max() <= 1e-7 * scale, key   # (another adapter: other refinement / scaling defaults)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_factor_solve_matches_single_gpu(world):
    """Elimination-tree sharding (SURVEY.md 8e) with all ranks emulated on one GPU: same kernels, contribution blocks /
    update vectors / solution pieces exchanged between the rank handles -> must reproduce the unsharded result."""
    from ipopt_b200.sharded import ShardedLdlt
    dim, irn, jcn, val, nc = mbndry_kkt(60, sigma_spread=3.0, seed=9)
    _, _, _, v0, _ = mbndry_kkt(60, w_zero=True)
    b = np.random.default_rng(3).standard_normal(dim)
    s = gpu_solver(dim, irn, jcn)
    s.GetValuesArrayPtr()[:] = v0
    assert s.factor(True, nc)[0] == SYMSOLVER_SUCCESS       # analysis on the first (W = 0) matrix, like Ipopt
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, nc)
    assert st == SYMSOLVER_SUCCESS and neg == nc
    x1 = b.copy()
    s.solve(x1)
    sh = ShardedLdlt(dim, irn, jcn, v0, local_world=world)
    assert sh.n_subtrees >= 2 * world
    st, neg = sh.factor(val, True, nc)
    assert st == SYMSOLVER_SUCCESS and neg == nc
    x2 = sh.solve(b)
    assert np.linalg.norm(x2 - x1) <= 1e-12 * np.linalg.norm(x1)
    assert scaled_residual(dim, irn, jcn, val, x2, b) < 1e-13
    # a second matrix on the same shard plan
    val2 = val.copy(); val2[:dim // 2] *= 1.5
    st, neg = sh.factor(val2, True, nc)
    assert st == SYMSOLVER_SUCCESS and neg == nc
    assert scaled_residual(dim, irn, jcn, val2, sh.solve(b), b) < 1e-13
    sh.close(); s.close()


@pytest.mark.parametrize("problem,N", [("hs071", 0), ("MBndryCntrl1", 30)])
def test_warm_start_same_structure_keeps_the_analysis(problem, N, tmp_path):
    """Second solve of the same NLP with warm_start_same_structure=yes (ReOptimizeNLP): the adapter keeps its handle and
    symbolic analysis (reference contract: IpMumpsSolverInterface.cpp:227-236), and the second solve converges like the first."""
    summ, _ = _run_driver("b200", problem, N, tmp_path, extra=["--reopt"])
    assert summ["status"] == 0 and summ["reopt_status"] == 0
    assert summ["n_analyse"] == 1                                  # one InitializeStructure reached the backend, not two
    assert summ["reopt_iterations"] == summ["iterations"]
    assert summ["n_factor"] == 2 * summ["n_factor_first"]
