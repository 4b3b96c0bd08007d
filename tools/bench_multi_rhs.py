"""Blocked multi-right-hand-side solve against the per-column loop (B200_SOLVE_BLOCK=1) on MBndryCntrl1 N=400.

  python tools/bench_multi_rhs.py [--N 400] [--reps 21] [--out DIR]

Part 1: device-resident solves (b200ldlt_solve_device) for nrhs in {1, 2, 4, 6, 8, 12, 16}, timed by the library's CUDA
events (info()["ms_solve_gpu"]) after warm-up, median over --reps, the two handles alternating call by call.  The outputs
of the two handles are compared bit for bit.
Part 2: GPU time by kernel of one single-column and one 8-column solve (torch.profiler, its own run).
Part 3: host-memory solves (b200ldlt_solve) for nrhs 1..6, wall time per call, the two handles alternating.
Part 4: the reference IP loop (tests/driver/ipopt_driver) in L-BFGS mode on MBndryCntrl1 N, the two settings alternating,
three runs each.
Prints one JSON document (and writes it to --out/bench_multi_rhs.json when --out is given)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ipopt_b200 import B200Ldlt  # noqa: E402
from ipopt_b200.kkt import mbndry_kkt  # noqa: E402

NRHS = (1, 2, 4, 6, 8, 12, 16)


def gpu_props():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def handle(block, dim, irn, jcn, val, nc, **opts):
    if block is None:
        os.environ.pop("B200_SOLVE_BLOCK", None)
    else:
        os.environ["B200_SOLVE_BLOCK"] = str(block)
    s = B200Ldlt(**opts)    # B200_* switches are read here
    os.environ.pop("B200_SOLVE_BLOCK", None)
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    s.GetValuesArrayPtr()[:] = val
    st, neg = s.factor(True, nc)
    assert st == 0 and neg == nc, s.info()
    return s


def solve_times(N, reps):
    import torch
    dim, irn, jcn, val, nc = mbndry_kkt(N, sigma_spread=2.0, seed=1)
    h = {"loop": handle(1, dim, irn, jcn, val, nc), "blocked": handle(None, dim, irn, jcn, val, nc)}
    rng = np.random.default_rng(0)
    rows = []
    for nrhs in NRHS:
        B = torch.tensor(rng.standard_normal(dim * nrhs), dtype=torch.float64, device="cuda")
        bufs = {k: B.clone() for k in h}
        ms = {k: [] for k in h}
        launches = {}
        for it in range(3 + reps):
            for k in (("loop", "blocked") if it % 2 == 0 else ("blocked", "loop")):
                bufs[k].copy_(B)
                torch.cuda.synchronize()
                assert h[k].solve_device(bufs[k].data_ptr(), nrhs) == 0
                inf = h[k].info()
                launches[k] = inf["launches_solve"]
                if it >= 3:
                    ms[k].append(inf["ms_solve_gpu"])
        same = bool(torch.equal(bufs["loop"].view(torch.int64), bufs["blocked"].view(torch.int64)))
        row = dict(nrhs=nrhs, bit_identical=same)
        for k in h:
            med = float(np.median(ms[k]))
            row[k] = dict(ms_median=med, ms_min=float(np.min(ms[k])), ms_max=float(np.max(ms[k])),
                          ms_per_column=med / nrhs, launches=launches[k])
        row["speedup"] = row["loop"]["ms_median"] / row["blocked"]["ms_median"]
        rows.append(row)
        print("nrhs %2d  loop %7.3f ms (%6.3f/col)  blocked %7.3f ms (%6.3f/col)  x%.2f  launches %d / %d  identical %s" % (
            nrhs, row["loop"]["ms_median"], row["loop"]["ms_per_column"], row["blocked"]["ms_median"],
            row["blocked"]["ms_per_column"], row["speedup"], launches["loop"], launches["blocked"], same), flush=True)
    for s in h.values():
        s.close()
    return dict(system="mbndry_kkt(%d, sigma_spread=2, seed=1)" % N, dim=dim, nnz=len(irn), reps=reps, rows=rows)


def host_calls(N, reps):
    """Host-memory solves (b200ldlt_solve, the path Ipopt's MultiSolve takes) for nrhs 1..6, wall time per call around
    the synchronous call, median over reps, the two handles alternating."""
    import time
    dim, irn, jcn, val, nc = mbndry_kkt(N, sigma_spread=2.0, seed=1)
    h = {"loop": handle(1, dim, irn, jcn, val, nc), "blocked": handle(None, dim, irn, jcn, val, nc)}
    rng = np.random.default_rng(2)
    rows = []
    for nrhs in range(1, 7):
        B = rng.standard_normal(dim * nrhs)
        t = {k: [] for k in h}
        for it in range(2 + reps):
            for k in (("loop", "blocked") if it % 2 == 0 else ("blocked", "loop")):
                X = B.copy()
                t0 = time.perf_counter()
                assert h[k].solve(X, nrhs) == 0
                if it >= 2:
                    t[k].append(1e3 * (time.perf_counter() - t0))
        row = dict(nrhs=nrhs, **{k + "_ms": float(np.median(v)) for k, v in t.items()})
        rows.append(row)
        print("host solve nrhs %d: loop %.3f ms, blocked %.3f ms (wall, median of %d)" % (nrhs, row["loop_ms"], row["blocked_ms"], reps), flush=True)
    for s in h.values():
        s.close()
    return rows


def kernel_phases(N, nrhs=8):
    """GPU time by kernel (torch.profiler, CUDA activities) of one single-column solve and one blocked nrhs-column solve."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    dim, irn, jcn, val, nc = mbndry_kkt(N, sigma_spread=2.0, seed=1)
    s = handle(None, dim, irn, jcn, val, nc, verbose=1)   # (stderr: the size of the per-column state of the blocked solve)
    B = torch.tensor(np.random.default_rng(1).standard_normal(dim * nrhs), dtype=torch.float64, device="cuda")
    res = {}
    for k in (1, nrhs):
        for _ in range(3):
            assert s.solve_device(B.data_ptr(), k) == 0
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            assert s.solve_device(B.data_ptr(), k) == 0
            torch.cuda.synchronize()
        tot = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("b200::", "")
                name += "<fwd>" if "<true>" in e.name else ("<bwd>" if "<false>" in e.name else "")
                tot[name] = tot.get(name, 0.0) + e.device_time / 1e3
        res["nrhs_%d" % k] = {n: round(v, 4) for n, v in sorted(tot.items(), key=lambda kv: -kv[1])}
        print("kernel ms, nrhs=%d:" % k, res["nrhs_%d" % k], flush=True)
    s.close()
    return res


def ip_loop(N, out):
    drv = os.path.join(ROOT, "tests", "driver", "ipopt_driver")
    if not os.path.exists(drv):
        return "not measured: tests/driver/ipopt_driver not built"
    res = {}
    for tag, block in [(t + "_%d" % r, b) for r in range(1, 4) for t, b in (("loop", "1"), ("blocked", None))]:
        js = os.path.join(out, "lbfgs_%s.json" % tag)
        env = dict(os.environ, OMP_NUM_THREADS=str(min(16, os.cpu_count() or 1)))
        env.pop("B200_SOLVE_BLOCK", None)
        if block:
            env["B200_SOLVE_BLOCK"] = block
        p = subprocess.run([drv, "--backend", "b200", "--problem", "MBndryCntrl1", "--N", str(N), "--print-level", "0",
                            "--json", js, "--opt", "hessian_approximation=limited-memory"],
                           capture_output=True, text=True, env=env, timeout=1800)
        if p.returncode != 0:
            res[tag] = "failed: " + (p.stdout + p.stderr)[-500:]
            continue
        r = json.load(open(js))
        res[tag] = {k: r[k] for k in ("status", "iterations", "n_factor", "n_solve", "n_rhs", "t_factor_s", "t_solve_s", "t_total_s")}
        print("L-BFGS IP loop %-9s" % tag, res[tag], flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=400)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-ip-loop", action="store_true")
    a = ap.parse_args()
    out = a.out or os.path.join(os.environ.get("TMPDIR", "/tmp"), "bench_multi_rhs")
    os.makedirs(out, exist_ok=True)
    doc = dict(gpu_props())
    print(doc, flush=True)
    doc["solve_device"] = solve_times(a.N, a.reps)
    doc["host_solve"] = host_calls(a.N, a.reps)
    doc["kernel_ms"] = kernel_phases(a.N)
    doc["ip_loop_lbfgs"] = "not measured" if a.no_ip_loop else ip_loop(a.N, out)
    if a.out:
        with open(os.path.join(a.out, "bench_multi_rhs.json"), "w") as f:
            json.dump(doc, f, indent=1)
    print(json.dumps(doc))


if __name__ == "__main__":
    main()
