"""Iterative refinement by the componentwise backward error (b200ldlt_solve_refined_device): device time at MBndryCntrl1
N=400 and on the lifted tridiagonal (n = 2000, 1e-10 diagonal, num_forced > 0), against the plain solve of the same
handle.

  python tools/bench_refine.py [--N 400] [--reps 21] [--warmup 3] [--out DIR]

Device-resident b and x.  Each round times, alternating, one solve of nrhs columns and the refined solve of the same
columns (nrhs = 1, 4, 8; max_steps 10, tol 2^-52); the time of a call is the library's CUDA-event time
(info()["ms_solve_gpu"], which includes the host decision after each iterate and its synchronisation).  Also per round,
at nrhs = 1, the older normwise refinement (b200ldlt_solve_refine_device, min_steps 1, max_steps 10, tol 1e-10), and
the working-precision row pass (error analysis with cond = 0) at each width, to set against the double-double one.
Median / min / max over --reps rounds after warm-up, each column's steps and status, launches, omega_first and omega,
and the time relative to one solve of the same width.  Prints the card name, power limit and max SM clock and one JSON
document (also written to --out/bench_refine.json)."""
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

EPS = 2.0 ** -52


def gpu_props():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def stats(v):
    v = np.asarray(v)
    return dict(median_ms=float(np.median(v)), min_ms=float(v.min()), max_ms=float(v.max()))


def tridiag(n=2000):
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    return n, irn, jcn, val


def run(name, system, reps, warmup):
    import torch
    dim, irn, jcn, val = system
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    dv = torch.tensor(val, dtype=torch.float64, device="cuda")
    assert s.factor_device(dv.data_ptr())[0] == 0, s.last_error()
    B = torch.randn(8, dim, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    X = torch.empty_like(B)
    W = torch.empty_like(B)
    X0 = B.clone()
    assert s.solve_device(X0.data_ptr(), 8) == 0, s.last_error()
    t = {k: {"solve": [], "refined": [], "ea_cond0": []} for k in (1, 4, 8)}
    t_old, outc, launches, old = [], {}, {}, {}
    for r in range(warmup + reps):
        for k in (1, 4, 8):
            W[:k].copy_(B[:k])
            assert s.solve_device(W.data_ptr(), k) == 0
            ts = s.info()["ms_solve_gpu"]
            st, d = s.solve_refined_device(B.data_ptr(), X.data_ptr(), k, 10, EPS)
            assert st == 0, s.last_error()
            tr, launches[k] = s.info()["ms_solve_gpu"], s.info()["launches_solve"]
            outc[k] = {f: v.tolist() for f, v in d.items()}
            st, _ = s.error_analysis_device(B.data_ptr(), X0.data_ptr(), k, 0)
            assert st == 0, s.last_error()
            te = s.info()["ms_solve_gpu"]
            if r >= warmup:
                t[k]["solve"].append(ts)
                t[k]["refined"].append(tr)
                t[k]["ea_cond0"].append(te)
        W[0].copy_(B[0])
        st, steps, ratio = s.solve_refine_device(W[0].data_ptr(), 1, 10, 1e-10)
        assert st == 0, s.last_error()
        old = dict(steps=steps, residual_ratio=ratio, launches=s.info()["launches_solve"])
        if r >= warmup:
            t_old.append(s.info()["ms_solve_gpu"])
    x = torch.empty(dim, dtype=torch.float64, device="cuda")
    x.copy_(B[0])
    assert s.solve_device(x.data_ptr(), 1) == 0
    L0 = s.info()["launches_solve"]
    res = dict(system=name, dim=dim, num_forced=s.info()["num_forced"], L0=L0, widths={})
    for k in (1, 4, 8):
        sv, rf, ea = stats(t[k]["solve"]), stats(t[k]["refined"]), stats(t[k]["ea_cond0"])
        res["widths"]["nrhs%d" % k] = dict(solve=sv, refined=dict(rf, vs_solve=rf["median_ms"] / sv["median_ms"]),
                                           ea_cond0=ea, launches=launches[k], columns=outc[k])
    res["solve_refine_device_nrhs1"] = dict(stats(t_old), **old)
    s.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=400)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU path")
    props = gpu_props()
    print("card: %s, power limit %s, max SM clock %s" % (props["gpu"], props["power_limit"], props["max_sm_clock"]))
    res = dict(props, runs=[])
    for name, system in (("MBndryCntrl1 N=%d" % a.N, mbndry_kkt(a.N)[:4]), ("tridiag 2000 (lifted)", tridiag())):
        r = run(name, system, a.reps, a.warmup)
        res["runs"].append(r)
        print("%s: dim=%d num_forced=%d L0=%d" % (name, r["dim"], r["num_forced"], r["L0"]))
        for key, w in r["widths"].items():
            c = w["columns"]
            print("  %-6s solve %7.3f ms  refined %7.3f ms (%.3f-%.3f) = %5.2f x  ea(cond=0) %6.3f ms  launches %d"
                  % (key, w["solve"]["median_ms"], w["refined"]["median_ms"], w["refined"]["min_ms"],
                     w["refined"]["max_ms"], w["refined"]["vs_solve"], w["ea_cond0"]["median_ms"], w["launches"]))
            print("         steps %s status %s nres %s" % (c["steps"], c["status"], c["nres"]))
            print("         omega_first %s" % ["%.2e" % v for v in c["omega_first"]])
            print("         omega       %s" % ["%.2e" % (u + v) for u, v in zip(c["omega1"], c["omega2"])])
        o = r["solve_refine_device_nrhs1"]
        print("  solve_refine_device nrhs=1: %.3f ms (%.3f-%.3f), steps %d, ratio %.2e, launches %d" % (
            o["median_ms"], o["min_ms"], o["max_ms"], o["steps"], o["residual_ratio"], o["launches"]))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_refine.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
