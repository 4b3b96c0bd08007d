"""Error analysis and condition estimation (b200ldlt_error_analysis_device, b200ldlt_condest): device time at MBndryCntrl1
N=400, against the plain solve of the same handle.

  python tools/bench_error_analysis.py [--N 400] [--reps 21] [--warmup 3] [--out DIR]

Device-resident b and x.  Each round times, alternating, one solve of nrhs columns and each call (condest; error analysis
with cond = 0 and 1 at nrhs = 1, 4, 8); the time of a call is the library's CUDA-event time (info()["ms_solve_gpu"],
which includes the host decisions of the estimator steps and their synchronisations).  Median / min / max over --reps
rounds after warm-up, the products each call took and the time relative to one single-column solve.  Prints the card
name, power limit and max SM clock and one JSON document (also written to --out/bench_error_analysis.json)."""
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


def gpu_props():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def stats(v):
    v = np.asarray(v)
    return dict(median_ms=float(np.median(v)), min_ms=float(v.min()), max_ms=float(v.max()))


def run(N, reps, warmup):
    import torch
    dim, irn, jcn, val, nc = mbndry_kkt(N)
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    dv = torch.tensor(val, dtype=torch.float64, device="cuda")
    assert s.factor_device(dv.data_ptr())[0] == 0, s.last_error()
    B = torch.randn(8, dim, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    X = B.clone()
    assert s.solve_device(X.data_ptr(), 8) == 0, s.last_error()
    W = torch.empty_like(B)
    calls = [("condest", 0, None)] + [("ea_cond%d" % c, k, c) for k in (1, 4, 8) for c in (0, 1)]
    t = {}
    ts = {k: [] for k in (1, 4, 8)}
    nprod = {}
    for r in range(warmup + reps):
        for name, k, cond in calls:
            key = name if cond is None else "%s_nrhs%d" % (name, k)
            t.setdefault(key, [])
            w = max(k, 1)
            W[:w].copy_(B[:w])
            assert s.solve_device(W.data_ptr(), w) == 0
            if r >= warmup:
                ts[w].append(s.info()["ms_solve_gpu"])
            if cond is None:
                nprod[key] = s.condest()[3]
            else:
                st, d = s.error_analysis_device(B.data_ptr(), X.data_ptr(), k, cond)
                assert st == 0, s.last_error()
                nprod[key] = [int(p) for p in d["nprod"]]
            if r >= warmup:
                t[key].append(s.info()["ms_solve_gpu"])
    one = float(np.median(ts[1]))
    res = dict(N=N, dim=dim, solve={"nrhs%d" % k: stats(v) for k, v in ts.items()}, calls={})
    for key, v in t.items():
        if not v:
            continue
        st = stats(v)
        res["calls"][key] = dict(st, nprod=nprod[key], vs_one_solve=st["median_ms"] / one)
    s.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, nargs="+", default=[400])
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
    for N in a.N:
        r = run(N, a.reps, a.warmup)
        res["runs"].append(r)
        print("N=%d dim=%d: solve nrhs=1 %.3f ms, nrhs=4 %.3f ms, nrhs=8 %.3f ms" % (
            N, r["dim"], r["solve"]["nrhs1"]["median_ms"], r["solve"]["nrhs4"]["median_ms"], r["solve"]["nrhs8"]["median_ms"]))
        for key, c in r["calls"].items():
            print("  %-16s %8.3f ms (%.3f-%.3f)  %5.2f x one solve  nprod %s" % (
                key, c["median_ms"], c["min_ms"], c["max_ms"], c["vs_one_solve"], c["nprod"]))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_error_analysis.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
