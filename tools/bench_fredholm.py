"""Fredholm alternative (b200ldlt_solve_fredholm_device) against job 0 on the same columns, MBndryCntrl1 N=400 with three
variables' rows and columns zeroed (values only, same pattern), keep mode.

  python tools/bench_fredholm.py [--N 400] [--reps 21] [--out DIR]

Device-resident.  Each round times, for nrhs 1, 4 and 8, solve_fredholm and job 0 (b200ldlt_solve_device) on the same
columns, alternating call by call, and the factor call on the singular values and on the original values (two handles,
device-resident values); the time of a call is the library's CUDA-event time (info()["ms_solve_gpu"] /
["ms_factor_gpu"], device part only).  Per case: median / min / max over --reps rounds after warm-up, and the launches.
Prints the card name and power limit and one JSON document (also written to --out/bench_fredholm.json)."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=400)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU path")
    props = gpu_props()
    print("card: %s, power limit %s, max SM clock %s" % (props["gpu"], props["power_limit"], props["max_sm_clock"]))
    dim, irn, jcn, val, nc = mbndry_kkt(a.N)
    rows = np.sort(np.random.default_rng(0).choice(dim, 3, replace=False))
    vz = val.copy()
    vz[np.isin(irn - 1, rows) | np.isin(jcn - 1, rows)] = 0.0
    hs = {}
    for tag, v in (("singular", vz), ("original", val)):
        s = B200Ldlt()
        assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
        s.set_singular_action(1)
        hs[tag] = (s, torch.tensor(v, dtype=torch.float64, device="cuda"))
    s = hs["singular"][0]
    assert s.factor_device(hs["singular"][1].data_ptr())[0] == 1, s.last_error()
    assert len(s.enquire_zero_pivots()) == 3
    rng = np.random.default_rng(1)
    B = torch.tensor(rng.standard_normal((8, dim)), dtype=torch.float64, device="cuda")
    X = torch.zeros(16 * dim, dtype=torch.float64, device="cuda")
    Y = torch.zeros(8 * dim, dtype=torch.float64, device="cuda")
    NR = (1, 4, 8)
    t = {("fred", k): [] for k in NR}
    t.update({("job0", k): [] for k in NR})
    tf = {"singular": [], "original": []}
    launches = {}
    for r in range(a.warmup + a.reps):
        for k in NR:
            X[:k * dim] = B[:k].reshape(-1)
            st, _ = s.solve_fredholm_device(X.data_ptr(), k, 1e-10)
            assert st == 0, s.last_error()
            i = s.info()
            if r >= a.warmup: t[("fred", k)].append(i["ms_solve_gpu"])
            launches[("fred", k)] = i["launches_solve"]
            Y[:k * dim] = B[:k].reshape(-1)
            assert s.solve_device(Y.data_ptr(), k) == 0, s.last_error()
            i = s.info()
            if r >= a.warmup: t[("job0", k)].append(i["ms_solve_gpu"])
            launches[("job0", k)] = i["launches_solve"]
        for tag in ("singular", "original"):
            h, dv = hs[tag]
            h.factor_device(dv.data_ptr())
            if r >= a.warmup: tf[tag].append(h.info()["ms_factor_gpu"])
    out = dict(props, N=a.N, dim=dim, reps=a.reps, zeroed_rows=rows.tolist(), solve={}, factor={})
    print("%-10s %-6s %28s %28s %9s" % ("call", "nrhs", "fredholm ms med (min-max)", "job 0 ms med (min-max)", "launches"))
    for k in NR:
        f, j = stats(t[("fred", k)]), stats(t[("job0", k)])
        out["solve"][k] = dict(fredholm=f, job0=j, launches_fredholm=launches[("fred", k)], launches_job0=launches[("job0", k)])
        print("%-10s %-6d %12.3f (%.3f-%.3f) %14.3f (%.3f-%.3f) %5d/%d" % (
            "solve", k, f["median_ms"], f["min_ms"], f["max_ms"], j["median_ms"], j["min_ms"], j["max_ms"],
            launches[("fred", k)], launches[("job0", k)]))
    for tag in ("singular", "original"):
        out["factor"][tag] = stats(tf[tag])
        print("factor %-9s %12.3f (%.3f-%.3f)" % (tag, out["factor"][tag]["median_ms"], out["factor"][tag]["min_ms"],
                                                out["factor"][tag]["max_ms"]))
    print(json.dumps(out))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_fredholm.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
