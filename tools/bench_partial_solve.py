"""Partial solves (b200ldlt_solve_partial_device, jobs 1-4) against the full solve (job 0) on MBndryCntrl1 N=400.

  python tools/bench_partial_solve.py [--N 400] [--reps 21] [--out DIR]

Device-resident, one column.  Each round times job 0, job 1, job 2, job 3, job 4 and the chain 1 -> 2 -> 3, alternating
call by call; the time of a call is the library's CUDA-event time (info()["ms_solve_gpu"], device part only), and for the
chain the sum of its three calls.  Medians over --reps rounds after warm-up.  The chain's result is checked bit for bit
against job 0.  Prints one JSON document (and writes it to --out/bench_partial_solve.json when --out is given)."""
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
    dim, irn, jcn, val, nc = mbndry_kkt(a.N)
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == 0, s.last_error()
    b = torch.tensor(np.random.default_rng(0).standard_normal(dim), dtype=torch.float64, device="cuda")
    x = torch.empty_like(b)

    def call(job):
        assert s.solve_partial_device(job, x.data_ptr(), 1) == 0, s.last_error()
        i = s.info()
        return i["ms_solve_gpu"], i["launches_solve"]

    names = ["job0", "job1", "job2", "job3", "job4", "job1+2+3"]
    t = {k: [] for k in names}
    launches = {}
    identical = True
    for r in range(a.warmup + a.reps):
        row = {}
        for job in range(5):
            x.copy_(b)
            row["job%d" % job], launches["job%d" % job] = call(job)
            if job == 0:
                x0 = x.clone()
        x.copy_(b)
        chain = sum(call(job)[0] for job in (1, 2, 3))
        identical &= bool(torch.equal(x.view(torch.int64), x0.view(torch.int64)))
        row["job1+2+3"] = chain
        if r >= a.warmup:
            for k in names:
                t[k].append(row[k])
    res = dict(gpu_props(), N=a.N, dim=dim, reps=a.reps,
               ms_median={k: float(np.median(v)) for k, v in t.items()},
               ms_min={k: float(np.min(v)) for k, v in t.items()},
               ms_max={k: float(np.max(v)) for k, v in t.items()},
               launches=launches, chain_bit_identical_to_job0=identical)
    s.close()
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_partial_solve.json"), "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
