"""Multiplication by the factors (b200ldlt_lmultiply_device) on MBndryCntrl1 N=400, against job 1 of the partial solves.

  python tools/bench_lmultiply.py [--N 400] [--reps 21] [--out DIR]

Device-resident.  Each round times trans 0 and trans 1 at nrhs 1 and 8 and job 1 (one column), alternating call by
call; the time of a call is the library's CUDA-event time (info()["ms_solve_gpu"], device part only).  Medians over --reps
rounds after warm-up.  The rate is over the algorithmic bytes: the strictly lower part of L read once per call,
8 (nnz_L - n), plus the vectors, 16 n per column (x read, y written), against the H100 SXM data-sheet HBM3 bandwidth of
3.35 TB/s.  Every round's results are checked bit for bit against the first round's.  Prints one JSON document (and
writes it to --out/bench_lmultiply.json when --out is given)."""
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

HBM_TBS = 3.35   # H100 SXM data sheet


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
    nnz_l = s.info()["nnz_L"]
    X = torch.tensor(np.random.default_rng(0).standard_normal((8, dim)), dtype=torch.float64, device="cuda")
    Y = torch.empty_like(X)
    cases = [("trans0_nrhs1", 0, 1), ("trans1_nrhs1", 1, 1), ("trans0_nrhs8", 0, 8), ("trans1_nrhs8", 1, 8)]
    t = {k: [] for k, _, _ in cases}
    t["job1"] = []
    launches, first = {}, {}
    identical = True
    for r in range(a.warmup + a.reps):
        for name, trans, nrhs in cases:
            assert s.lmultiply_device(trans, X.data_ptr(), Y.data_ptr(), nrhs) == 0, s.last_error()
            i = s.info()
            launches[name] = i["launches_solve"]
            out = Y[:nrhs].clone()
            if name not in first:
                first[name] = out
            identical &= bool(torch.equal(out.view(torch.int64), first[name].view(torch.int64)))
            if r >= a.warmup:
                t[name].append(i["ms_solve_gpu"])
        Y[0].copy_(X[0])
        assert s.solve_partial_device(1, Y.data_ptr(), 1) == 0, s.last_error()
        if r >= a.warmup:
            t["job1"].append(s.info()["ms_solve_gpu"])
    med = {k: float(np.median(v)) for k, v in t.items()}
    gbs, peak = {}, {}
    for name, trans, nrhs in cases:
        byts = 8.0 * (nnz_l - dim) + 16.0 * dim * nrhs
        gbs[name] = byts / (med[name] * 1e-3) / 1e9
        peak[name] = gbs[name] / (HBM_TBS * 1e3)
    res = dict(gpu_props(), N=a.N, dim=dim, nnz_L=nnz_l, reps=a.reps, ms_median=med,
               ms_min={k: float(np.min(v)) for k, v in t.items()}, ms_max={k: float(np.max(v)) for k, v in t.items()},
               algorithmic_GBps=gbs, share_of_datasheet_hbm=peak, launches=launches, bit_reproducible=identical)
    s.close()
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_lmultiply.json"), "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
