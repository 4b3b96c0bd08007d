"""Sparse forward solve (b200ldlt_sparse_fwd_solve_device) against job 1 on the dense right-hand side, MBndryCntrl1 N=400.

  python tools/bench_sparse_fwd_solve.py [--N 400] [--reps 21] [--out DIR]

Device-resident, one column.  Patterns: one variable in a leaf front, one variable in the root front, 10 random
variables, 1 % random variables, all n variables.  Each round times, for every pattern, the sparse call and job 1 on the
dense b of the same pattern, alternating call by call; the time of a call is the library's CUDA-event time
(info()["ms_solve_gpu"], device part only).  Each round also checks that the sparse values equal job 1's at xindex (as
values) and that job 1 is zero elsewhere.  Per pattern: median / min / max over --reps rounds after warm-up, |reach| and
|R| (fronts; R = the fronts the pruned sweep runs, symbolic_array "sparse_run_set"), nxi, the share of nnz(L) in the
reach and in R (from L_off), launches of both calls, and the median host wall time of the host entry point.  Prints one
JSON document (and writes it to --out/bench_sparse_fwd_solve.json when --out is given)."""
import argparse
import json
import os
import subprocess
import sys
import time

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
    sn_start, sn_parent, L_off = s.symbolic("sn_start"), s.symbolic("sn_parent"), s.symbolic("L_off")
    nsn = len(sn_start) - 1
    nnzL = float(L_off[-1])
    var = s.enquire_indef()[0]
    pos = np.empty(dim, np.int64)
    pos[var] = np.arange(dim)
    has_child = np.zeros(nsn, bool)
    has_child[sn_parent[sn_parent >= 0]] = True
    leaf = int(np.flatnonzero(~has_child)[0])
    root = int(np.flatnonzero(sn_parent < 0)[-1])

    def reach(bi):
        fr = set()
        for v in bi:
            f = int(np.searchsorted(sn_start, pos[v], side="right") - 1)
            while f >= 0 and f not in fr:
                fr.add(f)
                f = int(sn_parent[f])
        return sorted(fr)

    rng = np.random.default_rng(0)
    pats = {
        "leaf_1": np.array([var[sn_start[leaf]]]),
        "root_1": np.array([var[sn_start[root]]]),
        "random_10": rng.choice(dim, 10, replace=False),
        "random_1pct": rng.choice(dim, dim // 100, replace=False),
        "all_n": np.arange(dim),
    }
    pats = {k: (v.astype(np.int32), rng.standard_normal(len(v))) for k, v in pats.items()}
    dev = {}
    for k, (bi, bv) in pats.items():
        dense = np.zeros(dim)
        dense[bi] = bv
        dev[k] = (torch.tensor(bv, device="cuda"), torch.tensor(dense, device="cuda"))
    dx = torch.empty(dim, dtype=torch.float64, device="cuda")
    dy = torch.empty(dim, dtype=torch.float64, device="cuda")

    t = {k: {"sparse": [], "job1": [], "host_wall": []} for k in pats}
    meta = {}
    values_equal = {k: True for k in pats}
    for r in range(a.warmup + a.reps):
        for k, (bi, bv) in pats.items():
            db, dd = dev[k]
            xi = s.sparse_fwd_solve_device(bi, db.data_ptr(), dx.data_ptr())
            i = s.info()
            ms_sp, l_sp = i["ms_solve_gpu"], i["launches_solve"]
            dy.copy_(dd)
            assert s.solve_partial_device(1, dy.data_ptr(), 1) == 0, s.last_error()
            i = s.info()
            ms_j1, l_j1 = i["ms_solve_gpu"], i["launches_solve"]
            w0 = time.perf_counter()
            s.sparse_fwd_solve(bi, bv)
            wall = (time.perf_counter() - w0) * 1e3
            y = dy.cpu().numpy()
            x = dx[:len(xi)].cpu().numpy()
            mask = np.ones(dim, bool)
            mask[xi] = False
            values_equal[k] &= bool(np.array_equal(x, y[xi]) and np.all(y[mask] == 0.0))
            if r >= a.warmup:
                t[k]["sparse"].append(ms_sp)
                t[k]["job1"].append(ms_j1)
                t[k]["host_wall"].append(wall)
            if k not in meta:
                rf, run = reach(bi), s.symbolic("sparse_run_set")
                share = lambda fr: float(sum(L_off[f + 1] - L_off[f] for f in fr)) / nnzL   # noqa: E731
                meta[k] = dict(nbi=len(bi), reach_fronts=len(rf), run_fronts=len(run), nxi=len(xi),
                               nnzL_share_reach=share(rf), nnzL_share_run=share(run),
                               launches_sparse=l_sp, launches_job1=l_j1)
    res = dict(gpu_props(), N=a.N, dim=dim, nsn=nsn, reps=a.reps, patterns={})
    for k in pats:
        d = dict(meta[k])
        for kind in ("sparse", "job1"):
            v = t[k][kind]
            d["ms_%s" % kind] = dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))
        d["host_wall_ms_median"] = float(np.median(t[k]["host_wall"]))
        d["values_equal_job1_every_round"] = values_equal[k]
        res["patterns"][k] = d
    s.close()
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_sparse_fwd_solve.json"), "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
