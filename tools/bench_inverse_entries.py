"""Entries of A^-1 (b200ldlt_inverse_entries_device) against the routes a caller has without it, MBndryCntrl1 N=400.

  python tools/bench_inverse_entries.py [--N 400] [--reps 21] [--warmup 5] [--out DIR]

Device-resident.  Patterns: one diagonal entry in a leaf front, one in the root front, the variances of 10 random
variables, the lower triangle of a 32 x 32 block of random variables (the reduced-Hessian shape), 1000 random diagonal
entries.  Each round times, for every pattern and alternating call by call: the call; today's route (blocked job-0
solves of the unit columns, then the gather of the entries); for the diagonal patterns selected_inverse (diagonal
only); and the call on a second handle created with B200_SOLVE_BLOCK=1 (one column per pruned sweep).  The time of a
library call is its CUDA-event time (info()["ms_solve_gpu"], device part only); the gather of today's route is timed
with CUDA events on the torch stream and added to its solve.  Per pattern: median / min / max over --reps rounds after
warm-up, launches, the distinct columns, |run set| (union over the blocks, symbolic_array "inverse_run_set") and its
share of nnz(L), the bytes of the y store (12 per element), and the largest deviation from today's route relative to
the max-norm of its entries.  Prints one JSON document (and writes it to --out/bench_inverse_entries.json)."""
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


def handle(dim, irn, jcn, val, block=None):
    old = os.environ.pop("B200_SOLVE_BLOCK", None)
    if block is not None:
        os.environ["B200_SOLVE_BLOCK"] = block
    try:
        s = B200Ldlt()
    finally:
        os.environ.pop("B200_SOLVE_BLOCK", None)
        if old is not None:
            os.environ["B200_SOLVE_BLOCK"] = old
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    s.GetValuesArrayPtr()[:] = val
    assert s.factor(False, 0)[0] == 0, s.last_error()
    return s


def stats(v):
    return dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))


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
    dim, irn, jcn, val, _ = mbndry_kkt(a.N)
    s = handle(dim, irn, jcn, val)
    s1 = handle(dim, irn, jcn, val, block="1")
    sn_start, sn_parent, L_off = s.symbolic("sn_start"), s.symbolic("sn_parent"), s.symbolic("L_off")
    nsn = len(sn_start) - 1
    nnzL = float(L_off[-1])
    var = s.enquire_indef()[0]
    has_child = np.zeros(nsn, bool)
    has_child[sn_parent[sn_parent >= 0]] = True
    leaf = int(np.flatnonzero(~has_child)[0])
    root = int(np.flatnonzero(sn_parent < 0)[-1])
    k = np.diff(sn_start)
    pathlen = np.zeros(nsn, np.int64)
    for f in range(nsn - 1, -1, -1):
        pathlen[f] = k[f] + (pathlen[sn_parent[f]] if sn_parent[f] >= 0 else 0)
    pos = np.empty(dim, np.int64)
    pos[var] = np.arange(dim)
    front = lambda v: int(np.searchsorted(sn_start, pos[v], side="right") - 1)   # noqa: E731

    rng = np.random.default_rng(0)
    b32 = rng.choice(dim, 32, replace=False)
    ti, tj = np.tril_indices(32)
    d10, d1000 = rng.choice(dim, 10, replace=False), rng.choice(dim, 1000, replace=False)
    pats = {
        "leaf_diag_1": ([var[sn_start[leaf]]],) * 2,
        "root_diag_1": ([var[sn_start[root]]],) * 2,
        "variances_10": (d10, d10),
        "block32_lower": (b32[ti], b32[tj]),
        "diag_1000": (d1000, d1000),
    }
    pats = {p: (np.asarray(i, np.int32), np.asarray(j, np.int32)) for p, (i, j) in pats.items()}
    cols = {p: np.unique(np.concatenate(v)) for p, v in pats.items()}
    dev = {}
    for p, (i, j) in pats.items():
        c = cols[p]
        where = {int(v): q for q, v in enumerate(c)}
        ci = torch.tensor([where[int(v)] for v in i], device="cuda")
        dev[p] = dict(vals=torch.empty(len(i), dtype=torch.float64, device="cuda"),
                      X=torch.empty(len(c) * dim, dtype=torch.float64, device="cuda"),
                      unit=torch.tensor(np.arange(len(c)) * dim + c, device="cuda"),
                      gather=(ci * dim + torch.tensor(j.astype(np.int64), device="cuda")))
    ddiag = torch.empty(dim, dtype=torch.float64, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kinds = ("call", "job0_route", "selected_inverse", "call_block1")
    t = {p: {kd: [] for kd in kinds} for p in pats}
    meta = {}
    dev_max = {p: 0.0 for p in pats}
    for r in range(a.warmup + a.reps):
        for p, (i, j) in pats.items():
            D = dev[p]
            assert s.inverse_entries_device(i, j, D["vals"].data_ptr()) == 0, s.last_error()
            inf = s.info()
            ms_call, l_call = inf["ms_solve_gpu"], inf["launches_solve"]
            # today's route: unit columns, blocked job 0, gather
            D["X"].zero_()
            D["X"][D["unit"]] = 1.0
            torch.cuda.synchronize()
            assert s.solve_device(D["X"].data_ptr(), len(cols[p])) == 0, s.last_error()
            inf = s.info()
            ms_j0, l_j0 = inf["ms_solve_gpu"], inf["launches_solve"]
            e0.record()
            ref = D["X"][D["gather"]]
            e1.record()
            torch.cuda.synchronize()
            ms_j0 += e0.elapsed_time(e1)
            ms_si = None
            if np.array_equal(i, j):
                assert s.selected_inverse_device(ddiag.data_ptr(), 0) == 0, s.last_error()
                ms_si = s.info()["ms_solve_gpu"]
            v1 = torch.empty_like(D["vals"])
            assert s1.inverse_entries_device(i, j, v1.data_ptr()) == 0, s1.last_error()
            ms_b1, l_b1 = s1.info()["ms_solve_gpu"], s1.info()["launches_solve"]
            v, rv, b1 = D["vals"].cpu().numpy(), ref.cpu().numpy(), v1.cpu().numpy()
            assert np.array_equal(v, b1), (p, "B200_SOLVE_BLOCK=1 gives other values")
            dev_max[p] = max(dev_max[p], float(np.abs(v - rv).max() / max(np.abs(rv).max(), 1e-300)))
            if r >= a.warmup:
                t[p]["call"].append(ms_call)
                t[p]["job0_route"].append(ms_j0)
                t[p]["call_block1"].append(ms_b1)
                if ms_si is not None:
                    t[p]["selected_inverse"].append(ms_si)
            if p not in meta:
                run = s.symbolic("inverse_run_set")
                ny = int(sum(pathlen[front(v)] for v in cols[p]))
                meta[p] = dict(entries=len(i), columns=len(cols[p]), run_fronts=len(run),
                               nnzL_share_run=float(sum(L_off[f + 1] - L_off[f] for f in run)) / nnzL,
                               y_store_bytes=12 * ny, launches_call=l_call, launches_call_block1=l_b1,
                               launches_job0_route=l_j0)
    res = dict(gpu_props(), N=a.N, dim=dim, nsn=nsn, reps=a.reps, patterns={})
    for p in pats:
        d = dict(meta[p])
        for kd in kinds:
            if t[p][kd]:
                d["ms_" + kd] = stats(t[p][kd])
        d["max_rel_dev_from_job0_route"] = dev_max[p]
        res["patterns"][p] = d
    s.close()
    s1.close()
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_inverse_entries.json"), "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
