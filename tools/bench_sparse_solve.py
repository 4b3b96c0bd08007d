"""Sparse solve (b200ldlt_sparse_solve_device) against job 0 on the dense right-hand side, MBndryCntrl1 N=400.

  python tools/bench_sparse_solve.py [--N 400] [--reps 21] [--warmup 5] [--out DIR]

Device-resident, one column.  Patterns of b and selections of x, every pair of: one variable in a leaf front, one
variable in the root front, 10 random variables, 1 % random variables, and dense b / every entry (bindex / xsel NULL).
Each round times, for every pair, the sparse call and job 0 (b200ldlt_solve_device) on the dense b, alternating call by
call; the time of a call is the library's CUDA-event time (info()["ms_solve_gpu"]).  Each round also checks that the
sparse values equal job 0's at the selection.  Per pair: median / min / max over --reps rounds after warm-up, |R_f| and
|R_b| (fronts, symbolic_array "sparse_solve_fwd_run_set" / "sparse_solve_bwd_run_set"), their shares of nnz(L) (from
L_off) and the launches of both calls.  Prints one JSON document (and writes it to --out/bench_sparse_solve.json when
--out is given)."""
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
    sn_start, sn_parent, L_off = s.symbolic("sn_start"), s.symbolic("sn_parent"), s.symbolic("L_off")
    nsn = len(sn_start) - 1
    nnzL = float(L_off[-1])
    var = s.enquire_indef()[0]
    has_child = np.zeros(nsn, bool)
    has_child[sn_parent[sn_parent >= 0]] = True
    leaves = np.flatnonzero(~has_child)
    root = int(np.flatnonzero(sn_parent < 0)[-1])
    rng = np.random.default_rng(0)
    kinds = {
        "leaf_1": lambda q: np.array([var[sn_start[leaves[q]]]]),
        "root_1": lambda q: np.array([var[sn_start[root] + q]]),
        "random_10": lambda q: rng.choice(dim, 10, replace=False),
        "random_1pct": lambda q: rng.choice(dim, dim // 100, replace=False),
        "dense": lambda q: None,
    }
    # b patterns take the first leaf / root pivot, selections the second: a leaf-to-leaf pair crosses two leaf paths
    bpats = {k: f(0) for k, f in kinds.items()}
    sels = {k: f(1) for k, f in kinds.items()}
    bpats = {k: None if v is None else v.astype(np.int32) for k, v in bpats.items()}
    sels = {k: None if v is None else v.astype(np.int32) for k, v in sels.items()}
    bvals = {k: rng.standard_normal(dim if v is None else len(v)) for k, v in bpats.items()}
    dev = {}
    for k, bi in bpats.items():
        dense = bvals[k].copy() if bi is None else np.zeros(dim)
        if bi is not None:
            dense[bi] = bvals[k]
        dev[k] = (torch.tensor(bvals[k], device="cuda"), torch.tensor(dense, device="cuda"))
    dx = torch.empty(dim, dtype=torch.float64, device="cuda")
    dy = torch.empty(dim, dtype=torch.float64, device="cuda")
    pairs = [(kb, kx) for kb in bpats for kx in sels]
    t = {p: {"sparse": [], "job0": []} for p in pairs}
    meta = {}
    values_equal = {p: True for p in pairs}
    share = lambda fr: float(sum(L_off[f + 1] - L_off[f] for f in fr)) / nnzL   # noqa: E731
    for r in range(a.warmup + a.reps):
        for kb, kx in pairs:
            bi, xs = bpats[kb], sels[kx]
            db, dd = dev[kb]
            assert s.sparse_solve_device(bi, db.data_ptr(), xs, dx.data_ptr()) == 0, s.last_error()
            i = s.info()
            ms_sp, l_sp = i["ms_solve_gpu"], i["launches_solve"]
            dy.copy_(dd)
            assert s.solve_device(dy.data_ptr(), 1) == 0, s.last_error()
            i = s.info()
            ms_j0, l_j0 = i["ms_solve_gpu"], i["launches_solve"]
            y = dy.cpu().numpy()
            nxs = dim if xs is None else len(xs)
            x = dx[:nxs].cpu().numpy()
            values_equal[(kb, kx)] &= bool(np.array_equal(x, y if xs is None else y[xs]))
            if r >= a.warmup:
                t[(kb, kx)]["sparse"].append(ms_sp)
                t[(kb, kx)]["job0"].append(ms_j0)
            if (kb, kx) not in meta:
                s.sparse_solve_device(bi, db.data_ptr(), xs, dx.data_ptr())
                rf, rb = s.symbolic("sparse_solve_fwd_run_set"), s.symbolic("sparse_solve_bwd_run_set")
                meta[(kb, kx)] = dict(b=kb, x=kx, nbi=dim if bi is None else len(bi), nxs=nxs, fwd_run_fronts=len(rf),
                                      bwd_run_fronts=len(rb), nnzL_share_fwd=share(rf), nnzL_share_bwd=share(rb),
                                      launches_sparse=l_sp, launches_job0=l_j0)
    res = dict(gpu_props(), N=a.N, dim=dim, nsn=nsn, reps=a.reps, pairs=[])
    for p in pairs:
        d = dict(meta[p])
        for kind in ("sparse", "job0"):
            v = t[p][kind]
            d["ms_%s" % kind] = dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))
        d["values_equal_job0_every_round"] = values_equal[p]
        res["pairs"].append(d)
    s.close()
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_sparse_solve.json"), "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
