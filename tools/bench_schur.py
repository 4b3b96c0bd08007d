"""Schur mode (b200ldlt_set_schur): the direct route to S_c = A_SS - A_SE A_EE^-1 A_ES against the route a caller has
without it, at MBndryCntrl1 N=400.

  python tools/bench_schur.py [--N 400] [--m 64 256 1024] [--reps 7] [--warmup 2] [--nrhs 8] [--out DIR]

Schur sets: m seeded variables, half drawn uniformly from the constraint rows and half from the primal variables (numpy
default_rng(m + t), t = 0..3), the first draw whose A_EE factorises without lifted pivots (pivots are not delayed into
S, so a constraint row of E that loses its best primal partners to S can need one); if none does, m constraint rows
(default_rng(m)), which leave every primal variable in E.  The JSON says which set was used.  Per m:
  * the Schur-mode factorisation (factor_device, device-resident values): the library's CUDA-event time;
  * schur_reduce_device and schur_expand_device on --nrhs columns: the library's event time over nrhs (per column);
  * today's route, timed with CUDA events around all of it: a full factorisation, m job-0 solves on the identity
    columns e_vars[j] (one blocked solve_device call), the gather of (A^-1)_SS and torch.linalg.inv of it on the GPU;
  * the max-norm difference of the two S_c, relative to max |S_c|.
Median / min / max over --reps rounds after warm-up.  Prints the card name and power limit (read in the same run) and one
JSON document (also written to --out/bench_schur.json)."""
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


def schur_sets(dim, nc, m):
    nx = dim - nc
    for t in range(4):
        rng = np.random.default_rng(m + t)
        yield "mixed, seed %d" % (m + t), np.concatenate([nx + rng.choice(nc, m // 2, replace=False),
                                                          rng.choice(nx, m - m // 2, replace=False)])
    yield "constraint rows, seed %d" % m, nx + np.random.default_rng(m).choice(nc, m, replace=False)


def run(N, m, reps, warmup, nrhs):
    import torch
    dim, irn, jcn, val, nc = mbndry_kkt(N)
    dv = torch.tensor(val, dtype=torch.float64, device="cuda")
    # direct route
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    for kind, vars in schur_sets(dim, nc, m):
        assert s.set_schur(vars) == 0, s.last_error()
        assert s.factor_device(dv.data_ptr())[0] == 0, s.last_error()
        if s.info()["num_forced"] == 0:
            break
    B = torch.randn(dim, nrhs, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    B = B.t().contiguous()    # column-major dim x nrhs
    Y = torch.zeros(nrhs, m, dtype=torch.float64, device="cuda")
    X = torch.zeros(nrhs, dim, dtype=torch.float64, device="cuda")
    sc = torch.zeros(m, m, dtype=torch.float64, device="cuda")
    tf, tr, te = [], [], []
    for r in range(warmup + reps):
        st = s.factor_device(dv.data_ptr())[0]
        assert st == 0, s.last_error()
        if r >= warmup: tf.append(s.info()["ms_factor_gpu"])
        assert s.schur_reduce_device(B.data_ptr(), Y.data_ptr(), nrhs) == 0, s.last_error()
        if r >= warmup: tr.append(s.info()["ms_solve_gpu"] / nrhs)
        assert s.schur_expand_device(B.data_ptr(), Y.data_ptr(), X.data_ptr(), nrhs) == 0, s.last_error()
        if r >= warmup: te.append(s.info()["ms_solve_gpu"] / nrhs)
    info = s.info()
    assert s.schur_complement_device(sc.data_ptr()) == 0
    sc_direct = sc.t().contiguous()     # (symmetric anyway)
    launches = dict(factor=info["launches_factor"])
    s.close()
    # today's route: full factorisation, m solves on identity columns, (A^-1)_SS inverted on the GPU
    o = B200Ldlt()
    assert o.InitializeStructure(dim, len(irn), irn, jcn) == 0
    vt = torch.tensor(vars, dtype=torch.long, device="cuda")
    E = torch.zeros(m, dim, dtype=torch.float64, device="cuda")     # column-major dim x m
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    to = []
    for r in range(warmup + reps):
        torch.cuda.synchronize()
        ev0.record()
        assert o.factor_device(dv.data_ptr())[0] == 0, o.last_error()
        E.zero_()
        E[torch.arange(m, device="cuda"), vt] = 1.0
        assert o.solve_device(E.data_ptr(), m) == 0, o.last_error()
        ainv_ss = E[:, vt]                   # row j = column j of A^-1, restricted to S: (A^-1)_SS (symmetric)
        sc_old = torch.linalg.inv(ainv_ss)
        ev1.record()
        torch.cuda.synchronize()
        if r >= warmup: to.append(ev0.elapsed_time(ev1))
    o.close()
    diff = float((sc_direct - sc_old).abs().max() / sc_direct.abs().max())
    return dict(N=N, dim=dim, m=m, schur_set=kind, num_forced=info["num_forced"], launches=launches, schur_factor=stats(tf),
                reduce_per_col=stats(tr), expand_per_col=stats(te), todays_route=stats(to), sc_rel_maxdiff=diff)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=400)
    ap.add_argument("--m", type=int, nargs="+", default=[64, 256, 1024])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--nrhs", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU path")
    props = gpu_props()
    print("card: %s, power limit %s, max SM clock %s" % (props["gpu"], props["power_limit"], props["max_sm_clock"]))
    res = dict(props, runs=[])
    for m in a.m:
        r = run(a.N, m, a.reps, a.warmup, a.nrhs)
        res["runs"].append(r)
        print("N=%d m=%d: Schur-mode factor %.3f ms, reduce %.3f ms/col, expand %.3f ms/col; today's route %.3f ms; "
              "S_c rel. max diff %.2e (%s, forced %d)"
              % (a.N, m, r["schur_factor"]["median_ms"], r["reduce_per_col"]["median_ms"], r["expand_per_col"]["median_ms"],
                 r["todays_route"]["median_ms"], r["sc_rel_maxdiff"], r["schur_set"], r["num_forced"]))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_schur.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
