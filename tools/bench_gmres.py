"""FGMRES preconditioned by the factors (b200ldlt_solve_gmres_device) at MBndryCntrl1 N=400, device-resident: against the
plain solve, the classical refinement of the same handle, and, for A + delta I over the primal block, against a
factorisation of those values plus a solve.

  python tools/bench_gmres.py [--N 400] [--reps 21] [--warmup 3] [--out DIR]

Each round times, alternating, one column through: job 0 (b200ldlt_solve_device); b200ldlt_solve_refined_device
(max_steps 10, tol 2^-52); b200ldlt_solve_gmres_device with vals = NULL; and for each delta, b200ldlt_solve_gmres_device
on A + delta I over the primal block (the factors stay those of A) and then b200ldlt_factor_device on those values plus
a solve (info ms_factor_gpu + ms_solve_gpu), after which the factors of A are restored (not timed).  The time of a call
is the library's CUDA-event time (info()["ms_solve_gpu"], which includes each host decision and its synchronisation).
FGMRES runs with restart 20, max_cycles 10, tol 2^-52 and each --inner-tol.  Median (min-max) over --reps rounds after
--warmup rounds, each call's cycles, iterations, status and omega.  One more FGMRES call per configuration runs under
torch.profiler: the device idle time inside the call, divided by its synchronisations (nres + iters), is the
per-synchronisation cost.  Prints the card name, power limit and max SM clock and one JSON document (also written to
--out/bench_gmres.json; the profiler traces go to --out too)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ipopt_b200 import B200Ldlt  # noqa: E402
from ipopt_b200.kkt import mbndry_kkt  # noqa: E402

EPS = 2.0 ** -52
DELTAS = (1e-9, 1e-7, 1e-5)


def gpu_props():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [v.strip() for v in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def stats(v):
    v = np.asarray(v)
    return dict(median_ms=float(np.median(v)), min_ms=float(v.min()), max_ms=float(v.max()))


def idle_per_sync(call, nsync, trace):
    """device idle time inside one call (the span of its kernels and copies minus their union), per synchronisation"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    with open(trace) as fh:
        ev = json.load(fh)["traceEvents"]
    iv = sorted((e["ts"], e["ts"] + e.get("dur", 0)) for e in ev
                if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset"))
    busy, end = 0.0, None
    for a, b in iv:
        if end is None or a > end:
            busy += b - a
            end = b
        elif b > end:
            busy += b - end
            end = b
    span = iv[-1][1] - iv[0][0]
    return dict(span_us=span, busy_us=busy, idle_us=span - busy, syncs=nsync,
                idle_per_sync_us=(span - busy) / max(nsync, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=400)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--inner-tol", type=float, nargs="+", default=[1e-6, 1e-10, 1e-14])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU path")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    props = gpu_props()
    print("card: %s, power limit %s, max SM clock %s" % (props["gpu"], props["power_limit"], props["max_sm_clock"]))
    dim, irn, jcn, val, nc = mbndry_kkt(a.N)
    nx = dim - nc
    diag = np.flatnonzero((irn == jcn) & (irn <= nx))
    _, first = np.unique(irn[diag], return_index=True)
    primal_diag = diag[first]
    assert len(primal_diag) == nx
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    dv = torch.tensor(val, dtype=torch.float64, device="cuda")
    shifted = {}
    for d in DELTAS:
        v = val.copy()
        v[primal_diag] += d
        shifted[d] = torch.tensor(v, dtype=torch.float64, device="cuda")
    assert s.factor_device(dv.data_ptr())[0] == 0, s.last_error()
    b = torch.randn(dim, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    x = torch.empty_like(b)
    confs = [("gmres_A", None)] + [("gmres_A+%gI" % d, d) for d in DELTAS]
    t = {"solve": [], "refined": [], **{"%s tol%g" % (k, it): [] for k, _ in confs for it in a.inner_tol},
         **{"refactor_solve_A+%gI" % d: [] for d in DELTAS}}
    out, launches = {}, {}

    def gm(d, it):
        vp = None if d is None else shifted[d].data_ptr()
        st, o = s.solve_gmres_device(b.data_ptr(), x.data_ptr(), 1, vp, restart=20, max_cycles=10, tol=EPS,
                                     inner_tol=it)
        assert st == 0, s.last_error()
        return {k: v.tolist()[0] for k, v in o.items()}

    for r in range(a.warmup + a.reps):
        keep = r >= a.warmup
        x.copy_(b)
        assert s.solve_device(x.data_ptr(), 1) == 0
        ms = {"solve": s.info()["ms_solve_gpu"]}
        launches["solve"] = s.info()["launches_solve"]
        st, o = s.solve_refined_device(b.data_ptr(), x.data_ptr(), 1, 10, EPS)
        assert st == 0, s.last_error()
        ms["refined"] = s.info()["ms_solve_gpu"]
        out["refined"] = {k: v.tolist()[0] for k, v in o.items()}
        for k, d in confs:
            for it in a.inner_tol:
                key = "%s tol%g" % (k, it)
                out[key] = gm(d, it)
                ms[key] = s.info()["ms_solve_gpu"]
                launches[key] = s.info()["launches_solve"]
            if d is not None:
                assert s.factor_device(shifted[d].data_ptr())[0] == 0, s.last_error()
                tf = s.info()["ms_factor_gpu"]
                x.copy_(b)
                assert s.solve_device(x.data_ptr(), 1) == 0
                ms["refactor_solve_A+%gI" % d] = tf + s.info()["ms_solve_gpu"]
                assert s.factor_device(dv.data_ptr())[0] == 0, s.last_error()
        if keep:
            for k, v in ms.items():
                t[k].append(v)
    res = dict(props, system="MBndryCntrl1 N=%d" % a.N, dim=dim, nnz=len(irn), num_forced=s.info()["num_forced"],
               calls={})
    for k, v in t.items():
        res["calls"][k] = dict(stats(v), launches=launches.get(k), outcome=out.get(k))
    res["sync"] = {}
    for k, d in confs:
        for it in a.inner_tol:
            key = "%s tol%g" % (k, it)
            o = out[key]
            name = "gmres_trace_%s.json" % key.replace(" ", "_").replace("+", "p")
            trace = os.path.join(a.out or tempfile.gettempdir(), name)
            res["sync"][key] = idle_per_sync(lambda: gm(d, it), o["nres"] + o["iters"], trace)
    print("%s: dim=%d num_forced=%d" % (res["system"], dim, res["num_forced"]))
    for k, c in res["calls"].items():
        o = c["outcome"] or {}
        om = o.get("omega1", 0.0) + o.get("omega2", 0.0) if o else float("nan")
        print("  %-26s %8.3f ms (%.3f-%.3f)  launches %s  %s" % (
            k, c["median_ms"], c["min_ms"], c["max_ms"], c["launches"],
            "" if not o else "cycles/steps %s iters %s status %s omega_first %.2e omega %.2e" % (
                o.get("cycles", o.get("steps")), o.get("iters", "-"), o["status"], o["omega_first"], om)))
    for k, v in res["sync"].items():
        print("  sync %-22s span %.0f us, device idle %.0f us over %d syncs = %.1f us each" % (
            k, v["span_us"], v["idle_us"], v["syncs"], v["idle_per_sync_us"]))
    print(json.dumps(res))
    if a.out:
        with open(os.path.join(a.out, "bench_gmres.json"), "w") as fh:
            json.dump(res, fh, indent=1)
    s.close()


if __name__ == "__main__":
    main()
