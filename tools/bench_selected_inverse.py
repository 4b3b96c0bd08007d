"""Selected inversion (b200ldlt_selected_inverse_device): device time at MBndryCntrl1 N=400 and N=800, achieved FP64 rate,
and (--profile) a torch.profiler breakdown by kernel in a separate run.

  python tools/bench_selected_inverse.py [--N 400 800] [--reps 11] [--warmup 3] [--profile] [--out DIR]

Device-resident outputs.  Each round times the call and a factorisation of the same handle (device-resident values),
alternating; the time of a call is the library's CUDA-event time (info()["ms_solve_gpu"] / ["ms_factor_gpu"]).  Median /
min / max over --reps rounds after warm-up.  The flop count (flops() below) is computed from the symbolic arrays.
Prints the card name and power limit and one JSON document (also written to --out/bench_selected_inverse.json)."""
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


def flops(s):
    """useful FP64 flops of the recurrence (2 per multiply-add, structural zeros of the triangles skipped):
    L11^-1 (fronts of order <= 256): k^3/3; B = L21 L11^-1: r k^2; Z_RJ = -G B: 2 r^2 k; Z_JJ lower: k^3/3 + r k^2"""
    ss, rp = s.symbolic("sn_start"), s.symbolic("rows_ptr")
    k, r = np.diff(ss).astype(float), np.diff(rp).astype(float)
    f = k + r
    linv = np.where(f <= 256, k ** 3 / 3, 0.0)
    return float(np.sum(linv + r * k * k + 2 * r * r * k + k ** 3 / 3 + r * k * k))


def run(N, reps, warmup):
    import torch
    dim, irn, jcn, val, nc = mbndry_kkt(N)
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    dv = torch.tensor(val, dtype=torch.float64, device="cuda")
    assert s.factor_device(dv.data_ptr())[0] == 0, s.last_error()
    d = torch.zeros(dim, dtype=torch.float64, device="cuda")
    v = torch.zeros(len(irn), dtype=torch.float64, device="cuda")
    ts, tf = [], []
    for r in range(warmup + reps):
        assert s.selected_inverse_device(d.data_ptr(), v.data_ptr()) == 0, s.last_error()
        i = s.info()
        if r >= warmup: ts.append(i["ms_solve_gpu"])
        launches = i["launches_solve"]
        assert s.factor_device(dv.data_ptr())[0] == 0
        if r >= warmup: tf.append(s.info()["ms_factor_gpu"])
    fl = flops(s)
    st = stats(ts)
    info = s.info()
    out = dict(N=N, dim=dim, nnz_L=info["nnz_L"], launches=launches, selinv=st, factor=stats(tf), flops=fl,
               gflops_per_s=fl / (st["median_ms"] * 1e-3) / 1e9)
    s.close()
    return out


def profile(N, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    dim, irn, jcn, val, nc = mbndry_kkt(N)
    s = B200Ldlt()
    assert s.InitializeStructure(dim, len(irn), irn, jcn) == 0
    dv = torch.tensor(val, dtype=torch.float64, device="cuda")
    assert s.factor_device(dv.data_ptr())[0] == 0
    d = torch.zeros(dim, dtype=torch.float64, device="cuda")
    v = torch.zeros(len(irn), dtype=torch.float64, device="cuda")
    s.selected_inverse_device(d.data_ptr(), v.data_ptr())
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(5):
            s.selected_inverse_device(d.data_ptr(), v.data_ptr())
        torch.cuda.synchronize()
    rows = {}
    for e in p.key_averages():
        if "k_si_" in e.key:
            rows[e.key] = dict(calls=e.count // 5, ms_per_call=e.device_time_total / 5 / 1e3)
    for k_, r in sorted(rows.items(), key=lambda kv: -kv[1]["ms_per_call"]):
        print("  %-40s %5d launches %9.3f ms" % (k_[:40], r["calls"], r["ms_per_call"]))
    if out_dir:
        p.export_chrome_trace(os.path.join(out_dir, "selinv_trace_N%d.json" % N))
    s.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, nargs="+", default=[400, 800])
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU path")
    props = gpu_props()
    print("card: %s, power limit %s, max SM clock %s" % (props["gpu"], props["power_limit"], props["max_sm_clock"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    res = dict(props, runs=[])
    for N in a.N:
        if a.profile:
            print("N=%d kernel breakdown (torch.profiler, per call):" % N)
            res["runs"].append(dict(N=N, profile=profile(N, a.out)))
            continue
        r = run(N, a.reps, a.warmup)
        res["runs"].append(r)
        print("N=%d dim=%d: selected inverse %.3f ms (%.3f-%.3f), %d launches, %.1f GFLOP/s (%.3g flop); factor %.3f ms"
              % (N, r["dim"], r["selinv"]["median_ms"], r["selinv"]["min_ms"], r["selinv"]["max_ms"], r["launches"],
                 r["gflops_per_s"], r["flops"], r["factor"]["median_ms"]))
    print(json.dumps(res))
    if a.out:
        with open(os.path.join(a.out, "bench_selected_inverse%s.json" % ("_profile" if a.profile else "")), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
