#!/usr/bin/env python
"""bench.py -- KKT LDL^T factor+solve throughput of the GPU backend on an H100.

A "step" = the linear algebra of ONE interior-point iteration: one numeric factorisation of a new KKT matrix (inertia
check on) + two back-solves (step + one refinement), the call pattern measured on the reference's IP loop (SURVEY.md 8c:
1 factorisation + 2 back-solves per iteration).  Workload: --gpus 1 -> MBndryCntrl1 N=400 (KKT dim 321 600, 1 283 200
triplets: the configuration BASELINE.json's target is quoted on); --gpus > 1 -> BASELINE config 5, MBndryCntrl1 N=800
(dim 1 283 200), ONE system factorised + solved by all GPUs together (elimination-tree sharding, "strong" scaling), with
the single-GPU time of the same N=800 step measured in the same run and printed in the same line.

  value : steps/s with the KKT values and right-hand sides already resident in HBM (b200ldlt_factor_device /
          b200ldlt_solve_device), CUDA events on the launching stream, max over ranks.
  e2e   : the same through the reference-facing C-ABI calls with HOST buffers (b200ldlt_factor reads the pinned
          values array Ipopt fills, b200ldlt_solve takes/returns host rhs) -- H2D/D2H inside the timed region.
  roofline : the HBM-bound triangular solve (bottom-level kernels + the two persistent sweeps): algorithmic bytes 2*8*nnz(L) +
          vector traffic (SURVEY.md 8d) / their measured duration, against MEASURED_PEAKS.json's hbm_gbs when present,
          else the H100 SXM data-sheet HBM3 bandwidth (3350 GB/s).
  cpu_baseline : the CPU oracle (oracle/cpu_ldlt.cpp, "port") on the host cores on the same matrix.  The reference's own
          comparator, MUMPS, is probed for at run time (ldconfig / pkg-config) and is absent from this image.
  ip_loop : the reference's unmodified interior-point loop (tests/driver/ipopt_driver) on the same problem with the
          GPU backend and with the CPU oracle: iterations, wall seconds, IP iterations per second.
--impl reference times the CPU path alone, same steps / warm-up as the product arm.
--dump-outputs DIR writes, after the timed steps, what the timed path returned to its caller in its last step: the
          solution vector (solution.npy, float64) and the inertia / status of the factorisation (factor.npy, float64:
          [status, number of negative eigenvalues]).  The inputs are the same from run to run with the same arguments.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOAD_N = 400
SHARDED_N = 800
SNAP_ITERS = [2, 8, 15]


def probe_mumps():
    """BASELINE.md section 3 step 1: is the reference's CPU comparator (MUMPS) installed on this box?"""
    found = []
    try:
        out = subprocess.run(["ldconfig", "-p"], capture_output=True, text=True, timeout=10).stdout
        found += [l.split()[0] for l in out.splitlines() if "mumps" in l.lower()]
    except Exception:
        pass
    try:
        if subprocess.run(["pkg-config", "--exists", "coinmumps"], timeout=10).returncode == 0:
            found.append("pkg-config:coinmumps")
    except Exception:
        pass
    return {"found": found, "note": "MUMPS present: rebuild oracle/_ref --with-mumps for a MUMPS column" if found else
            "no MUMPS library on this box (ldconfig -p | grep -i mumps; pkg-config --exists coinmumps): the CPU column is the oracle port"}


def run_ip_loop(backend, N, threads):
    """The reference's own IP loop on MBndryCntrl1(N) with the given linear-solver backend (tests/driver/ipopt_driver)."""
    drv = os.path.join(ROOT, "tests", "driver", "ipopt_driver")
    if not os.path.exists(drv):
        return None
    env = dict(os.environ, OMP_NUM_THREADS=str(threads))
    try:
        out = subprocess.run([drv, "--backend", backend, "--problem", "MBndryCntrl1", "--N", str(N), "--print-level", "0"],
                             env=env, timeout=900, capture_output=True, text=True).stdout
        d = json.loads([l for l in out.splitlines() if l.startswith("DRIVER_JSON ")][-1][len("DRIVER_JSON "):])
    except Exception as e:      # noqa: BLE001
        return {"error": str(e)[:200]}
    it = d["iterations"]
    return {"iterations": it, "status": d["status"], "total_s": d["t_total_s"], "iters_per_sec": it / d["t_total_s"],
            "analysis_first_factor_s": d["t_first_factor_s"], "factor_ms_per_call": 1e3 * d["t_factor_s"] / max(d["n_factor"] - 1, 1),
            "solve_ms_per_call": 1e3 * d["t_solve_s"] / max(d["n_solve"], 1), "n_factor": d["n_factor"], "n_solve": d["n_solve"],
            "objective": d["objective"]}


def get_snapshots(rank, N=None, backend="oracle"):
    """Real KKT systems of the reference's MBndryCntrl1(N) run, captured at the solver boundary by running the
    reference IP loop (driver binary) with the CPU oracle for a few iterations; synthetic same-pattern fallback."""
    import struct
    N = N or WORKLOAD_N
    drv = os.path.join(ROOT, "tests", "driver", "ipopt_driver")
    cache = os.path.join(tempfile.gettempdir(), "b200_bench_snap_%d" % N)
    paths = [cache + "_%d.bin" % k for k in SNAP_ITERS]
    src = "reference IP loop (MBndryCntrl1 N=%d) KKT snapshots at factorisations %s" % (N, SNAP_ITERS)
    if rank == 0 and not all(os.path.exists(p) for p in paths) and os.path.exists(drv):
        env = dict(os.environ, OMP_NUM_THREADS=str(min(32, os.cpu_count() or 1)))
        try:
            subprocess.run([drv, "--backend", backend, "--problem", "MBndryCntrl1", "--N", str(N),
                            "--print-level", "0", "--dump", cache, "--dump-iters", ",".join(map(str, SNAP_ITERS)),
                            "--opt", "max_iter=%d" % (max(SNAP_ITERS) + 1)], env=env, timeout=600,
                           stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        except Exception:
            pass
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist
        dist.barrier()
    snaps = []
    if all(os.path.exists(p) for p in paths):
        for p in paths:
            with open(p, "rb") as f:
                dim, nnz, nrhs, neg = struct.unpack("iiii", f.read(16))
                irn = np.frombuffer(f.read(4 * nnz), dtype=np.int32).copy()
                jcn = np.frombuffer(f.read(4 * nnz), dtype=np.int32).copy()
                val = np.frombuffer(f.read(8 * nnz), dtype=np.float64).copy()
                rhs = np.frombuffer(f.read(8 * dim * nrhs), dtype=np.float64).copy()[:dim]
            snaps.append(dict(dim=dim, irn=irn, jcn=jcn, val=val, rhs=rhs, neg=neg))
    else:
        from ipopt_b200.kkt import mbndry_kkt
        src = "synthetic MBndryCntrl1-pattern KKT (driver binary unavailable)"
        for k, spread in zip(SNAP_ITERS, (1.0, 4.0, 8.0)):
            dim, irn, jcn, val, nc = mbndry_kkt(N, sigma_spread=spread, seed=k)
            snaps.append(dict(dim=dim, irn=irn, jcn=jcn, val=val, rhs=np.random.default_rng(k).standard_normal(dim), neg=nc))
    return snaps, src


class ClockSampler(threading.Thread):
    def __init__(self, gpu_index):
        super().__init__(daemon=True)
        self.gpu, self.rows, self.stop_flag = gpu_index, [], False

    def run(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        while not self.stop_flag:
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.gpu), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.split(",")])
            except Exception:
                pass
            time.sleep(0.2)

    def summary(self):
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        sm = sorted(int(r[0]) for r in self.rows if r[0].isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(r[2 + i].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": int(self.rows[0][1]) if self.rows[0][1].isdigit() else None,
                "reasons": reasons, "samples": len(self.rows)}


def time_oracle(snaps, steps, warmup, threads):
    from oracle_api import OracleLdlt, oracle_lib
    oracle_lib().oracle_ldlt_set_threads(int(threads))
    s0 = snaps[0]
    o = OracleLdlt()
    o.InitializeStructure(s0["dim"], len(s0["irn"]), s0["irn"], s0["jcn"])
    t_steps = []
    last = None
    for it in range(warmup + steps):
        sn = snaps[it % len(snaps)]
        t0 = time.perf_counter()
        o.GetValuesArrayPtr()[:] = sn["val"]
        st, neg = o.factor(True, sn["neg"])
        assert st == 0, "oracle status %d" % st
        for _ in range(2):
            x = sn["rhs"].copy()
            o.solve(x)
        dt = time.perf_counter() - t0
        if it >= warmup:
            t_steps.append(dt)
        last = (x, st, neg)
    return float(np.mean(t_steps)), o.stats(), last


def dump_outputs(out_dir, x, status, neg):
    """What the timed path handed its caller in the last timed step (float64, a few MB at the benchmark sizes)."""
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "solution.npy"), np.ascontiguousarray(x, dtype=np.float64))
    np.save(os.path.join(out_dir, "factor.npy"), np.array([status, neg], dtype=np.float64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's outputs (solution, inertia) as DIR/<name>.npy")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    K, W = args.steps, max(args.warmup, 0)
    host_cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    cpu_threads = min(host_cores, 32)

    wl_N = WORKLOAD_N if world == 1 else SHARDED_N
    wl_dim = wl_N * wl_N * 2 + 4 * wl_N
    config = {"workload": "MBndryCntrl1 N=%d KKT (dim %d): 1 numeric LDL^T + 2 back-solves per step" % (wl_N, wl_dim),
              "parallelism": ("elimination-tree sharding over %d GPUs" % world) if world > 1 else "single GPU",
              "l2_policy": "working set (L + contribution blocks: hundreds of MB) exceeds the 50 MB L2; 3 different matrices cycled",
              "scaling_note": "one KKT system per step on all GPUs (strong scaling); --gpus 1 runs BASELINE config 3 (N=400, the metric's configuration), --gpus > 1 config 5 (N=800, the one north_star shards) with its single-GPU time in the same line"}

    if args.impl == "reference":
        # CPU path of the same workload (the reference's MUMPS is a third-party library absent from /root/reference and
        # from this image -- see probe_mumps(): this is the oracle port on all host threads), rank 0 only.
        if rank != 0:
            return 0
        snaps, src = get_snapshots_nodist(wl_N)
        sec, st, (x_last, st_last, neg_last) = time_oracle(snaps, K, W, cpu_threads)
        if args.dump_outputs:
            dump_outputs(args.dump_outputs, x_last, st_last, neg_last)
        line = {"impl": "reference", "metric": "kkt_factor_solve_iters_per_sec", "value": 1.0 / sec, "unit": "iter/s",
                "n_gpus": args.gpus, "steps": K, "warmup": W, "ms_per_step": sec * 1e3, "higher_is_better": True,
                "scaling": "strong", "vs_baseline": None, "dtype": "f64", "data": src, "config": config,
                "cpu_baseline": {"value": 1.0 / sec, "unit": "iter/s", "cores": cpu_threads, "kind": "port",
                                 "sample": "%d steps (1 factorisation + 2 solves each) of the same KKT snapshots; CPU oracle, NOT MUMPS" % K},
                "mumps_probe": probe_mumps(),
                "e2e": {"value": 1.0 / sec, "unit": "iter/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line))
        return 0

    import torch
    import torch.distributed as dist
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    torch.cuda.set_device(local_rank)
    from ipopt_b200 import B200Ldlt

    if world > 1:
        # config 5 (N=800): the snapshots come from the reference IP loop driven by the GPU backend itself on rank 0
        # (the CPU oracle needs minutes per run at this size)
        snaps, src = get_snapshots(rank, SHARDED_N, backend="b200")
        return run_sharded(args, snaps, src, config, rank, local_rank, world, K, W, host_cores)
    snaps, src = get_snapshots(rank)
    s0 = snaps[0]
    dim, nnz = s0["dim"], len(s0["irn"])
    stream = torch.cuda.Stream(local_rank)     # a real stream (handle 0 would make the library create its own)
    torch.cuda.set_stream(stream)              # torch copies / events below run on the stream the kernels are launched on
    solver = B200Ldlt(device=local_rank, stream=stream.cuda_stream)
    assert solver.InitializeStructure(dim, nnz, s0["irn"], s0["jcn"]) == 0
    # one-off symbolic phase on the first matrix (not part of a step)
    solver.GetValuesArrayPtr()[:] = s0["val"]
    t0 = time.perf_counter()
    st, neg = solver.factor(True, s0["neg"])
    t_analyse = time.perf_counter() - t0
    assert st == 0 and neg == s0["neg"], (st, neg, solver.last_error())
    info = solver.info()

    d_vals = [torch.from_numpy(sn["val"]).cuda() for sn in snaps]
    d_rhs0 = [torch.from_numpy(sn["rhs"]).cuda() for sn in snaps]
    d_work = torch.empty(dim, dtype=torch.float64, device="cuda")
    h_rhs = [sn["rhs"].copy() for sn in snaps]
    launches = 0
    last_factor = [None, None]

    def step_device(i):
        nonlocal launches
        sn = snaps[i % len(snaps)]
        st, neg = solver.factor_device(d_vals[i % len(snaps)].data_ptr(), True, sn["neg"])
        assert st == 0, (st, solver.last_error())
        last_factor[:] = [st, neg]
        launches += solver.info()["launches_factor"]
        for _ in range(2):
            d_work.copy_(d_rhs0[i % len(snaps)])
            assert solver.solve_device(d_work.data_ptr(), 1) == 0
            launches += solver.info()["launches_solve"] + 1

    def step_host(i):
        sn = snaps[i % len(snaps)]
        solver.GetValuesArrayPtr()[:] = sn["val"]           # what TSymLinearSolver::GiveMatrixToSolver does (host fill)
        x = None
        for r in range(2):
            x = h_rhs[i % len(snaps)].copy()
            st = solver.MultiSolve(r == 0, sn["irn"], sn["jcn"], 1, x, True, sn["neg"])
            assert st == 0, (st, solver.last_error())
        return x

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn):
        for i in range(W):
            fn(i)
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        for i in range(K):
            fn(W + i)
        e1.record(stream)
        barrier()
        wall = time.perf_counter() - t0
        ms = e0.elapsed_time(e1)
        t = torch.tensor([ms, wall * 1e3], dtype=torch.float64, device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0]), float(t[1])

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    launches = 0
    ms_dev, _ = timed(step_device)
    launches_timed = launches * K // (K + W)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, d_work.cpu().numpy(), *last_factor)
    ms_e2e, wall_e2e = timed(step_host)
    ms_e2e = max(ms_e2e, wall_e2e)   # host fill + memcpy of the step are part of the end-to-end time

    # roofline leg: the HBM-bound triangular solve sweep, timed alone on the launching stream
    solver.factor_device(d_vals[1].data_ptr(), True, snaps[1]["neg"])
    for _ in range(3):
        d_work.copy_(d_rhs0[1]); solver.solve_device(d_work.data_ptr(), 1)
    torch.cuda.synchronize()
    reps = 10
    tri_ms = 0.0
    for _ in range(reps):
        d_work.copy_(d_rhs0[1])
        solver.solve_device(d_work.data_ptr(), 1)
        tri_ms += solver.info()["ms_solve_gpu"]
    tri_ms /= reps
    solver.factor_device(d_vals[1].data_ptr(), True, snaps[1]["neg"])
    fac_ms = solver.info()["ms_factor_gpu"]
    sampler.stop_flag = True

    # parity of what was timed: residual of the last end-to-end solve
    x = step_host(1)
    r, xi, bi = solver.residual(x, snaps[1]["rhs"])
    info = solver.info()

    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
        nnzL = info["nnz_L"]
        tri_bytes = 2 * 8 * nnzL + 8 * 4 * dim   # L streamed twice + 2 reads/2 writes of the vector (SURVEY.md 8d)
        ach = tri_bytes / (tri_ms * 1e-3) / 1e9
        # CPU baseline, bounded sample on the host cores of this box
        # the oracle's rank-1 updates are memory-bound: more threads are not always faster -> report the best of a few
        skip_cpu = bool(os.environ.get("B200_BENCH_SKIP_CPU"))   # GPU-only runs (the CPU legs take minutes)
        cands = sorted({t for t in (8, 16, cpu_threads) if t <= cpu_threads})
        trials = [(time_oracle(snaps, 1, 0, t)[0], t) for t in cands[:-1]] if len(cands) > 1 and not skip_cpu else []
        best_t = min(trials)[1] if trials else cpu_threads
        sec_last = float("inf") if skip_cpu else time_oracle(snaps, 3, 1, cpu_threads)[0]
        sec_cpu = sec_last
        if trials and min(trials)[0] < sec_last:
            sec_cpu = time_oracle(snaps, 3, 1, best_t)[0]
            cpu_threads = best_t
        step_ms = ms_dev / K
        # the metric's other half: IP iterations per second of the reference's own loop, both backends
        ip_loop = None
        if not skip_cpu:
            ip_loop = {"problem": "MBndryCntrl1 N=%d, default Ipopt options (reference examples/ScalableProblems)" % WORKLOAD_N,
                       "b200": run_ip_loop("b200", WORKLOAD_N, 1), "cpu_oracle": run_ip_loop("oracle", WORKLOAD_N, cpu_threads)}
        line = {
            "metric": "kkt_factor_solve_iters_per_sec", "value": world * K / (ms_dev * 1e-3), "unit": "iter/s",
            "n_gpus": world, "steps": K, "warmup": W, "ms_per_step": step_ms, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "f64", "data": src, "config": config,
            "e2e": {"value": world * K / (ms_e2e * 1e-3), "unit": "iter/s", "ms_per_step": ms_e2e / K,
                    "h2d_bytes_per_step": 8 * nnz + 2 * 8 * dim, "d2h_bytes_per_step": 2 * 8 * dim + 32},
            "gpu_launches": launches_timed,
            "kkt_factor_solve_ms_per_iter": {"device_resident": step_ms, "e2e_host_buffers": ms_e2e / K,
                                             "factor_ms": fac_ms, "solve_ms_per_rhs": tri_ms},
            "roofline": {"kernel": "supernodal triangular solve, all launches of one right-hand side (k_rhs_in, k_solve_direct x2 levels, k_solve<fwd>, k_solve<bwd>, k_solve_direct x2, k_sol_out)",
                         "bound": "hbm", "achieved": ach, "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak,
                         "peak_source": "MEASURED_PEAKS.json hbm_gbs (burst)" if peaks else "H100 SXM data sheet (3.35 TB/s HBM3)",
                         "algorithmic_bytes_per_solve": tri_bytes},
            "factor": {"flops_panel": info["flops_panel"], "flops_schur": info["flops_schur"],
                       "gflops_achieved": (info["flops_panel"] + info["flops_schur"]) / (fac_ms * 1e-3) / 1e9,
                       "nnz_L": nnzL, "supernodes": info["nsupernodes"], "levels": info["nlevels"], "max_front": info["max_front"]},
            "cpu_baseline": None if skip_cpu else
                            {"value": 1.0 / sec_cpu, "unit": "iter/s", "ms_per_step": sec_cpu * 1e3, "cores": cpu_threads, "kind": "port",
                             "sample": "3 steps (1 factorisation + 2 solves each) of the same KKT snapshots; CPU oracle, not MUMPS"},
            "mumps_probe": probe_mumps(),
            "ip_loop": ip_loop,
            "analysis_once_s": {"wall_first_factor": t_analyse, "ordering": info["t_order_s"], "symbolic": info["t_symbolic_s"]},
            "parity": {"scaled_residual": r / (xi + bi), "num_neg": info["num_neg"], "expected_neg": snaps[1]["neg"]},
            "clocks": sampler.summary(), "host_cores": host_cores,
        }
        print(json.dumps(line))
    solver.close()
    if world > 1:
        dist.destroy_process_group()
    return 0


def run_sharded(args, snaps, src, config, rank, local_rank, world, K, W, host_cores):
    """N > 1: ONE KKT system factorised+solved by all GPUs together (elimination-tree subtree sharding, contribution
    blocks over NCCL send/recv) -> strong scaling of the same workload."""
    import torch
    import torch.distributed as dist
    from ipopt_b200.sharded import ShardedLdlt
    s0 = snaps[0]
    dim, nnz = s0["dim"], len(s0["irn"])
    # like-for-like point of the scaling curve: the SAME N=800 step on one GPU (rank 0, unsharded), measured in this run
    single = None
    if rank == 0:
        from ipopt_b200 import B200Ldlt
        one = B200Ldlt(device=local_rank)
        assert one.InitializeStructure(dim, nnz, s0["irn"], s0["jcn"]) == 0
        one.GetValuesArrayPtr()[:] = s0["val"]
        assert one.factor(True, s0["neg"])[0] == 0
        dv = [torch.from_numpy(sn["val"]).cuda() for sn in snaps]
        dr = [torch.from_numpy(sn["rhs"]).cuda() for sn in snaps]
        dw = torch.empty(dim, dtype=torch.float64, device="cuda")
        ks = max(3, min(K, 10))
        tot = 0.0
        for i in range(2 + ks):
            q = i % len(snaps)
            torch.cuda.synchronize(); t1 = time.perf_counter()
            assert one.factor_device(dv[q].data_ptr(), True, snaps[q]["neg"])[0] == 0
            for _ in range(2):
                dw.copy_(dr[q]); one.solve_device(dw.data_ptr(), 1)
            torch.cuda.synchronize()
            if i >= 2:
                tot += time.perf_counter() - t1
        single = {"ms_per_step": 1e3 * tot / ks, "steps": ks, "note": "same workload, unsharded, one GPU (rank 0), device-resident"}
        one.close(); del dv, dr, dw
        torch.cuda.empty_cache()
    dist.barrier()
    t0 = time.perf_counter()
    sh = ShardedLdlt(dim, s0["irn"], s0["jcn"], s0["val"], device=local_rank)
    t_analyse = time.perf_counter() - t0
    d_vals = [torch.from_numpy(sn["val"]).cuda() for sn in snaps]
    d_rhs = [torch.from_numpy(sn["rhs"]).cuda() for sn in snaps]

    last = [None, None, None]

    def step_device(i):
        sn = snaps[i % len(snaps)]
        st, neg = sh.factor_device(d_vals[i % len(snaps)], True, sn["neg"])
        assert st == 0 and neg == sn["neg"], (st, neg)
        for _ in range(2):
            x = sh.solve_device(d_rhs[i % len(snaps)])
        last[:] = [x, st, neg]

    def step_host(i):
        sn = snaps[i % len(snaps)]
        st, neg = sh.factor(sn["val"], True, sn["neg"])
        assert st == 0, st
        x = None
        for _ in range(2):
            x = sh.solve(sn["rhs"])
        return x

    def timed(fn):
        for i in range(W):
            fn(i)
        dist.barrier(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(sh.stream)
        for i in range(K):
            fn(W + i)
        e1.record(sh.stream)
        dist.barrier(); torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
        t = torch.tensor([e0.elapsed_time(e1), wall], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0]), float(t[1])

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    ms_dev, wall_dev = timed(step_device)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last[0].cpu().numpy(), last[1], last[2])
    ms_e2e, wall_e2e = timed(step_host)
    ms_dev, ms_e2e = max(ms_dev, wall_dev), max(ms_e2e, wall_e2e)
    sampler.stop_flag = True
    x = step_host(1)
    if rank == 0:
        r, xi, bi = sh.ranks[0].s.residual(x, snaps[1]["rhs"])
        own = sh.owner
        cfg = dict(config, parallelism="elimination-tree sharding over %d GPUs: %d subtrees below the cut, %d top fronts on rank 0; "
                   "contribution blocks / update vectors by NCCL send/recv" % (world, sh.n_subtrees, int((own == -1).sum())))
        line = {"metric": "kkt_factor_solve_iters_per_sec", "value": K / (ms_dev * 1e-3), "unit": "iter/s", "n_gpus": world,
                "steps": K, "warmup": W, "ms_per_step": ms_dev / K, "higher_is_better": True, "scaling": "strong",
                "vs_baseline": None, "dtype": "f64", "data": src, "config": cfg,
                "e2e": {"value": K / (ms_e2e * 1e-3), "unit": "iter/s", "ms_per_step": ms_e2e / K,
                        "h2d_bytes_per_step": world * 8 * nnz + 2 * world * 8 * dim, "d2h_bytes_per_step": 2 * 8 * dim + 32 * world},
                "gpu_launches": K * (sh.ranks[0].s.info()["launches_factor"] + 2 * 8), "analysis_once_s": {"wall": t_analyse},
                "single_gpu": single, "speedup_vs_single_gpu": (single["ms_per_step"] / (ms_dev / K)) if single else None,
                "parity": {"scaled_residual": r / (xi + bi)}, "clocks": sampler.summary(), "host_cores": host_cores}
        print(json.dumps(line))
    sh.close()
    dist.destroy_process_group()
    return 0


def get_snapshots_nodist(N=None):
    ws = os.environ.pop("WORLD_SIZE", None)
    try:
        return get_snapshots(0, N)
    finally:
        if ws is not None:
            os.environ["WORLD_SIZE"] = ws


if __name__ == "__main__":
    sys.exit(main())
