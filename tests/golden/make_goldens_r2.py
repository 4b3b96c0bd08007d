"""Round-2 golden fixtures, all produced by the REFERENCE's own interior-point loop (oracle/_ref libipopt.so) with the
CPU oracle as linear solver (tests/driver/ipopt_driver --backend oracle).  Needs the reference sources (driver build).

  python tests/golden/make_goldens_r2.py [small] [full] [control]

small   : <case>_final.npz for problems that exercise inertia correction (LukVlE2/E5), the restoration phase
          (start_with_resto=yes -> AugRestoSystemSolver) and L-BFGS (hessian_approximation=limited-memory ->
          LowRankAugSystemSolver, multi-rhs MultiSolve).
full    : BASELINE.json configs 4 and 5 (MDistCntrl3a N=600, MBndryCntrl1 N=800) and config 3 (N=400):
          runs/oracle_<problem>_<N>.json + <case>_final_sample.npz = every STRIDE-th entry of the final x / lambda / z
          (the full iterates are 5-20 MB; the sample keeps the fixture small) with max-norms.
control : runs/control_dual_spread.json -- the SAME oracle run again with another nested-dissection seed
          (ORACLE_METIS_SEED=7) and, at N=400, another pivot threshold / no scaling: the solver-to-solver spread of the
          final primal/dual iterates that two correct LDL^T solvers produce through the reference's IP loop.  The GPU
          parity test takes its dual-iterate tolerance from this file.
"""
import json
import os
import struct
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
DRIVER = os.path.join(ROOT, "tests", "driver", "ipopt_driver")
STRIDE = 97

SMALL = [
    ("LukVlE2", 1000, {}),
    ("LukVlE5", 1000, {}),
    ("MBndryCntrl1", 20, {"start_with_resto": "yes"}),
    ("LukVlI1", 200, {"start_with_resto": "yes"}),
    ("MDistCntrl3a", 20, {"hessian_approximation": "limited-memory"}),
    ("LukVlE1", 200, {"hessian_approximation": "limited-memory"}),
]
FULL = [("MBndryCntrl1", 400), ("MDistCntrl3a", 600), ("MBndryCntrl1", 800)]


def case_tag(name, N, opts):
    return "%s_%d" % (name, N) + "".join("_%s" % v.replace("-", "") for v in opts.values())


def read_final(path):
    with open(path, "rb") as f:
        n, m = struct.unpack("ii", f.read(8))
        obj, = struct.unpack("d", f.read(8))
        v = np.frombuffer(f.read(), dtype=np.float64)
    return dict(obj=obj, x=v[:n], z_L=v[n:2 * n], z_U=v[2 * n:3 * n], lam=v[3 * n:3 * n + m])


def run(name, N, opts=None, env=None, threads=8):
    with tempfile.TemporaryDirectory() as td:
        cmd = [DRIVER, "--backend", "oracle", "--problem", name, "--N", str(N), "--print-level", "0",
               "--json", os.path.join(td, "r.json"), "--final", os.path.join(td, "f.bin")]
        for k, v in (opts or {}).items():
            cmd += ["--opt", "%s=%s" % (k, v)]
        e = dict(os.environ, OMP_NUM_THREADS=str(threads))
        e.update(env or {})
        subprocess.check_call(cmd, stdout=subprocess.DEVNULL, env=e)
        return json.load(open(os.path.join(td, "r.json"))), read_final(os.path.join(td, "f.bin"))


def spread(a, b):
    zs = max(np.abs(a["z_L"]).max(), np.abs(a["z_U"]).max(), 1e-300)
    return {k: float(np.abs(a[k] - b[k]).max() / (zs if k.startswith("z_") else max(np.abs(a[k]).max(), 1e-300)))
            for k in ("x", "lam", "z_L", "z_U")}


def main(what):
    if "small" in what:
        for name, N, opts in SMALL:
            summ, fin = run(name, N, opts, threads=2)
            tag = case_tag(name, N, opts)
            np.savez_compressed(os.path.join(HERE, tag + "_final.npz"), iterations=summ["iterations"], n_factor=summ["n_factor"],
                                n_solve=summ["n_solve"], n_rhs=summ["n_rhs"], n_wrong_inertia=summ["n_wrong_inertia"],
                                status=summ["status"], **fin)
            print(tag, summ["iterations"], summ["n_factor"], summ["n_solve"], summ["n_rhs"], summ["n_wrong_inertia"], summ["objective"])
    base = {}
    if "full" in what or "control" in what:
        for name, N in FULL:
            summ, fin = run(name, N)
            base[(name, N)] = fin
            if "full" in what:
                json.dump(summ, open(os.path.join(HERE, "runs", "oracle_%s_%d.json" % (name, N)), "w"))
                np.savez_compressed(os.path.join(HERE, "%s_%d_final_sample.npz" % (name, N)), stride=STRIDE, obj=fin["obj"],
                                    iterations=summ["iterations"], n_factor=summ["n_factor"], n_solve=summ["n_solve"],
                                    **{k: fin[k][::STRIDE] for k in ("x", "lam", "z_L", "z_U")},
                                    **{k + "_absmax": np.abs(fin[k]).max() for k in ("x", "lam", "z_L", "z_U")})
            print(name, N, summ["iterations"], summ["objective"])
    if "control" in what:
        out = {"what": "max-norm relative difference of the final iterates between two runs of the SAME CPU oracle through the "
                       "reference's IP loop (z relative to max(|z_L|,|z_U|)); variant = environment of the second run",
               "runs": []}
        variants = {("MBndryCntrl1", 400): [{"ORACLE_METIS_SEED": "7"}, {"ORACLE_PIVTOL": "1e-8"}, {"ORACLE_SCALING": "0"}],
                    ("MDistCntrl3a", 600): [{"ORACLE_METIS_SEED": "7"}], ("MBndryCntrl1", 800): [{"ORACLE_METIS_SEED": "7"}]}
        for (name, N), vs in variants.items():
            for env in vs:
                summ, fin = run(name, N, env=env)
                rec = {"problem": name, "N": N, "variant": env, "iterations": summ["iterations"], "objective": summ["objective"],
                       "spread": spread(base[(name, N)], fin)}
                out["runs"].append(rec)
                print(rec)
        json.dump(out, open(os.path.join(HERE, "runs", "control_dual_spread.json"), "w"), indent=1)


if __name__ == "__main__":
    main(sys.argv[1:] or ["small", "full", "control"])
