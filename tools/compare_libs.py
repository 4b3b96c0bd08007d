"""Bit-for-bit comparison of two builds of libb200ldlt.so on the same seeded systems: every output array of every call
that reads the factors, every launch count and the pivoting counters of every factorisation.  Meant for changes that
must not change a bit: refactors of the host code, and of the factor kernels, whose every front class (B200_NO_WARP2=1
sends the fronts of order 33..64 through the shared-memory kernel) and forced-pivot path (lifted pivots, zero pivots,
lifted zeros) is dumped.  Build the other library into a directory of its own, then

  python tools/compare_libs.py dump <libb200ldlt.so> <out.json>    (one process per library: one CUDA context each)
  python tools/compare_libs.py compare <a.json> <b.json>           (exit 1 on any difference)

The dump holds the SHA-256 of the bytes of each array (the full arrays run to gigabytes), the launch counts, and after
every factorisation num_neg, num_forced, num_tiny, num_2x2 and num_growth.

What is dumped, per system (seeded generators, the golden systems of tests/golden and a tridiagonal whose pivots are
lifted):
  * factor with use_graph 1 (and its replay), use_graph 0, B200_ONE_STREAM=1, B200_SOLVE_BLOCK=1, B200_SOLVE_BLOCK=3,
    B200_SOLVE_DIRECT=0 and B200_NO_WARP2=1: status, inertia, launches_factor, D^-1 (enquire_indef) and host solves of
    1, 8 and 13 columns with launches_solve;
  * on the use_graph 1 handle: device solves of 1, 8 and 13 columns, jobs 1..4 (host 1 and 13 columns, device 8),
    lmultiply (trans 0 / 1, host 1 and 13, device 8), selected inversion, solve_refine_device, the Fredholm solve
    without zero pivots, the error analysis (host 1 and 13 columns with and without the condition estimate, device 8)
    and the refined solve (host 3 columns, device 1);
  * on every handle of the first item, the calls that run pruned sweeps, host and device, each followed by the four run
    sets of symbolic_array: the sparse forward solve; inverse_entries (a diagonal, an off-diagonal entry in both orders,
    the first and last variable -- different trees on the two-component system --, and a block of 20 x 20 entries,
    wider than the blocked-solve width); the sparse solve with 1 and 13 columns (sparse b with a selection, dense b with
    a selection, sparse b with every entry, both NULL);
  * the Fredholm solve on kept singular factors, blocked, with B200_SOLVE_BLOCK=1 and with B200_NO_WARP2=1 (host 1, 5
    and 13 columns, device 5);
  * the duplicated-constraint systems of tests/test_fredholm.py in keep mode, both orderings, default and
    B200_NO_WARP2=1: status, last_error, the counters and the zero pivots where the factors are kept (a "lifted zero"
    keeps none);
  * Schur mode with the root in each solve class: S_c, reduce and expand (host 1 and 11 columns, device 8);
  * the sharded factor and solve with 2 and 4 ranks emulated on one GPU, on two matrices.
Needs a GPU, torch and the test helpers in tests/."""
import contextlib
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COUNTERS = ("num_neg", "num_forced", "num_tiny", "num_2x2", "num_growth")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


@contextlib.contextmanager
def env(**kw):
    """environment switches of the handles created inside (the library reads them at b200ldlt_create)"""
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update(kw)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def lifted_tridiagonal(n=2000):
    """the system of tests/test_error_analysis.py::test_lifted_pivots_give_finite_estimates: a tiny diagonal under a unit
    off-diagonal, whose factorisation lifts pivots (num_forced > 0)"""
    irn = np.concatenate([np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int32)
    jcn = np.concatenate([np.arange(1, n + 1), np.arange(1, n)]).astype(np.int32)
    val = np.concatenate([1e-10 * (1 + np.arange(n) % 3), np.ones(n - 1)])
    return n, irn, jcn, val


# (nx, nc, seed) of the duplicated-constraint systems (dup_kkt) of tests/test_fredholm.py::test_dependent_rows
DEPENDENT_ROWS = [(40, 12, 0), (120, 40, 1), (300, 100, 2)]


def dump(lib, out):
    import ipopt_b200.capi as capi
    capi.lib_path = lambda: os.path.abspath(lib)
    import torch
    from ipopt_b200 import B200Ldlt, SYMSOLVER_SUCCESS
    from ipopt_b200.kkt import mbndry_kkt
    from ipopt_b200.sharded import ShardedLdlt
    from test_partial_solve import LARGE, SYSTEMS
    from test_fredholm import dup_kkt, zeroed
    from test_inverse_entries import two_components
    from test_schur import dense, pick_vars

    rec = {}

    def put(key, *arrays):
        assert key not in rec, key
        h = hashlib.sha256()
        for a in arrays:
            a = np.asarray(a)
            h.update(np.ascontiguousarray(a, dtype=np.float64 if a.dtype.kind == "f" else np.int64).tobytes())
        rec[key] = h.hexdigest()

    def launches(s, key):
        inf = s.info()
        rec[key + "#launches"] = [inf["launches_factor"], inf["launches_solve"]]

    def dev(a):
        return torch.tensor(np.ascontiguousarray(a).ravel(), dtype=torch.float64, device="cuda")

    def handle(dim, irn, jcn, val, keep=0, **opts):
        s = B200Ldlt(**opts)
        assert s.InitializeStructure(dim, len(irn), irn, jcn) == SYMSOLVER_SUCCESS
        if keep:
            assert s.set_singular_action(1) == SYMSOLVER_SUCCESS
        s.GetValuesArrayPtr()[:] = val
        return s

    def factor(s, key):
        st, neg = s.factor(False, 0)
        put(key + "/factor", np.array([st, neg]))
        launches(s, key + "/factor")
        inf = s.info()
        rec[key + "/factor#counters"] = [inf[k] for k in COUNTERS]
        return st

    def host_solves(s, key, dim, rng, widths=(1, 8, 13)):
        for w in widths:
            X = rng.standard_normal(dim * w)
            assert s.solve(X, w) == SYMSOLVER_SUCCESS, s.last_error()
            put("%s/solve%d" % (key, w), X)
            launches(s, "%s/solve%d" % (key, w))

    def run_sets(s, key):
        for name in ("sparse_run_set", "inverse_run_set", "sparse_solve_fwd_run_set", "sparse_solve_bwd_run_set"):
            put("%s/%s" % (key, name), s.symbolic(name))

    def pruned_suite(s, key, dim, rng):
        for k in (1, 5, min(50, dim)):
            bi = np.sort(rng.choice(dim, k, replace=False)).astype(np.int32)
            b = rng.standard_normal(k)
            xi, x = s.sparse_fwd_solve(bi, b)
            put("%s/sfs%d" % (key, k), xi, x)
            launches(s, "%s/sfs%d" % (key, k))
            run_sets(s, "%s/sfs%d" % (key, k))
            Bd, Xd = dev(b), torch.zeros(dim, dtype=torch.float64, device="cuda")
            xi = s.sparse_fwd_solve_device(bi, Bd.data_ptr(), Xd.data_ptr())
            put("%s/sfs_dev%d" % (key, k), xi, Xd.cpu().numpy()[:len(xi)])
            launches(s, "%s/sfs_dev%d" % (key, k))
            run_sets(s, "%s/sfs_dev%d" % (key, k))
        i, j = (int(v) for v in rng.choice(dim, 2, replace=False))
        blk = rng.choice(dim, min(20, dim), replace=False)
        bi, bj = np.meshgrid(blk, blk, indexing="ij")
        sets = {"diag": ([i], [i]), "ij": ([i], [j]), "ji": ([j], [i]), "ends": ([0, dim - 1], [dim - 1, 0]),
                "block20": (bi.ravel(), bj.ravel())}
        for name, (irow, jcol) in sets.items():
            irow, jcol = np.asarray(irow, np.int32), np.asarray(jcol, np.int32)
            tag = "%s/inv_%s" % (key, name)
            put(tag, s.inverse_entries(irow, jcol))
            launches(s, tag)
            run_sets(s, tag)
            V = torch.zeros(len(irow), dtype=torch.float64, device="cuda")
            assert s.inverse_entries_device(irow, jcol, V.data_ptr()) == SYMSOLVER_SUCCESS, s.last_error()
            put(tag + "_dev", V.cpu().numpy())
            launches(s, tag + "_dev")
            run_sets(s, tag + "_dev")
        bi = np.sort(rng.choice(dim, min(5, dim), replace=False)).astype(np.int32)
        xs = rng.choice(dim, min(7, dim), replace=False).astype(np.int32)
        for w in (1, 13):
            for mode, (bindex, xsel) in (("sparse_sel", (bi, xs)), ("dense_sel", (None, xs)), ("sparse_all", (bi, None)),
                                         ("dense_all", (None, None))):
                nbi = dim if bindex is None else len(bindex)
                nxs = dim if xsel is None else len(xsel)
                B = rng.standard_normal((w, nbi))
                tag = "%s/sps_%s_%d" % (key, mode, w)
                put(tag, s.sparse_solve(bindex, B, xsel))
                launches(s, tag)
                run_sets(s, tag)
                Bd, Xd = dev(B), torch.zeros(w * nxs, dtype=torch.float64, device="cuda")
                assert s.sparse_solve_device(bindex, Bd.data_ptr(), xsel, Xd.data_ptr(), w) == SYMSOLVER_SUCCESS, \
                    s.last_error()
                put(tag + "_dev", Xd.cpu().numpy())
                launches(s, tag + "_dev")
                run_sets(s, tag + "_dev")

    def full_suite(s, key, dim, nnz, rng):
        for w in (1, 8, 13):
            X = dev(rng.standard_normal(dim * w))
            assert s.solve_device(X.data_ptr(), w) == SYMSOLVER_SUCCESS, s.last_error()
            put("%s/solve_dev%d" % (key, w), X.cpu().numpy())
            launches(s, "%s/solve_dev%d" % (key, w))
        for job in (1, 2, 3, 4):
            for w in (1, 13):
                X = rng.standard_normal(dim * w)
                assert s.solve_partial(job, X, w) == SYMSOLVER_SUCCESS, s.last_error()
                put("%s/job%d_%d" % (key, job, w), X)
                launches(s, "%s/job%d_%d" % (key, job, w))
            X = dev(rng.standard_normal(dim * 8))
            assert s.solve_partial_device(job, X.data_ptr(), 8) == SYMSOLVER_SUCCESS, s.last_error()
            put("%s/job%d_dev8" % (key, job), X.cpu().numpy())
            launches(s, "%s/job%d_dev8" % (key, job))
        for trans in (0, 1):
            for w in (1, 13):
                put("%s/lmul%d_%d" % (key, trans, w), s.lmultiply(trans, rng.standard_normal(dim * w), w))
                launches(s, "%s/lmul%d_%d" % (key, trans, w))
            X, Y = dev(rng.standard_normal(dim * 8)), torch.zeros(dim * 8, dtype=torch.float64, device="cuda")
            assert s.lmultiply_device(trans, X.data_ptr(), Y.data_ptr(), 8) == SYMSOLVER_SUCCESS, s.last_error()
            put("%s/lmul%d_dev8" % (key, trans), Y.cpu().numpy())
            launches(s, "%s/lmul%d_dev8" % (key, trans))
        d, v = s.selected_inverse(True, True)
        put(key + "/selinv", d, v)
        launches(s, key + "/selinv")
        X = dev(rng.standard_normal(dim))
        st, steps, ratio = s.solve_refine_device(X.data_ptr(), 1, 3, 0.0)
        put(key + "/refine", np.array([st, steps]), np.array([ratio]), X.cpu().numpy())
        X, F, c = s.solve_fredholm(rng.standard_normal((dim, 3)), 1e-10)
        put(key + "/fred_nonsingular", X, F, c)
        launches(s, key + "/fred_nonsingular")
        for w in (1, 13):
            B, X = rng.standard_normal((dim, w)), rng.standard_normal((dim, w))
            for cond in (0, 1):
                e = s.error_analysis(B, X, cond)
                put("%s/ea%d_cond%d" % (key, w, cond), *(e[k] for k in sorted(e)))
                launches(s, "%s/ea%d_cond%d" % (key, w, cond))
        Bd, Xd = dev(rng.standard_normal(dim * 8)), dev(rng.standard_normal(dim * 8))
        st, e = s.error_analysis_device(Bd.data_ptr(), Xd.data_ptr(), 8)
        put(key + "/ea_dev8", np.array([st]), *(e[k] for k in sorted(e)))
        launches(s, key + "/ea_dev8")
        X, r = s.solve_refined(rng.standard_normal((dim, 3)), 3)
        put(key + "/refined3", X, *(r[k] for k in sorted(r)))
        launches(s, key + "/refined3")
        Bd, Xd = dev(rng.standard_normal(dim)), torch.zeros(dim, dtype=torch.float64, device="cuda")
        st, r = s.solve_refined_device(Bd.data_ptr(), Xd.data_ptr(), 1, 3)
        put(key + "/refined_dev1", np.array([st]), Xd.cpu().numpy(), *(r[k] for k in sorted(r)))
        launches(s, key + "/refined_dev1")
        assert nnz == len(v)

    rng = np.random.default_rng(2024)
    systems = {name: SYSTEMS[name] for name in ("MBndryCntrl1_30", "LukVlE1_1000", "random", "mbndry30_wzero")}
    systems["mbndry400"] = LARGE
    systems["mbndry60"] = lambda: mbndry_kkt(60, sigma_spread=3.0, seed=9)[:4]
    systems["forest"] = two_components
    systems["lifted"] = lifted_tridiagonal
    for name, make in systems.items():
        dim, irn, jcn, val = make()
        for tag, opts, sw in (("graph", {}, {}), ("nograph", {"use_graph": 0}, {}),
                              ("onestream", {}, {"B200_ONE_STREAM": "1"}), ("block1", {}, {"B200_SOLVE_BLOCK": "1"}),
                              ("block3", {}, {"B200_SOLVE_BLOCK": "3"}), ("direct0", {}, {"B200_SOLVE_DIRECT": "0"}),
                              ("nowarp2", {}, {"B200_NO_WARP2": "1"})):
            key = "%s/%s" % (name, tag)
            with env(**sw):
                s = handle(dim, irn, jcn, val, **opts)
                if factor(s, key) != SYMSOLVER_SUCCESS:
                    s.close()
                    continue
                factor(s, key + "/again")
                put(key + "/dinv", s.enquire_indef()[2])
                host_solves(s, key, dim, rng)
                pruned_suite(s, key, dim, rng)
                if tag == "graph":
                    full_suite(s, key, dim, len(irn), rng)
                s.close()
        print("dumped", name, flush=True)

    for system, k in (("random", 1), ("random", 3), ("mbndry400", 3)):
        dim, irn, jcn, val, rows = zeroed(system, k)
        for tag, sw in (("blocked", {}), ("block1", {"B200_SOLVE_BLOCK": "1"}), ("nowarp2", {"B200_NO_WARP2": "1"})):
            key = "fred/%s_%d/%s" % (system, k, tag)
            with env(**sw):
                s = handle(dim, irn, jcn, val, keep=1)
                factor(s, key)
                put(key + "/zpos", s.enquire_zero_pivots())
                for w in (1, 5, 13):
                    X, F, c = s.solve_fredholm(rng.standard_normal((dim, w)), 1e-10)
                    put("%s/host%d" % (key, w), X, F, c)
                    launches(s, "%s/host%d" % (key, w))
                Xd = torch.zeros(2 * 5 * dim, dtype=torch.float64, device="cuda")
                Xd[:5 * dim] = dev(rng.standard_normal(5 * dim))
                st, c = s.solve_fredholm_device(Xd.data_ptr(), 5, 1e-10)
                put(key + "/dev5", np.array([st]), Xd.cpu().numpy(), c)
                launches(s, key + "/dev5")
                host_solves(s, key, dim, rng, (1, 8))
                s.close()
        print("dumped fredholm", system, flush=True)

    for nx, nc, seed in DEPENDENT_ROWS:
        dim, irn, jcn, val, _ = dup_kkt(nx, nc, seed)
        for ordering in (0, 1):
            for tag, sw in (("default", {}), ("nowarp2", {"B200_NO_WARP2": "1"})):
                key = "dependent/%d_%d_%d/o%d/%s" % (nx, nc, seed, ordering, tag)
                with env(**sw):
                    s = handle(dim, irn, jcn, val, keep=1, ordering=ordering)
                    factor(s, key)
                    err = s.last_error()
                    rec[key + "/last_error"] = err
                    if "no factors" not in err:
                        put(key + "/zpos", s.enquire_zero_pivots())
                    s.close()
    print("dumped dependent rows", flush=True)

    for system, m in (("random", 20), ("random", 64), ("random_300_100", 150), ("random", 300)):
        dim, irn, jcn, val, A = dense(system)
        vars = pick_vars(A, m, m)
        key = "schur/%s_%d" % (system, m)
        s = handle(dim, irn, jcn, val)
        assert s.set_schur(vars) == SYMSOLVER_SUCCESS
        factor(s, key)
        put(key + "/sc", s.schur_complement())
        launches(s, key + "/sc")
        for w in (1, 11):
            B = rng.standard_normal((dim, w))
            put("%s/reduce%d" % (key, w), s.schur_reduce(B))
            launches(s, "%s/reduce%d" % (key, w))
            put("%s/expand%d" % (key, w), s.schur_expand(B, rng.standard_normal((m, w))))
            launches(s, "%s/expand%d" % (key, w))
        Bd, Y = dev(rng.standard_normal(dim * 8)), torch.zeros(m * 8, dtype=torch.float64, device="cuda")
        assert s.schur_reduce_device(Bd.data_ptr(), Y.data_ptr(), 8) == SYMSOLVER_SUCCESS, s.last_error()
        put(key + "/reduce_dev8", Y.cpu().numpy())
        launches(s, key + "/reduce_dev8")
        Xs, Xd = dev(rng.standard_normal(m * 8)), torch.zeros(dim * 8, dtype=torch.float64, device="cuda")
        assert s.schur_expand_device(Bd.data_ptr(), Xs.data_ptr(), Xd.data_ptr(), 8) == SYMSOLVER_SUCCESS, s.last_error()
        put(key + "/expand_dev8", Xd.cpu().numpy())
        launches(s, key + "/expand_dev8")
        s.close()
        print("dumped schur", system, m, flush=True)

    dim, irn, jcn, val, nc = mbndry_kkt(60, sigma_spread=3.0, seed=9)
    v0 = mbndry_kkt(60, w_zero=True)[3]
    for world in (2, 4):
        key = "shard/%d" % world
        sh = ShardedLdlt(dim, irn, jcn, v0, local_world=world)
        for i, v in enumerate((val, val * np.where(np.arange(len(val)) < dim // 2, 1.5, 1.0))):
            st, neg = sh.factor(v, True, nc)
            put("%s/factor%d" % (key, i), np.array([st, neg]))
            rec["%s/factor%d#launches" % (key, i)] = [inf["launches_factor"] for inf in sh.info().values()]
            put("%s/solve%d" % (key, i), sh.solve(rng.standard_normal(dim)))
            Xd = sh.solve_device(dev(rng.standard_normal(dim)))
            sh.stream.synchronize()
            put("%s/solve_dev%d" % (key, i), Xd.cpu().numpy())
        sh.close()
        print("dumped shard", world, flush=True)
    with open(out, "w") as f:
        json.dump(rec, f, indent=0, sort_keys=True)
    print("%d entries -> %s" % (len(rec), out))


def compare(a, b):
    with open(a) as f:
        A = json.load(f)
    with open(b) as f:
        B = json.load(f)
    bad = sorted(k for k in set(A) | set(B) if A.get(k) != B.get(k))
    n = sum(1 for k in A if k.endswith("#launches"))
    c = sum(1 for k in A if k.endswith("#counters"))
    print("%d entries (%d launch counts, %d factorisations' counters) compared, %d differ%s" % (
        len(set(A) | set(B)), n, c, len(bad), "" if not bad else ": " + ", ".join(bad[:20])))

    def nonzero(field, nowarp2):
        i = COUNTERS.index(field)
        return sum(1 for k, v in A.items() if k.endswith("#counters") and v[i] > 0 and ("/nowarp2/" in k) == nowarp2)
    print("factorisations with num_forced > 0: %d default, %d B200_NO_WARP2=1; with num_tiny > 0: %d default, %d "
          "B200_NO_WARP2=1" % (nonzero("num_forced", False), nonzero("num_forced", True), nonzero("num_tiny", False),
                               nonzero("num_tiny", True)))
    return 1 if bad else 0


if __name__ == "__main__":
    cmd = sys.argv[1] if len(sys.argv) > 1 else ""
    if cmd == "dump" and len(sys.argv) == 4:
        dump(sys.argv[2], sys.argv[3])
    elif cmd == "compare" and len(sys.argv) == 4:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
