"""The Ipopt-side adapter (ipopt_b200/plugin/B200LdltSolverInterface) driven by the reference's own IP loop with the CPU
oracle as its backend -- host logic only, no GPU: warm_start_same_structure, counters.  Test infrastructure: the oracle is
the checker's stand-in here, not a product path.  Needs tests/driver/ipopt_driver (built against the reference artefacts in oracle/_ref)."""
import json, os, subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "tests", "driver", "ipopt_driver")


def run_driver(args, tmp_path):
    if not os.path.exists(DRIVER):
        pytest.skip("tests/driver/ipopt_driver not built (needs the reference artefacts in oracle/_ref at build time)")
    js = str(tmp_path / "r.json")
    env = dict(os.environ, OMP_NUM_THREADS="4")
    p = subprocess.run([DRIVER, "--backend", "oracle", "--print-level", "0", "--json", js] + args, capture_output=True,
                       text=True, env=env, timeout=600)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    return json.load(open(js))


@pytest.mark.parametrize("problem,N", [("hs071", 0), ("MBndryCntrl1", 12)])
def test_warm_start_same_structure_keeps_the_analysis(problem, N, tmp_path):
    """reference contract IpMumpsSolverInterface.cpp:227-236: with warm_start_same_structure the second OptimizeNLP keeps the
    solver object's symbolic data; InitializeStructure must not hand the structure to the backend again."""
    s = run_driver(["--problem", problem, "--N", str(N), "--reopt"], tmp_path)
    assert s["status"] == 0 and s["reopt_status"] == 0
    assert s["n_analyse"] == 1
    assert s["reopt_iterations"] == s["iterations"]
    assert s["n_factor"] == 2 * s["n_factor_first"]


def test_counters_without_warm_start(tmp_path):
    s = run_driver(["--problem", "hs071"], tmp_path)
    assert s["n_analyse"] == 1 and s["reopt_status"] == -99
    assert s["iterations"] == 7 and s["n_factor"] == 12 and s["n_solve"] == 22      # SURVEY 8c: the reference's hs071 run
