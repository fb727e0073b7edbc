"""The transpose product's launch sequence on the host build (tests/hostsim): dab_bench_device runs the full product (selector 0),
the forward (1) and each reverse stage of the product alone (2-4: RevA, RevB, RevC; compressible: cRevA, cRevB, cRevE + cRevC; tile
product: the RevA tile, the fused RevB + RevC tile, nothing).  The per-kernel timings of bench.py and scripts/kbench.py are only
meaningful while each selector launches what the product launches, so the launch counts of every path are pinned here: one rank
with and without tiles, rolled face loops, a cyclic passage (ghost cells on one rank: the interior / cut-adjacent overlap of the
incompressible product, the blocking exchanges of the compressible one) and DARhoSimpleFoam.  The bench must also leave the
product's state alone: the public product after the bench is bitwise the one before it."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from tests.common import HOSTSIM, setup

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = 2  # bench calls per selector: the counts below are totals over both

# kernel launches of selectors 0-4 over CALLS calls
LAUNCHES = {
    "naca": [6, 6, 2, 2, 2],
    "naca_tile": [4, 6, 2, 2, 0],
    "naca_rolled": [6, 6, 2, 2, 2],
    "passage": [28, 18, 2, 2, 2],
    "passage_turbo": [28, 22, 2, 2, 4],
    "rhosimple": [8, 8, 2, 2, 4],
}


def _solver(path):
    """the solver of one path with its states assigned, and a seeded vector of its size"""
    if path.startswith("naca"):
        from tests.test_compressible_products import rolled_face_loops
        with rolled_face_loops(path == "naca_rolled"):
            mesh, bcs, orc, sol, W, _ = setup("naca", True, "linearUpwindV", lib_path=HOSTSIM)
        assert sol.getFaceLoopWidth() == (0 if path == "naca_rolled" else 6)
        sol.updateOFFields(W)
    elif path in ("passage", "passage_turbo"):
        from tests.test_cyclic import Pair
        P = Pair(True, "linearUpwind", lib_path=HOSTSIM, solver="DATurboFoam" if path == "passage_turbo" else "DASimpleFoam")
        sol = P.sol
        sol.updateOFFields(P.local(P.state()))
    else:
        from tests.test_compressible_products import Plain, make_solver
        c = Plain("channel_140")
        d = tempfile.mkdtemp(prefix="dab_drv_")
        c.write(d)
        sol = make_solver(c.spec["solver"], c.options, d, HOSTSIM)
        sol.updateOFFields(c.W)
    n = sol.getNLocalAdjointStates()
    return sol, np.random.default_rng(11).uniform(-1.0, 1.0, n)


def bench_launches(path):
    sol, psi = _solver(path)
    y0 = np.zeros(psi.size)
    sol.calcdRdWTPsiAD(psi, y0)
    sol.benchSetVector(psi[::-1].copy())
    counts = [sol.benchDevice(which, CALLS)[1] for which in range(5)]
    y1 = np.zeros(psi.size)
    sol.calcdRdWTPsiAD(psi, y1)
    assert np.array_equal(y0, y1), path
    assert np.any(y0 != 0.0)
    return counts


@pytest.mark.parametrize("path", ["naca", "naca_rolled", "passage", "passage_turbo", "rhosimple"])
def test_bench_selectors_launch_what_the_product_launches(path):
    assert bench_launches(path) == LAUNCHES[path]


def test_bench_selectors_of_the_tile_product():
    """DAB_TILE=1 is read when the solver is built: a child process, so that no other test's solver sees it"""
    code = "import json; from tests.test_product_driver import bench_launches; print('COUNTS', json.dumps(bench_launches('naca_tile')))"
    env = dict(os.environ, DAB_TILE="1", DAB_TILE_INFO="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "tiles:" in r.stderr  # the tile product is the one measured
    assert json.loads(r.stdout.split("COUNTS")[-1]) == LAUNCHES["naca_tile"]
