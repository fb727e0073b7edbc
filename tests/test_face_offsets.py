"""The transpose product reads the face-centre offsets Cf - C[own] and Cf - C[nei] that the mesh stores per internal face
(MeshView::offOwn / offNei) instead of gathering the face and cell centres on every face.  The stored arrays must give bitwise
the product taken from the centres, on every path that builds or rebuilds the geometry: the upload of the mesh, updateOFMesh
(on a partitioned mesh through the device geometry and the ghost-centre exchange), the geometry restored after a volCoord
product, and merged cyclic pairs whose neighbour is a periodic image.

The reference is a second host build of the same sources with DAB_FACE_OFFSETS_FROM_CENTRES, which takes the differences from
the centres in the accessor on every call (views.hpp faceOffsets); the comparison is exact equality, not a tolerance."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import pyDASolvers
from tests.common import HOSTSIM, NORM_STATES, ALL_RES, make_bcs, make_mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def centres_lib(tmp_path_factory):
    """The host build with the offsets taken from the centres: the recipe of tests/hostsim/Makefile plus the switch."""
    text = open(os.path.join(ROOT, "tests", "hostsim", "Makefile")).read()
    m = re.search(r"^\t\$\(CXX\) (.+?) -o \$@ \$\(SRC\)/capi\.cpp\s*$", text, re.M)
    assert m, "no host-build recipe in tests/hostsim/Makefile"
    out = str(tmp_path_factory.mktemp("offsets") / "libdab200_hostsim_centres.so")
    cmd = [os.environ.get("CXX", "g++"), *m.group(1).split(), "-DDAB_FACE_OFFSETS_FROM_CENTRES", "-o", out,
           os.path.join(ROOT, "dafoam_b200", "csrc", "capi.cpp")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    return out


def naca_case(kind, divU):
    mesh = make_mesh(kind, nk=2)
    d = tempfile.mkdtemp(prefix="dab_off_")
    cases.write_case(d, mesh, make_bcs(kind, True), div_u="bounded Gauss %s grad(U)" % divU)
    return d, (10.0, 0.5, 0.0)


def passage_case():
    """One passage of an annular duct with cyclic sides and an MRF zone over all its cells (DATurboFoam config-5 topology)."""
    mesh = cases.annular_passage(nr=4, nt=4, nz=6, n_sectors=5, sectors=1)
    bcs = cases.default_bcs_passage(Uin=(0.0, 0.0, 10.0), turbulent=True, cyclic=True)
    mrf = dict(cellZone="rotor", cells=np.arange(mesh.n_cells), origin=(0.0, 0.0, 0.0), axis=(0.0, 0.0, 1.0), omega=30.0,
               nonRotatingPatches=["inlet", "outlet", "shroud"])
    d = tempfile.mkdtemp(prefix="dab_off_")
    cases.write_case(d, mesh, bcs, div_u="bounded Gauss linearUpwind grad(U)", mrf=mrf)
    return d, (0.0, 0.0, 10.0)


CASES = {
    "naca_sa": lambda: naca_case("naca", "linearUpwind"),
    "naca_wallfunction_luv": lambda: naca_case("nacawf", "linearUpwindV"),  # the FEAT 3 kernel: limiter + wall function
    "passage_cyclic_mrf": passage_case,
}


def state(sol, U0, rng):
    nC, n = sol.getNLocalCells(), sol.getNLocalAdjointStates()
    W = np.empty(n)
    W[:3 * nC] = (np.array(U0) + rng.uniform(-1.0, 1.0, (nC, 3))).ravel()
    W[3 * nC:4 * nC] = rng.uniform(-5.0, 5.0, nC)
    W[4 * nC:5 * nC] = 4.5e-5 * (1.0 + 0.5 * rng.uniform(-1.0, 1.0, nC))
    W[5 * nC:] = rng.uniform(-0.01, 0.01, n - 5 * nC)
    return W


def moved(pts, periodic):
    """A smooth displacement of the points; about the z axis it commutes with rotations (periodic across cyclic pairs)."""
    X = pts.reshape(-1, 3)
    if periodic:
        s = 1.0 + 0.02 * np.sin(7.0 * X[:, 2])
        out = np.stack([X[:, 0] * s, X[:, 1] * s, X[:, 2] + 0.01 * (X[:, 0] ** 2 + X[:, 1] ** 2)], axis=1)
    else:
        out = X + np.stack([2e-3 * np.sin(3.0 * X[:, 1]), 2e-3 * np.cos(2.0 * X[:, 0]), np.zeros(len(X))], axis=1)
    return np.ascontiguousarray(out.ravel())


def products(lib, name):
    """dRdWT psi at the mesh as read, after updateOFMesh, and after a volCoord product at the moved mesh."""
    d, U0 = CASES[name]()
    opts = dict(normalizeStates=NORM_STATES, normalizeResiduals=list(ALL_RES))
    sol = pyDASolvers("DASimpleFoam -python", opts, caseDir=d, _lib_path=lib)
    rng = np.random.default_rng(2024)
    W = state(sol, U0, rng)
    psi = rng.uniform(-1.0, 1.0, len(W))
    out = []

    def product():
        y = np.zeros(len(W))
        sol.calcdRdWTPsiAD(psi, y)
        out.append(y)

    sol.updateOFFields(W)
    product()
    pts = np.zeros(3 * sol.getNLocalPoints())
    sol.getOFMeshPoints(pts)
    sol.updateOFMesh(moved(pts, name.startswith("passage")))
    sol.updateOFFields(W)
    product()
    sol.getOFMeshPoints(pts)
    xv = np.zeros(len(pts))
    sol.calcJacTVecProduct("aero_vol_coords", "volCoord", pts, "R", "residual", psi, xv)
    sol.updateOFFields(W)
    product()
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_stored_offsets_give_the_product_of_the_centres_host_build(centres_lib, name):
    ours, ref = products(HOSTSIM, name), products(centres_lib, name)
    for y in ours:
        assert np.all(np.isfinite(y)) and np.any(y != 0.0)
    assert not np.array_equal(ours[0], ours[1]), "moving the points did not change the product"
    for k, what in enumerate(("mesh as read", "after updateOFMesh", "after a volCoord product")):
        diff = np.flatnonzero(ours[k] != ref[k])
        assert diff.size == 0, "%s, %s: %d entries differ, largest %.3e" % (name, what, diff.size, np.abs(ours[k] - ref[k]).max())
