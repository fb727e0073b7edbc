"""updateOFMesh and the `volCoord` input on partitioned local meshes: a cyclic passage on one rank (its periodic images are ghost
cells) and, through tests/mp_volcoord_worker.py, the NACA O-grid and the passage on several gloo ranks against one rank.

The device geometry pipeline rebuilds the local mesh from the full point list; a moved mesh must give the residual and the forces
of a solver constructed on a case written with the moved points, and the coloured central-difference products must agree with
finite differences through updateOFMesh."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import pyDASolvers
from tests.common import HOSTSIM, NORM_STATES, ROOT

N_SECTORS = 7
FN = {"CD": {"type": "force", "source": "patchToFace", "patches": ["hub"], "directionMode": "fixedDirection", "direction": [0.0, 0.0, 1.0],
             "scale": 1.0}}
TURBO_OPTS = dict(normalizeStates=dict(U=50.0, p=101325.0, T=300.0, nuTilda=1e-3, phi=1.0), function=FN)


def passage_mesh(kind):
    if "axial" in kind:
        return cases.annular_passage(nr=4, nt=4, nz=16, lz=0.9, n_sectors=N_SECTORS)
    return cases.annular_passage(nr=5, nt=6, nz=8, n_sectors=N_SECTORS)


def write_passage(d, kind, mesh=None, turbulent=True):
    """the passage of tests/test_multirank.py (DATurboFoam + MRF for 'turbo'); returns the solver name and its options"""
    mesh = passage_mesh(kind) if mesh is None else mesh
    bcs = cases.default_bcs_passage(Uin=(0.0, 0.0, 60.0 if "turbo" in kind else 10.0), turbulent=turbulent)
    kw = {}
    if "turbo" in kind:
        bcs = cases.compressible_bcs(bcs)
        kw = dict(thermo=cases.default_thermo(energy="sensibleEnthalpy"),
                  mrf=dict(cellZone="rotor", cells=list(range(mesh.n_cells)), origin=(0.0, 0.0, 0.0), axis=(0.0, 0.0, 1.0), omega=200.0,
                           nonRotatingPatches=["inlet", "outlet", "shroud"]))
    cases.write_case(d, mesh, bcs, **kw)
    if "turbo" in kind:
        return "DATurboFoam -python", dict(TURBO_OPTS)
    return "DASimpleFoam -python", dict(normalizeStates=NORM_STATES, function=FN)


def periodic_displacement(pts, amp=2e-3):
    """a smooth displacement of the passage that repeats from passage to passage (a function of r, z and N theta in the cylindrical
    frame); zero on the hub, the shroud, the inlet and the outlet"""
    X = pts.reshape(-1, 3)
    r, th, z = np.hypot(X[:, 0], X[:, 1]), np.arctan2(X[:, 1], X[:, 0]), X[:, 2]
    eta = (r - r.min()) / (r.max() - r.min())
    zeta = (z - z.min()) / (z.max() - z.min())
    bump = amp * np.sin(np.pi * eta) * np.sin(np.pi * zeta)
    dr = bump * (1.0 + 0.5 * np.cos(N_SECTORS * th))
    dt = 0.6 * bump * np.cos(2.0 * np.pi * zeta)
    dz = 0.5 * bump * np.sin(N_SECTORS * th)
    v = np.stack([dr * np.cos(th) - dt * np.sin(th), dr * np.sin(th) + dt * np.cos(th), dz], axis=1)
    return v.ravel()


def perturbed_state(sol, seed=5):
    W = np.zeros(sol.getNLocalAdjointStates())
    sol.getOFFields(W)
    rng = np.random.default_rng(seed)
    W *= 1.0 + 0.01 * rng.uniform(-1, 1, W.size)
    nC = sol.getNLocalCells()
    W[:3 * nC] += 0.3 * rng.uniform(-1, 1, 3 * nC)
    return W


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def run_moved_case(lib_path, kind):
    """after a periodic displacement, the residual and the force of a solver constructed on a case written with the moved points.
    Laminar: the wall distance stays frozen under updateOFMesh (meshWaveFrozen), a new solver computes it on the moved mesh."""
    d = tempfile.mkdtemp(prefix="dab_vcp_")
    mesh = passage_mesh(kind)
    name, opts = write_passage(d, kind, mesh, turbulent=False)
    sol = pyDASolvers(name, opts, caseDir=d, _lib_path=lib_path)
    W = perturbed_state(sol)
    sol.updateOFFields(W)
    n, nP3 = W.size, 3 * sol.getNLocalPoints()
    owned = np.concatenate([np.ones((W.size - sol.getNLocalFaces()), dtype=bool), sol.getLocalToGlobal("faceOwned").astype(bool)])
    pts = np.zeros(nP3)
    sol.getOFMeshPoints(pts)
    R0 = np.zeros(n)
    sol.getResiduals(R0)
    v = periodic_displacement(pts)
    sol.updateOFMesh(pts + v)
    Rm = np.zeros(n)
    sol.getResiduals(Rm)
    Fm = sol.calcFunction("CD")
    moved = cases.PolyMesh.__new__(cases.PolyMesh)
    moved.__dict__.update(mesh.__dict__)
    moved.points = np.ascontiguousarray((pts + v).reshape(-1, 3))
    d2 = tempfile.mkdtemp(prefix="dab_vcp_")
    write_passage(d2, kind, moved, turbulent=False)
    fresh = pyDASolvers(name, opts, caseDir=d2, _lib_path=lib_path)
    fresh.updateOFFields(W)
    Rf = np.zeros(n)
    fresh.getResiduals(Rf)
    assert rel(Rm[owned], Rf[owned]) < 1e-12, rel(Rm[owned], Rf[owned])
    assert rel(Rm[owned], R0[owned]) > 1e-6  # the displacement does change the residual
    Ff = fresh.calcFunction("CD")
    assert abs(Fm - Ff) <= 1e-12 * abs(Ff), (Fm, Ff)


def run_cyclic_passage(lib_path, kind):
    d = tempfile.mkdtemp(prefix="dab_vcp_")
    mesh = passage_mesh(kind)
    name, opts = write_passage(d, kind, mesh)
    sol = pyDASolvers(name, opts, caseDir=d, _lib_path=lib_path)
    W = perturbed_state(sol)
    sol.updateOFFields(W)
    n, nP3 = W.size, 3 * sol.getNLocalPoints()
    owned = np.concatenate([np.ones((W.size - sol.getNLocalFaces()), dtype=bool), sol.getLocalToGlobal("faceOwned").astype(bool)])
    pts = np.zeros(nP3)
    sol.getOFMeshPoints(pts)
    R0 = np.zeros(n)
    sol.getResiduals(R0)
    F0 = sol.calcFunction("CD")

    # the device pipeline at the unmoved points reproduces the host-sliced geometry
    sol.updateOFMesh(pts)
    R1 = np.zeros(n)
    sol.getResiduals(R1)
    assert rel(R1[owned], R0[owned]) < 1e-12, rel(R1[owned], R0[owned])

    # a periodic displacement (compared with a freshly constructed solver in run_moved_case)
    v = periodic_displacement(pts)
    sol.updateOFMesh(pts + v)
    Rm = np.zeros(n)
    sol.getResiduals(Rm)
    assert rel(Rm[owned], R0[owned]) > 1e-6

    # a displacement that is not periodic is refused and leaves the mesh as it was
    bad = pts + v
    cyc = [p for p in mesh.patches if p["type"] == "cyclic"][0]
    q = int(mesh.faces[cyc["start"]][0])
    bad[3 * q:3 * q + 3] += 1e-3
    with pytest.raises(RuntimeError, match="periodic"):
        sol.updateOFMesh(bad)
    R2 = np.zeros(n)
    sol.getResiduals(R2)
    assert np.array_equal(R2, Rm)

    # restoring the points restores the residual: bitwise the first rebuild at these points
    sol.updateOFMesh(pts)
    R3 = np.zeros(n)
    sol.getResiduals(R3)
    assert np.array_equal(R3, R1)
    assert abs(sol.calcFunction("CD") - F0) <= 1e-12 * abs(F0)

    # the products: directional checks through updateOFMesh for a periodic displacement
    rng = np.random.default_rng(3)
    psi = rng.uniform(-1, 1, n)
    psi[~owned] = 0.0
    prod = np.zeros(nP3)
    sol.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", psi, prod)
    R4 = np.zeros(n)
    sol.getResiduals(R4)
    assert np.array_equal(R4, R1)  # the geometry of before the product, exactly
    dFdx = np.zeros(nP3)
    sol.calcJacTVecProduct("x", "volCoord", pts, "CD", "function", np.array([1.0]), dFdx)
    assert np.linalg.norm(prod) > 0 and np.linalg.norm(dFdx) > 0
    h = 1e-3
    sol.updateOFMesh(pts + h * v)
    Rp, Fp = np.zeros(n), sol.calcFunction("CD")
    sol.getResiduals(Rp)
    sol.updateOFMesh(pts - h * v)
    Rq, Fq = np.zeros(n), sol.calcFunction("CD")
    sol.getResiduals(Rq)
    sol.updateOFMesh(pts)
    fd = psi @ (Rp - Rq) / (2 * h)
    assert abs(fd - prod @ v) <= 1e-5 * abs(fd), (fd, prod @ v)
    fdF = (Fp - Fq) / (2 * h)
    assert abs(fdF - dFdx @ v) <= 1e-5 * abs(fdF), (fdF, dFdx @ v)


def run_ring_comparison(lib_path, solver, mrf_omega, tol=1e-7):
    """[dR/dx_v]^T psi of the cyclic passage against the oracle's exact tape product through the geometry on the closed ring of
    passages (tests/test_cyclic.py Pair), per point, with a state and psi that repeat from passage to passage.

    Convention: the engine merges each coupled face pair into one face that keeps the points of the first patch (mesh.hpp
    mergeCyclics), so the coupled face's geometry depends on the first patch's points only, while the other faces at a second-patch
    point still depend on it.  The ring has one point where the passage has a coupled pair (x_hi = R x_lo).  Hence:
    * a point on neither cyclic patch: engine value == ring value at its passage-0 instance;
    * a coupled pair: g_lo + R^T g_hi == ring value at x_lo (the lumped derivative; exact for periodic displacements);
    * for a periodic displacement v: prod . v == ring jtvec_xv . v_ring / N_SECTORS."""
    from scipy.spatial import cKDTree
    from tests.common import rel_err
    from tests.test_cyclic import N_SECTORS as NS, Pair, rotz
    P = Pair(True, "linearUpwind", lib_path=lib_path, solver=solver, mrf_omega=mrf_omega)
    W = P.state()
    P.sol.updateOFFields(P.local(W))
    psi = np.random.default_rng(11).uniform(-1, 1, P.n_sec())
    nP = P.sec.n_points
    pts = np.ascontiguousarray(P.sec.points.ravel())
    prod = np.zeros(3 * nP)
    P.sol.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", P.local(psi), prod)
    ring = P.orc.jtvec_xv(P.to_ring(W), P.to_ring(psi)).reshape(-1, 3)
    g = prod.reshape(-1, 3)
    # passage point -> ring point at the same position (passage 0 of the ring is the passage)
    tree = cKDTree(P.full.points)
    dist, r_of = tree.query(P.sec.points)
    assert dist.max() < 1e-12
    # coupled pairs: the points of the two cyclic patches, x_hi = R x_lo
    Rot = rotz(P.sec.sector_angle)
    side = {}
    for pch in P.sec.patches:
        if pch["type"] == "cyclic":
            fp = P.sec.faces[pch["start"]:pch["start"] + pch["size"]]
            side[pch["name"]] = np.unique(fp[fp >= 0])
    lo, hi = side["per_lo"], side["per_hi"]
    d2, j = cKDTree(P.sec.points[hi]).query(P.sec.points[lo] @ Rot.T)
    assert d2.max() < 1e-12 and lo.size == hi.size
    hi_of_lo = hi[j]
    lumped = g.copy()
    lumped[lo] = g[lo] + g[hi_of_lo] @ Rot  # R^T g_hi as rows
    keep = np.ones(nP, dtype=bool)
    keep[hi] = False
    e = rel_err(lumped[keep].ravel(), ring[r_of[keep]].ravel())
    assert e < tol, e
    # per point as well, against the largest ring value (FD accuracy)
    scale = np.abs(ring).max()
    assert np.abs(lumped[keep] - ring[r_of[keep]]).max() < 10 * tol * scale
    # a periodic displacement: the passage product against the ring's, divided by the number of passages
    X = P.full.points
    rr, th, z = np.hypot(X[:, 0], X[:, 1]), np.arctan2(X[:, 1], X[:, 0]), X[:, 2]
    Xs = P.sec.points
    rs, ths, zs = np.hypot(Xs[:, 0], Xs[:, 1]), np.arctan2(Xs[:, 1], Xs[:, 0]), Xs[:, 2]

    def field(r, t, zz):
        eta = (r - rs.min()) / (rs.max() - rs.min())
        zeta = (zz - zs.min()) / (zs.max() - zs.min())
        bump = np.sin(np.pi * eta) * np.sin(np.pi * zeta)
        dr = bump * (1.0 + 0.5 * np.cos(NS * t))
        dt = 0.6 * bump * np.cos(2.0 * np.pi * zeta) + 0.2 * np.sin(NS * t)
        dz = 0.5 * bump * np.sin(NS * t)
        return np.stack([dr * np.cos(t) - dt * np.sin(t), dr * np.sin(t) + dt * np.cos(t), dz], axis=1)

    v, v_ring = field(rs, ths, zs), field(rr, th, z)
    lhs, rhs = float(np.sum(g * v)), float(np.sum(ring * v_ring)) / NS
    assert abs(lhs - rhs) <= tol * abs(rhs), (lhs, rhs)
    return e


@pytest.mark.parametrize("solver,omega", [("DASimpleFoam", None), ("DATurboFoam", 300.0)])
def test_cyclic_volcoord_matches_ring_tape_host_build(solver, omega):
    run_ring_comparison(HOSTSIM, solver, omega)


@pytest.mark.gpu
@pytest.mark.parametrize("solver,omega", [("DASimpleFoam", None), ("DATurboFoam", 300.0)])
def test_cyclic_volcoord_matches_ring_tape_cuda(solver, omega):
    run_ring_comparison(None, solver, omega)


@pytest.mark.parametrize("kind", ["passage", "passageturbo"])
def test_cyclic_passage_mesh_update_and_volcoord_host_build(kind):
    run_cyclic_passage(HOSTSIM, kind)


@pytest.mark.parametrize("kind", ["passage", "passageturbo"])
def test_cyclic_passage_moved_matches_new_solver_host_build(kind):
    run_moved_case(HOSTSIM, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["passage", "passageturbo"])
def test_cyclic_passage_moved_matches_new_solver_cuda(kind):
    run_moved_case(None, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["passage", "passageturbo"])
def test_cyclic_passage_mesh_update_and_volcoord_cuda(kind):
    run_cyclic_passage(None, kind)


def _run_ranks(kind, nproc, port, extra=(), env=None):
    d = tempfile.mkdtemp(prefix="dab_vcm_")
    if kind.startswith("passage"):
        write_passage(d, kind)
    else:
        cases.write_case(d, cases.naca0012_ogrid(ni=32, nj=16, nk=2), cases.default_bcs_naca())
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % nproc, "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "mp_volcoord_worker.py"), d, kind] + list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=dict(os.environ, OMP_NUM_THREADS="1", **(env or {})), cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count(" ok: ") == nproc, r.stdout


@pytest.mark.parametrize("kind,nproc,port", [("naca", 2, 29771), ("passage", 2, 29773), ("passageaxial", 3, 29775), ("passageturbo", 4, 29777)])
def test_volcoord_several_ranks_match_one_rank(kind, nproc, port):
    """the sum over ranks of the per-rank products equals the one-rank product; a moved mesh gives the one-rank residual and force"""
    _run_ranks(kind, nproc, port)


@pytest.mark.gpu
@pytest.mark.parametrize("p2p,port", [("1", 29781), ("0", 29783)])
def test_volcoord_two_gpus_match_one_gpu(p2p, port):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run_ranks("passage", 2, port, ["cuda"], env=dict(DAB_P2P=p2p))
