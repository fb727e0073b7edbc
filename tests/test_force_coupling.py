"""forceCouplingOutput (reference DAOutputForceCoupling.C): the nodal wall forces handed to the load transfer of an aerostructural
run, and their transpose products w.r.t. the states and the mesh points.  The layout and the split of each face force over its
points are restated here in numpy (patches sorted by name, np.unique per patch as pyDAFoam.getSurfaceCoordinates does); the face
forces and their tapes come from the oracle's residual work arrays (tests/coupling_oracle.cpp), whose face arithmetic is checked
against the oracle's own force function first."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import DAB200Error, KSP, Mat
from tests.common import HOSTSIM, ROOT, rel_err, setup
from tests.coupling_oracle import face_forces, face_forces_jtvec

FC = "forceCouplingOutput"


def outputs(patches, pRef):
    return {"f_aero": {"type": FC, "patches": list(patches), "pRef": pRef, "components": ["forceCoupling"]},
            "f_gauge0": {"type": FC, "patches": list(patches), "pRef": 0.0, "components": ["forceCoupling"]}}


def force_functions(patches):
    return {"F%d" % k: {"type": "force", "source": "patchToFace", "patches": list(patches), "directionMode": "fixedDirection",
                        "direction": [float(k == 0), float(k == 1), float(k == 2)], "scale": 1.0} for k in range(3)}


def layout(mesh, patches):
    """(node labels, [(boundary face, node slots)] in output face order) of an output on `patches`"""
    nIF, nodes, rows = mesh.n_internal_faces, [], []
    for name in sorted(patches):
        p = next(q for q in mesh.patches if q["name"] == name)
        fp = mesh.faces[p["start"]:p["start"] + p["size"]]
        lab = np.unique(fp[fp >= 0])
        base = len(nodes)
        for i in range(p["size"]):
            v = fp[i][fp[i] >= 0]
            rows.append((p["start"] + i - nIF, base + np.searchsorted(lab, v)))
        nodes.extend(lab.tolist())
    return np.array(nodes, dtype=np.int64), rows


def node_split(Ff, rows, nN):
    """each face force split equally over the face's points, added in face order"""
    out = np.zeros((nN, 3))
    for b, sl in rows:
        out[sl] += Ff[b] / len(sl)
    return out.ravel()


def face_seeds(seed, rows, nBF):
    """the transpose of node_split: d_b = sum of the node seeds of face b / nPoints_b"""
    s, d = seed.reshape(-1, 3), np.zeros((nBF, 3))
    for b, sl in rows:
        d[b] = s[sl].sum(axis=0) / len(sl)
    return d


def patch_ids(mesh, patches):
    names = [p["name"] for p in mesh.patches]
    return [names.index(n) for n in patches]


def wall_area_vector(orc, mesh, patches):
    Sf = orc.geometry("Sf").reshape(-1, 3)
    return sum(Sf[p["start"]:p["start"] + p["size"]].sum(axis=0) for p in mesh.patches if p["name"] in patches)


# ---- 0. the reference face forces ------------------------------------------------------------------------------------
def test_reference_face_forces_match_the_oracle_force_function():
    """tests/coupling_oracle.cpp restates the face loop of the oracle's forceFunction: per patch and axis, the sum of its face
    forces is orc.force, and the tape of a uniform per-face direction is orc.dforce_dw (incompressible with the Spalding wall
    function, compressible, DATurboFoam + MRF)."""
    from tests.test_compressible import CONFIGS, setup_comp
    from tests.test_mrf import setup_mrf
    _, _, orc_i, _, W_i, _ = setup("nacawf", True, "linearUpwindV", 1, lib_path=HOSTSIM)
    _, orc_c, _, W_c = setup_comp(CONFIGS[0], HOSTSIM)
    _, orc_t, _, W_t = setup_mrf("DATurboFoam", HOSTSIM)
    for orc, W in ((orc_i, W_i), (orc_c, W_c), (orc_t, W_t)):
        mesh = orc.mesh
        nBF = mesh.n_faces - mesh.n_internal_faces
        for name in ("wing", "sym1"):
            pid = patch_ids(mesh, [name])[0]
            p = mesh.patches[pid]
            Ff = face_forces(orc, W, [pid])
            on = np.zeros(nBF, dtype=bool)
            on[p["start"] - mesh.n_internal_faces:p["start"] - mesh.n_internal_faces + p["size"]] = True
            assert np.all(Ff[~on] == 0.0)
            for k in range(3):
                e = np.eye(3)[k]
                F, Fo = Ff[:, k].sum(), orc.force(W, pid, e, 1.0)
                assert abs(F - Fo) <= 1e-13 * np.abs(Ff[:, k]).sum(), (name, k, F, Fo)
                g = face_forces_jtvec(orc, W, [pid], np.outer(on, e))
                assert rel_err(g, orc.dforce_dw(W, pid, e, 1.0)) < 1e-13, (name, k)
        # pRef enters as Sf (p_b - pRef)
        pid = patch_ids(mesh, ["wing"])[0]
        Sf = orc.geometry("Sf").reshape(-1, 3)[mesh.n_internal_faces:]
        d = face_forces(orc, W, [pid], 2.5) - face_forces(orc, W, [pid])
        on = np.abs(face_forces(orc, W, [pid])).sum(axis=1) > 0
        assert np.allclose(d[on], -2.5 * Sf[on], rtol=1e-9, atol=1e-9 * np.abs(Sf).max())


# ---- 1. layout --------------------------------------------------------------------------------------------------------
def check_layout(lib_path):
    patches = ["wing", "sym1"]  # listed out of order; they share the trailing points of the wing's lower layer
    mesh, bcs, orc, sol, W, _ = setup("naca", True, nk=2, lib_path=lib_path, extra_options=dict(outputInfo=outputs(patches, 0.5)))
    nodes, rows = layout(mesh, patches)
    assert len(nodes) > len(np.unique(nodes))  # the shared points appear once per patch
    assert sol.getOutputSize("f_aero", FC) == 3 * len(nodes)
    assert np.array_equal(sol.getForceCouplingPoints("f_aero"), nodes)
    assert sol.getOutputDistributed("f_aero", FC) == 1


def test_force_coupling_layout_host_build():
    check_layout(HOSTSIM)


@pytest.mark.gpu
def test_force_coupling_layout_cuda():
    check_layout(None)


# ---- 2. value and 3. state product ------------------------------------------------------------------------------------
def comp_case(lib_path, extra):
    from tests.test_compressible import CONFIGS, NS, setup_comp
    mesh, orc, sol, W = setup_comp(CONFIGS[0], lib_path)  # DARhoSimpleFoam, linearUpwindV
    sol.updateDAOption(dict(normalizeStates=NS, normalizeResiduals=list(CONFIGS[0][7]), **extra))
    return mesh, orc, sol, W


def turbo_case(lib_path, extra):
    from tests.test_mrf import setup_mrf
    mesh, orc, sol, W = setup_mrf("DATurboFoam", lib_path, function=extra["function"])  # the wing rotates with the zone
    sol.updateDAOption(dict(outputInfo=extra["outputInfo"]))
    return mesh, orc, sol, W


def value_cases(lib_path):
    """(label, mesh, orc, sol, W, patches, pRef) for every solver family and wall treatment"""
    for label in ("DASimpleFoam SA linearUpwindV", "Spalding wall function", "DARhoSimpleFoam", "DATurboFoam MRF"):
        patches = ["wing", "sym1"] if label != "DATurboFoam MRF" else ["wing"]
        pRef = 0.7 if label.startswith("DASimple") or label.startswith("Spalding") else 101325.0
        extra = dict(outputInfo=outputs(patches, pRef), function=force_functions(patches))
        if label.startswith("DASimpleFoam"):
            mesh, bcs, orc, sol, W, _ = setup("naca", True, "linearUpwindV", 2, lib_path=lib_path, extra_options=extra)
        elif label.startswith("Spalding"):
            mesh, bcs, orc, sol, W, _ = setup("nacawf", True, "linearUpwindV", 1, lib_path=lib_path, extra_options=extra)
        elif label == "DARhoSimpleFoam":
            mesh, orc, sol, W = comp_case(lib_path, extra)
        else:
            mesh, orc, sol, W = turbo_case(lib_path, extra)
        yield label, mesh, orc, sol, W, patches, pRef


def check_value_and_state_product(lib_path, tol):
    rng = np.random.default_rng(17)
    for label, mesh, orc, sol, W, patches, pRef in value_cases(lib_path):
        sol.updateOFFields(W)
        nodes, rows = layout(mesh, patches)
        nBF = mesh.n_faces - mesh.n_internal_faces
        pid = patch_ids(mesh, patches)
        n3 = sol.getOutputSize("f_aero", FC)
        f, f2, f0 = np.zeros(n3), np.zeros(n3), np.zeros(n3)
        sol.calcOutput("f_aero", FC, f)
        ref = node_split(face_forces(orc, W, pid, pRef), rows, len(nodes))
        assert np.linalg.norm(ref) > 0
        assert rel_err(f, ref) < tol, (label, rel_err(f, ref))
        sol.calcOutput("f_aero", FC, f2)
        assert np.array_equal(f, f2), label  # deterministic: no atomics
        # with pRef = 0 the node sums are the force functions along the axes; pRef shifts them by -pRef * sum(Sf)
        sol.calcOutput("f_gauge0", FC, f0)
        tot0, scale = f0.reshape(-1, 3).sum(axis=0), np.abs(f0).sum()
        for k in range(3):
            Fk = sol.calcFunction("F%d" % k)
            assert abs(tot0[k] - Fk) <= 1e-12 * scale, (label, k, tot0[k], Fk)
        shift = (f - f0).reshape(-1, 3).sum(axis=0)
        S = wall_area_vector(orc, mesh, patches)
        assert np.all(np.abs(shift + pRef * S) <= 1e-12 * (abs(pRef) * np.abs(orc.geometry("Sf")).sum() + scale)), (label, shift, -pRef * S)
        # [d(s . f)/dW]^T for random node seeds against the oracle's tape of sum_f d_f . F_f
        seed = rng.uniform(-1, 1, n3)
        prod = np.zeros(orc.ndof)
        sol.calcJacTVecProduct("states", "stateVar", W, "f_aero", FC, seed, prod)
        pref = face_forces_jtvec(orc, W, pid, face_seeds(seed, rows, nBF), "states", pRef)
        assert np.linalg.norm(pref) > 0
        assert rel_err(prod, pref) < tol, (label, rel_err(prod, pref))
        print("%-30s value %.1e, state product %.1e" % (label, rel_err(f, ref), rel_err(prod, pref)))


def test_force_coupling_value_and_state_product_host_build():
    check_value_and_state_product(HOSTSIM, 1e-12)


@pytest.mark.gpu
def test_force_coupling_value_and_state_product_cuda():
    check_value_and_state_product(None, 1e-10)


# ---- 4. mesh product --------------------------------------------------------------------------------------------------
def check_mesh_product(lib_path):
    patches, pRef = ["wing", "sym1"], 0.7
    mesh, bcs, orc, sol, W, _ = setup("naca", True, "linearUpwind", 1, lib_path=lib_path, extra_options=dict(outputInfo=outputs(patches, pRef)))
    sol.updateOFFields(W)
    nodes, rows = layout(mesh, patches)
    nBF = mesh.n_faces - mesh.n_internal_faces
    nP3 = 3 * sol.getNLocalPoints()
    pts = np.zeros(nP3)
    sol.getOFMeshPoints(pts)
    seed = np.random.default_rng(23).uniform(-1, 1, sol.getOutputSize("f_aero", FC))
    prod = np.zeros(nP3)
    sol.calcJacTVecProduct("aero_vol_coords", "volCoord", pts, "f_aero", FC, seed, prod)
    ref = face_forces_jtvec(orc, W, patch_ids(mesh, patches), face_seeds(seed, rows, nBF), "points", pRef)
    # Points on a symmetry plane: the derivative along the plane normal differentiates |n_k| of the symmetry transform at n_k = 0,
    # a kink where the tape takes the one-sided convention and central differences the symmetric value (tests/test_volcoord.py).
    # Symmetry-plane points move in the plane in practice; every other component must agree.
    mask = np.ones((nP3 // 3, 3), dtype=bool)
    for pch in mesh.patches:
        if pch["type"] == "symmetry":
            fp = mesh.faces[pch["start"]:pch["start"] + pch["size"]]
            mask[np.unique(fp[fp >= 0]), 2] = False
    mask = mask.ravel()
    err = rel_err(prod[mask], ref[mask])
    assert err < 1e-7, err
    # directional central difference through updateOFMesh
    X = pts.reshape(-1, 3)
    v = np.stack([np.sin(3.0 * X[:, 1]) * 1e-3, np.cos(2.0 * X[:, 0]) * 1e-3, np.zeros(len(X))], axis=1).ravel()
    h = 1e-3
    fp_, fm_ = np.zeros(len(seed)), np.zeros(len(seed))
    sol.updateOFMesh(pts + h * v)
    sol.calcOutput("f_aero", FC, fp_)
    sol.updateOFMesh(pts - h * v)
    sol.calcOutput("f_aero", FC, fm_)
    sol.updateOFMesh(pts)
    fd = seed @ (fp_ - fm_) / (2 * h)
    assert abs(fd - prod @ v) <= 1e-5 * abs(fd), (fd, prod @ v)
    # the unperturbed geometry is restored: the output is bitwise what it was
    f1, f2 = np.zeros(len(seed)), np.zeros(len(seed))
    sol.calcOutput("f_aero", FC, f1)
    sol.updateOFFields(W)
    sol.calcOutput("f_aero", FC, f2)
    assert np.array_equal(f1, f2)


def test_force_coupling_mesh_product_host_build():
    check_mesh_product(HOSTSIM)


@pytest.mark.gpu
def test_force_coupling_mesh_product_cuda():
    check_mesh_product(None)


# ---- 5. adjoint use ---------------------------------------------------------------------------------------------------
def check_adjoint_shape_derivative(lib_path):
    """d(s . f_aero)/d(alpha) of a mesh deformation x0 + alpha v: the adjoint total derivative ds.f/dx . v - psi^T dR/dx . v against
    central differences over deformed meshes with re-converged primals (tests/test_primal.py's bar)."""
    from tests.test_primal import make
    mesh, bcs, sol = make(lib_path)
    sol.updateDAOption(dict(outputInfo=outputs(["walls"], 0.3)))
    n, nP3 = sol.getNLocalAdjointStates(), 3 * sol.getNLocalPoints()
    x0 = np.zeros(nP3)
    sol.getOFMeshPoints(x0)
    X = x0.reshape(-1, 3)
    s_ = (X[:, 0] - X[:, 0].min()) / np.ptp(X[:, 0])
    t_ = (X[:, 1] - X[:, 1].min()) / np.ptp(X[:, 1])
    v = np.zeros_like(X)
    v[:, 1] = 0.05 * np.ptp(X[:, 1]) * np.sin(np.pi * s_) ** 2 * (1.0 - t_)
    v = v.ravel()
    n3 = sol.getOutputSize("f_aero", FC)
    seed = np.random.default_rng(29).uniform(-1, 1, n3)

    def sf_at(alpha):
        sol.updateOFMesh(x0 + alpha * v)
        assert sol.solvePrimal() == 0
        f = np.zeros(n3)
        sol.calcOutput("f_aero", FC, f)
        return seed @ f

    sf_at(0.0)
    W = np.zeros(n)
    sol.getOFFields(W)
    dFdW, psi, dFdx, dRdxTpsi = np.zeros(n), np.zeros(n), np.zeros(nP3), np.zeros(nP3)
    sol.calcJacTVecProduct("states", "stateVar", W, "f_aero", FC, seed, dFdW)
    pc, ksp = Mat(), KSP()
    sol.calcdRdWT(1, pc)
    sol.createMLRKSPMatrixFree(pc, ksp)
    assert sol.solveLinearEqn(ksp, dFdW, psi) == 0
    sol.calcJacTVecProduct("aero_vol_coords", "volCoord", x0, "f_aero", FC, seed, dFdx)
    sol.calcJacTVecProduct("aero_vol_coords", "volCoord", x0, "R", "residual", psi, dRdxTpsi)
    total = (dFdx - dRdxTpsi) @ v
    h = 1e-3
    fd = (sf_at(h) - sf_at(-h)) / (2 * h)
    sol.updateOFMesh(x0)
    assert abs(fd) > 0 and abs(total - fd) <= 2e-5 * abs(fd), (total, fd)


def test_force_coupling_adjoint_shape_derivative_host_build():
    check_adjoint_shape_derivative(HOSTSIM)


@pytest.mark.gpu
def test_force_coupling_adjoint_shape_derivative_cuda():
    check_adjoint_shape_derivative(None)


# ---- 6. several ranks -------------------------------------------------------------------------------------------------
def _run_ranks(kind, nproc, port, extra=()):
    from tests.test_volcoord_partitioned import write_passage
    d = tempfile.mkdtemp(prefix="dab_fcm_")
    if kind == "passageturbo":
        write_passage(d, kind)
    else:
        cases.write_case(d, cases.naca0012_ogrid(ni=32, nj=16, nk=2), cases.default_bcs_naca())
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % nproc, "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "mp_coupling_worker.py"), d, kind] + list(extra)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=dict(os.environ, OMP_NUM_THREADS="1"), cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count(" ok: ") == nproc, r.stdout


@pytest.mark.parametrize("kind,port", [("naca", 29791), ("passageturbo", 29793)])
def test_force_coupling_two_ranks_match_one_rank(kind, port):
    _run_ranks(kind, 2, port)


@pytest.mark.gpu
def test_force_coupling_two_gpus_match_one_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run_ranks("passageturbo", 2, 29795, ["cuda"])


# ---- 7. errors --------------------------------------------------------------------------------------------------------
def check_errors(lib_path):
    mesh, bcs, orc, sol, W, _ = setup("naca", True, nk=1, lib_path=lib_path,
                                      extra_options=dict(outputInfo=outputs(["wing"], 0.0),
                                                         inputInfo={"patchV": {"type": "patchVelocity", "patches": ["inout"],
                                                                               "flowAxis": "x", "normalAxis": "y"}}))
    with pytest.raises(DAB200Error, match="pRef"):
        sol.updateDAOption(dict(outputInfo={"f": {"type": FC, "patches": ["wing"]}}))
    with pytest.raises(DAB200Error, match="unknown patch"):
        sol.updateDAOption(dict(outputInfo={"f": {"type": FC, "patches": ["flap"], "pRef": 0.0}}))
    with pytest.raises(DAB200Error, match="patches"):
        sol.updateDAOption(dict(outputInfo={"f": {"type": FC, "patches": [], "pRef": 0.0}}))
    # other output types parse, and are refused when used
    sol.updateDAOption(dict(outputInfo=dict(outputs(["wing"], 0.0), t_conduct={"type": "thermalCouplingOutput", "patches": ["wing"]})))
    with pytest.raises(DAB200Error, match="not supported"):
        sol.getOutputSize("t_conduct", FC)
    sol.updateOFFields(W)
    n3 = sol.getOutputSize("f_aero", FC)
    with pytest.raises(AssertionError, match="seed"):
        sol.calcJacTVecProduct("states", "stateVar", W, "f_aero", FC, np.zeros(n3 + 3), np.zeros(orc.ndof))
    with pytest.raises(DAB200Error, match="not supported"):
        sol.calcJacTVecProduct("patchV", "patchVelocity", np.array([10.0, 3.0]), "f_aero", FC, np.zeros(n3), np.zeros(2))


def test_force_coupling_errors_host_build():
    check_errors(HOSTSIM)


@pytest.mark.gpu
def test_force_coupling_errors_cuda():
    check_errors(None)
