"""GMRES + ILU(0) adjoint solve: psi from the engine vs a dense direct solve of the same operator
(assembled column by column through the engine's own matrix-free product)."""
import numpy as np
import pytest

from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import KSP, Mat, pyDASolvers
from tests.common import HOSTSIM, NORM_STATES

FN = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection",
             "direction": [1.0, 0.0, 0.0], "scale": 1.0}}


def adjoint_case(lib_path, ni=24, nj=12, restart=200, maxit=400):
    import tempfile
    mesh = cases.naca0012_ogrid(ni=ni, nj=nj, nk=1)
    d = tempfile.mkdtemp(prefix="dab_adj_")
    cases.write_case(d, mesh, cases.default_bcs_naca())
    opts = dict(normalizeStates=NORM_STATES, function=FN,
                adjEqnOption=dict(gmresRelTol=1e-9, gmresMaxIters=maxit, gmresRestart=restart))
    sol = pyDASolvers("DASimpleFoam -python", opts, caseDir=d, _lib_path=lib_path)
    nC = sol.getNLocalCells()
    y = np.zeros(nC)
    sol.getOFField("yWall", "scalar", y)
    W = cases.boundary_layer_state(mesh, y)
    sol.updateOFFields(W)
    return mesh, sol, W


def solve_and_check(lib_path):
    mesh, sol, W = adjoint_case(lib_path)
    n = sol.getNLocalAdjointStates()
    # the reference's call order: dFdW, dRdWTPC, KSP, solveLinearEqn (mphys_dafoam.py:433-574)
    dFdW = np.zeros(n)
    sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), dFdW)
    sol.runColoring()
    pc = Mat()
    sol.calcdRdWT(1, pc)
    ksp = KSP()
    sol.createMLRKSPMatrixFree(pc, ksp)
    psi = np.zeros(n)
    fail = sol.solveLinearEqn(ksp, dFdW, psi)
    st = ksp.stats
    assert fail == 0 and st.converged_reason == 2
    assert st.final_residual <= 1e-9 * st.initial_residual * 1.01
    # true residual through the matrix-free operator
    r = np.zeros(n)
    sol.calcdRdWTPsiAD(psi, r)
    assert np.linalg.norm(r - dFdW) <= 2e-9 * np.linalg.norm(dFdW)
    # dense direct solve of the same operator
    A = np.zeros((n, n))
    e, col = np.zeros(n), np.zeros(n)
    for i in range(n):
        e[:] = 0.0
        e[i] = 1.0
        sol.calcdRdWTPsiAD(e, col)
        A[:, i] = col
    psi_d = np.linalg.solve(A, dFdW)
    assert np.linalg.norm(psi - psi_d) <= 1e-5 * np.linalg.norm(psi_d)
    return st.iterations


def test_adjoint_solve_host_build():
    its = solve_and_check(HOSTSIM)
    assert 0 < its < 400


def test_failure_flag_follows_the_reference_rule():
    mesh, sol, W = adjoint_case(HOSTSIM, maxit=3, restart=3)
    n = sol.getNLocalAdjointStates()
    dFdW = np.zeros(n)
    sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), dFdW)
    pc = Mat()
    sol.calcdRdWT(1, pc)
    ksp = KSP()
    psi = np.zeros(n)
    # 3 iterations cannot reach 1e-9: relRatio and absRatio both exceed gmresTolDiff -> 1 (DALinearEqn.C:422-434)
    assert sol.solveLinearEqn(ksp, dFdW, psi) == 1
    assert ksp.stats.converged_reason == -3 and ksp.stats.iterations == 3


def test_two_level_preconditioner_reduces_iterations():
    its = {}
    for nagg in (0, 24):
        mesh, sol, W = adjoint_case(HOSTSIM, ni=48, nj=24)
        sol.updateDAOption(dict(adjEqnOption=dict(coarseAggregates=nagg, gmresRelTol=1e-8, gmresMaxIters=900, gmresRestart=150)))
        n = sol.getNLocalAdjointStates()
        b = np.zeros(n)
        sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), b)
        pc, ksp = Mat(), KSP()
        sol.calcdRdWT(1, pc)
        psi = np.zeros(n)
        assert sol.solveLinearEqn(ksp, b, psi) == 0
        r = np.zeros(n)
        sol.calcdRdWTPsiAD(psi, r)
        assert np.linalg.norm(r - b) <= 1e-7 * np.linalg.norm(b)
        its[nagg] = ksp.stats.iterations
    assert its[24] < its[0], its  # the gain grows with mesh size


@pytest.mark.gpu
def test_adjoint_solve_cuda():
    its = solve_and_check(None)
    assert 0 < its < 400


def idrs_check(lib_path):
    """adjEqnOption.kspType idrs (extension): IDR(s) with the same preconditioner, tolerance rule and statistics reaches the solution
    of the dense direct solve; switching back to gmres in the same solver object still works; the iteration cap sets the fail flag."""
    mesh, sol, W = adjoint_case(lib_path)
    n = sol.getNLocalAdjointStates()
    dFdW = np.zeros(n)
    sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), dFdW)
    pc, ksp = Mat(), KSP()
    sol.calcdRdWT(1, pc)
    sol.createMLRKSPMatrixFree(pc, ksp)
    psis, its = {}, {}
    for name, extra in (("gmres", dict(kspType="gmres")), ("idrs4", dict(kspType="idrs", idrS=4)), ("idrs1", dict(kspType="idrs", idrS=1)),
                        ("gmres2", dict(kspType="gmres"))):
        sol.updateDAOption(dict(adjEqnOption=dict(gmresRelTol=1e-9, gmresMaxIters=1500, gmresRestart=200, **extra)))
        psi = np.zeros(n)
        assert sol.solveLinearEqn(ksp, dFdW, psi) == 0, name
        st = ksp.stats
        assert st.converged_reason == 2 and st.final_residual <= 1e-9 * st.initial_residual * 1.01, name
        r = np.zeros(n)
        sol.calcdRdWTPsiAD(psi, r)
        assert np.linalg.norm(r - dFdW) <= 2e-9 * np.linalg.norm(dFdW), name
        psis[name], its[name] = psi, st.iterations
    assert np.array_equal(psis["gmres"], psis["gmres2"])
    for name in ("idrs4", "idrs1"):
        assert np.linalg.norm(psis[name] - psis["gmres"]) <= 1e-6 * np.linalg.norm(psis["gmres"]), name
    assert its["idrs4"] < 3 * its["gmres"], its  # short recurrences cost some operator applications, not multiples
    sol.updateDAOption(dict(adjEqnOption=dict(kspType="idrs", idrS=4, gmresMaxIters=5)))
    psi = np.zeros(n)
    assert sol.solveLinearEqn(ksp, dFdW, psi) == 1 and ksp.stats.converged_reason == -3 and ksp.stats.iterations == 5
    with pytest.raises(Exception, match="kspType"):
        sol.updateDAOption(dict(adjEqnOption=dict(kspType="cg")))


def test_idrs_host_build():
    idrs_check(HOSTSIM)


@pytest.mark.gpu
def test_idrs_cuda():
    idrs_check(None)


def test_coloured_probing_gives_the_same_coarse_operator(capfd):
    """The coarse Galerkin operator probed with a few coloured products (coarseProbeReach, default 6) is the one probed with one
    product per aggregate: same GMRES history, same solution; a reach that is too short is detected and falls back."""
    out = {}
    for reach in (0, 6, 1):
        mesh, sol, W = adjoint_case(HOSTSIM, ni=96, nj=48)
        sol.updateDAOption(dict(adjEqnOption=dict(coarseAggregates=100, coarseProbeReach=reach, gmresRelTol=1e-8, gmresMaxIters=900, gmresRestart=300, printInfo=1)))
        n = sol.getNLocalAdjointStates()
        b = np.zeros(n)
        sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), b)
        pc, ksp = Mat(), KSP()
        sol.calcdRdWT(1, pc)
        psi = np.zeros(n)
        assert sol.solveLinearEqn(ksp, b, psi) == 0
        out[reach] = (psi, ksp.stats.iterations, capfd.readouterr().err)
    import re
    for reach in (6, 1):
        assert out[reach][1] == out[0][1], {k: v[1] for k, v in out.items()}
        assert np.linalg.norm(out[reach][0] - out[0][0]) <= 1e-9 * np.linalg.norm(out[0][0])
    m = re.search(r"coarse space: (\d+) aggregates probed with (\d+) coloured products", out[6][2])
    assert m and int(m.group(1)) >= 100 and int(m.group(2)) < int(m.group(1)) // 2, out[6][2][-400:]
    assert "too short, falling back" in out[1][2] and "coloured products" not in out[0][2]


def test_host_threads_do_not_change_the_result():
    """The host-threaded set-up (pattern rows, coarse LU and inverse: DAB_HOST_THREADS) gives the same preconditioner whatever the thread
    count: identical GMRES history and solution bits with 1 and 4 threads (child processes: the count is read once)."""
    import os
    import subprocess
    import sys
    code = r'''
import numpy as np, tempfile
from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import pyDASolvers, Mat, KSP
from tests.common import HOSTSIM, NORM_STATES
mesh = cases.naca0012_ogrid(ni=128, nj=64, nk=1)
d = tempfile.mkdtemp(); cases.write_case(d, mesh, cases.default_bcs_naca(), binary=True)
fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection", "direction": [1.0, 0.0, 0.0], "scale": 1.0}}
sol = pyDASolvers("DASimpleFoam -python", dict(normalizeStates=NORM_STATES, function=fn,
      adjEqnOption=dict(gmresRelTol=1e-8, gmresMaxIters=900, gmresRestart=300, coarseAggregates=520, pcConLevel=2)), caseDir=d, _lib_path=HOSTSIM)
y = np.zeros(sol.getNLocalCells()); sol.getOFField("yWall", "scalar", y)
W = cases.boundary_layer_state(mesh, y); sol.updateOFFields(W)
n = sol.getNLocalAdjointStates(); b = np.zeros(n)
sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), b)
pc, ksp = Mat(), KSP(); sol.calcdRdWT(1, pc)
psi = np.zeros(n); f = sol.solveLinearEqn(ksp, b, psi)
print("RESULT", f, ksp.stats.iterations, float(np.abs(psi).sum()).hex())
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = []
    for nt in ("1", "4"):
        r = subprocess.run([sys.executable, "-c", code], cwd=root, env=dict(os.environ, DAB_HOST_THREADS=nt, PYTHONPATH=root),
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        out.append(r.stdout.strip().split("RESULT")[-1].split())
    assert out[0][0] == "0" and out[0] == out[1], out


def test_fixed_point_adjoint_host_build():
    """runFPAdj / solveAdjointFP: the stationary iteration reaches the Krylov solution on a small case and follows the reference's
    termination rule (strict, relaxed, failed)."""
    mesh, sol, W = adjoint_case(HOSTSIM)
    n = sol.getNLocalAdjointStates()
    dFdW = np.zeros(n)
    sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), dFdW)
    sol.updateDAOption(dict(adjEqnOption=dict(gmresRelTol=1e-10, gmresMaxIters=800, gmresRestart=400)))
    pc, ksp = Mat(), KSP()
    sol.calcdRdWT(1, pc)
    sol.createMLRKSPMatrixFree(pc, ksp)
    psi_k = np.zeros(n)
    assert sol.solveLinearEqn(ksp, dFdW, psi_k) == 0
    sol.updateDAOption(dict(adjEqnOption=dict(fpMaxIters=3000, fpRelTol=1e-7, fpMinResTolDiff=1e2)))
    psi = np.full(n, 7.0)  # the reference starts from zero whatever psi holds
    assert sol.runFPAdj(dFdW, psi) == 0
    its = sol.fpStats.iterations
    assert 1 < its < 3000 and np.linalg.norm(psi - psi_k) <= 1e-4 * np.linalg.norm(psi_k), (its, np.linalg.norm(psi - psi_k) / np.linalg.norm(psi_k))
    # too few sweeps for the strict tolerance, enough for the relaxed one -> still 0; far too few -> 1
    sol.updateDAOption(dict(adjEqnOption=dict(fpMaxIters=max(3, its // 2), fpRelTol=1e-7, fpMinResTolDiff=1e6)))
    assert sol.solveAdjointFP(dFdW, psi) == 0 and sol.fpStats.iterations == max(3, its // 2)
    sol.updateDAOption(dict(adjEqnOption=dict(fpMaxIters=3, fpRelTol=1e-7, fpMinResTolDiff=1e1)))
    assert sol.runFPAdj(dFdW, psi) == 1


def test_pydafoam_adjoint_method_switch():
    """PYDAFOAM.solveAdjoint follows adjEqnSolMethod like DAFoamSolver.solve_linear (reference mphys_dafoam.py:450-562)."""
    import tempfile
    from dafoam_b200.pyDAFoam import PYDAFOAM
    mesh = cases.naca0012_ogrid(ni=24, nj=12, nk=1)
    d = tempfile.mkdtemp(prefix="dab_pyd_")
    cases.write_case(d, mesh, cases.default_bcs_naca())
    opts = dict(solverName="DASimpleFoam", normalizeStates=NORM_STATES, function=FN,
                adjEqnOption=dict(gmresRelTol=1e-9, gmresMaxIters=600, gmresRestart=300, fpMaxIters=4000, fpRelTol=1e-7))
    DASolver = PYDAFOAM(options=opts, caseDir=d, _lib_path=HOSTSIM)
    y = np.zeros(DASolver.solver.getNLocalCells())
    DASolver.solver.getOFField("yWall", "scalar", y)
    DASolver.setStates(cases.boundary_layer_state(mesh, y))
    psi_k = DASolver.solveAdjoint("CD").copy()
    assert DASolver.adjointFail == 0
    DASolver.setOption("adjEqnSolMethod", "fixedPoint")
    psi_f = DASolver.solveAdjoint("CD")
    assert DASolver.adjointFail == 0 and np.linalg.norm(psi_f - psi_k) <= 1e-4 * np.linalg.norm(psi_k)
    DASolver.setOption("adjEqnSolMethod", "cg")
    with pytest.raises(RuntimeError, match="adjEqnSolMethod"):
        DASolver.solveAdjoint("CD")


def test_pydafoam_pc_lag_counts_derivative_iterations():
    """adjPCLag as in DAFoamSolver.solve_linear (reference mphys_dafoam.py:481-514): the counter advances with the first adjoint after
    a new primal solution; primal solutions without derivatives (line searches) and further functions of the same iteration do not
    age the preconditioner."""
    import tempfile
    from dafoam_b200.pyDAFoam import PYDAFOAM
    mesh = cases.naca0012_ogrid(ni=24, nj=12, nk=1)
    d = tempfile.mkdtemp(prefix="dab_pyd_")
    cases.write_case(d, mesh, cases.default_bcs_naca())
    fn = dict(FN, CL=dict(FN["CD"], direction=[0.0, 1.0, 0.0]))
    opts = dict(solverName="DASimpleFoam", normalizeStates=NORM_STATES, function=fn, adjPCLag=2, primalMaxIters=5,
                adjEqnOption=dict(gmresRelTol=1e-6, gmresMaxIters=600, gmresRestart=300))
    DASolver = PYDAFOAM(options=opts, caseDir=d, _lib_path=HOSTSIM)
    y = np.zeros(DASolver.solver.getNLocalCells())
    DASolver.solver.getOFField("yWall", "scalar", y)
    DASolver.setStates(cases.boundary_layer_state(mesh, y))
    DASolver.solveAdjoint("CD")          # iteration 1: nothing assembled yet -> assembly 1
    DASolver.solveAdjoint("CL")          # same iteration, second function: kept
    assert DASolver.nPCAssemblies == 1 and DASolver.solution_counter == 2
    DASolver()
    DASolver()                           # a line-search primal: no derivatives asked for
    DASolver.solveAdjoint("CD")          # iteration 2: (3 - 1) % 2 == 0 -> assembly 2
    assert DASolver.nPCAssemblies == 2 and DASolver.solution_counter == 3
    DASolver()
    DASolver.solveAdjoint("CD")          # iteration 3: (4 - 1) % 2 != 0 -> kept
    DASolver.solveAdjoint("CL")
    assert DASolver.nPCAssemblies == 2 and DASolver.solution_counter == 4 and DASolver.adjointFail == 0


def _solve_with(sol, W, extra):
    n = sol.getNLocalAdjointStates()
    sol.updateDAOption(dict(adjEqnOption=dict(gmresRelTol=1e-9, gmresMaxIters=600, gmresRestart=300, **extra)))
    dFdW = np.zeros(n)
    sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), dFdW)
    pc, ksp = Mat(), KSP()
    sol.calcdRdWT(1, pc)
    sol.createMLRKSPMatrixFree(pc, ksp)
    psi = np.zeros(n)
    fail = sol.solveLinearEqn(ksp, dFdW, psi)
    r = np.zeros(n)
    sol.calcdRdWTPsiAD(psi, r)
    assert fail == 0 and np.linalg.norm(r - dFdW) <= 2e-9 * np.linalg.norm(dFdW)
    return psi, ksp.stats.iterations


def test_preconditioner_variants_reach_the_same_adjoint():
    """Ordering / storage variants of the preconditioner (adjEqnOption.pcBlockCells: block-Jacobi ILU(0) with the natural cell order
    inside blocks, level-scheduled -- the reference's PCASM overlap 0 + natural-order PCILU; adjEqnOption.pcStorage fp32: fp32 copy
    of the factors) change the iteration count, never the converged adjoint."""
    mesh, sol, W = adjoint_case(HOSTSIM, ni=32, nj=16)
    psi0, it0 = _solve_with(sol, W, dict(pcBlockCells=0, pcStorage="fp64"))
    for extra in (dict(pcBlockCells=64, pcStorage="fp64"), dict(pcBlockCells=0, pcStorage="fp32"), dict(pcBlockCells=128, pcStorage="fp32")):
        psi, it = _solve_with(sol, W, extra)
        assert np.linalg.norm(psi - psi0) <= 1e-6 * np.linalg.norm(psi0), extra
        assert it < 600
    with pytest.raises(Exception):
        sol.updateDAOption(dict(adjEqnOption=dict(pcStorage="fp16")))
    # adjEqnOption.pcPattern "stateInfo": the reference's per-(residual, state) connectivity levels (DAStateInfoSimpleFoam.C:75-99,
    # DASpalartAllmaras.C:364-373, capped by maxResConLv4JacPCMat) -- a sparser matrix, the same adjoint
    pc = Mat()
    sol.updateDAOption(dict(adjEqnOption=dict(pcBlockCells=0, pcStorage="fp64", pcPattern="uniform", pcConLevel=3)))
    sol.calcdRdWT(1, pc)
    nnz_uniform = sol.getPCMatrixSize()[1]
    psi, it = _solve_with(sol, W, dict(pcBlockCells=0, pcStorage="fp64", pcPattern="stateInfo", pcConLevel=3))
    assert np.linalg.norm(psi - psi0) <= 1e-6 * np.linalg.norm(psi0) and it < 600
    sol.calcdRdWT(1, pc)
    assert sol.getPCMatrixSize()[1] < 0.8 * nnz_uniform, (sol.getPCMatrixSize(), nnz_uniform)
    sol.updateDAOption(dict(adjEqnOption=dict(pcPattern="uniform", pcConLevel=2)))
    with pytest.raises(Exception):
        sol.updateDAOption(dict(adjEqnOption=dict(pcPattern="dense")))


def test_fixed_point_then_gmres_on_the_same_handle():
    """ADVICE round 1: runFPAdj re-initialised the dot-product workspace to 34 vectors; a later GMRES with more than 34 iterations on
    the same handle then wrote past it.  The workspace now only grows."""
    mesh, sol, W = adjoint_case(HOSTSIM, ni=32, nj=16, restart=300, maxit=600)
    n = sol.getNLocalAdjointStates()
    dFdW = np.zeros(n)
    sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), dFdW)
    psi_fp = np.zeros(n)
    sol.updateDAOption(dict(adjEqnOption=dict(fpMaxIters=5)))
    sol.runFPAdj(dFdW, psi_fp)  # not expected to converge in 5 sweeps: only its workspace matters here
    sol.updateDAOption(dict(adjEqnOption=dict(gmresRelTol=1e-9, gmresMaxIters=600, gmresRestart=300)))
    pc, ksp = Mat(), KSP()
    sol.calcdRdWT(1, pc)
    sol.createMLRKSPMatrixFree(pc, ksp)
    psi = np.zeros(n)
    fail = sol.solveLinearEqn(ksp, dFdW, psi)
    assert fail == 0 and ksp.stats.iterations > 40
    r = np.zeros(n)
    sol.calcdRdWTPsiAD(psi, r)
    assert np.linalg.norm(r - dFdW) <= 2e-9 * np.linalg.norm(dFdW)


def test_sparse_coarse_columns_equal_the_matrix_free_product():
    """adjEqnOption.coarseSparseAP: the multiplicative two-level step t = v - A P yc through the columns A (P e_a) kept from the probing
    of the coarse operator (a short sparse product) gives the same preconditioner as the matrix-free product it replaces: same GMRES
    history, same adjoint; coloured probing (> 64 aggregates) and one-product-per-aggregate probing."""
    for nagg in (100, 12):
        mesh, sol, W = adjoint_case(HOSTSIM, ni=48, nj=24, restart=300, maxit=600)
        res = {}
        for sparse in (1, 0):
            psi, it = _solve_with(sol, W, dict(coarseAggregates=nagg, coarseSparseAP=sparse))
            res[sparse] = (psi, it)
        assert res[1][1] == res[0][1], (nagg, res[1][1], res[0][1])
        assert np.linalg.norm(res[1][0] - res[0][0]) <= 1e-9 * np.linalg.norm(res[0][0])
