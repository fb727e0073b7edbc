"""DATurboFoam's transonic SIMPLE primal (SIMPLE { transonic yes; }, reference pEqnTurbo.H transonic branch): the div(phid,p) -
laplacian(rho rAU, p) pressure equation, its BiCGStab solve and the loop whose fixed point is the root of the residual the adjoint
differentiates (DAResidualTurboFoam.C:148-189)."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from dafoam_b200 import cases
from oracle.pyoracle import Oracle
from tests.common import HOSTSIM, ROOT, rel_err, synthetic_state
from tests.test_mrf import NRES_C, NS_C, mrf_spec

SCHEMES = {"Gauss upwind": (0, 1.0), "Gauss linear": (2, 1.0), "Gauss limitedLinear 1.0": (4, 1.0)}
# relaxation factors that converge on the O-grid at Mach 0.66: fields p, equations p (pEqn.relax(); None: not relaxed), U, e|h,
# and the SIMPLE iterations they need.  Central differencing of p (linear, and limitedLinear where the limiter opens) loses the
# diagonal dominance that pEqn.relax() restores; the much larger relaxed diagonal then slows the pressure down (about 42 000
# iterations to 1e-9 instead of about 520 with upwind).  Without pEqn.relax() both diverge.
RELAX = {"Gauss upwind": (0.3, None, 0.7, 0.7, 4000), "Gauss linear": (0.5, 0.9, 0.7, 0.7, 50000),
         "Gauss limitedLinear 1.0": (0.5, 0.9, 0.7, 0.7, 50000)}
U0 = (230.0, 8.0, 0.0)  # about Mach 0.66 at 300 K


def transonic_case(energy, scheme, lib_path, function=None, inputs=None, solvers=None, omega=0.3):
    from dafoam_b200.pyDASolvers import pyDASolvers
    mesh = cases.naca0012_ogrid(ni=24, nj=12, nk=2)
    th = cases.default_thermo(energy=energy)
    bcs = cases.compressible_bcs(cases.default_bcs_naca(U0=U0))
    ns = dict(NS_C, U=float(U0[0]))
    orc = Oracle(mesh, bcs, normalizeStates=ns, normalizeResiduals=NRES_C, thermo=th, divU="linearUpwindV")
    orc.set_turbo(True)
    code, k = SCHEMES[scheme]
    orc.set_transonic(True, code, k, -1)
    W = synthetic_state(mesh, orc.geometry("C"), orc.geometry("Sf"), U0=U0, thermo=th)
    mrf = mrf_spec(mesh, orc.geometry("C").reshape(-1, 3), omega=omega)
    orc.set_mrf(mesh, mrf)
    rp, rpe, ru, rhe, its = RELAX[scheme]
    d = tempfile.mkdtemp(prefix="dab_tprimal_")
    cases.write_case(d, mesh, bcs, div_u="bounded Gauss linearUpwindV grad(U)", transonic=True, div_phid_p=scheme, thermo=th, mrf=mrf,
                     relax_p=rp, relax_p_eqn=rpe, relax_u=ru, relax_he=rhe)
    if solvers:
        with open(os.path.join(d, "system", "fvSolution"), "a") as f:
            f.write("\nsolvers\n{\n%s}\n" % solvers)
    opts = dict(normalizeStates=ns, normalizeResiduals=list(NRES_C), primalMinResTol=1e-9, primalMaxIters=its)
    if function:
        opts["function"] = function
    if inputs:
        opts["inputInfo"] = inputs
    sol = pyDASolvers("DATurboFoam -python", opts, caseDir=d, _lib_path=lib_path)
    return mesh, orc, sol, W


# ---- (a) the fixed point is the root of R ------------------------------------------------------------------------------------------
def check_fixed_point(lib_path, energy, scheme):
    mesh, orc, sol, W = transonic_case(energy, scheme, lib_path)
    n = orc.ndof
    W0 = np.zeros(n)
    sol.getOFFields(W0)
    assert sol.solvePrimal() == 0, (energy, scheme, sol.primalStats.max_residual, sol.primalStats.iterations)
    st = sol.primalStats
    assert st.converged == 1 and st.p_iterations > 0
    W1 = np.zeros(n)
    sol.getOFFields(W1)
    r0, r1 = np.linalg.norm(orc.residual(W0)), np.linalg.norm(orc.residual(W1))
    assert r1 < 1e-6 * r0, (energy, scheme, r0, r1)
    # the engine's own residual at the converged state agrees (its stored flux is the residual's F)
    R = np.zeros(n)
    sol.getResiduals(R)
    assert np.linalg.norm(R) < 1e-6 * r0
    # transonic: something is compressible here (the converged density varies by more than a few per cent)
    nC = mesh.n_cells
    rho = W1[3 * nC:4 * nC] / (287.0 * W1[4 * nC:5 * nC])
    assert rho.max() / rho.min() > 1.05


CASES_A = [(e, s) for e in ("sensibleEnthalpy", "sensibleInternalEnergy") for s in SCHEMES]
# the CUDA twin runs the upwind cases: the linear and limitedLinear ones need about 42 000 SIMPLE iterations, which the device loop
# (launch- and sync-bound on 576 cells) takes minutes for
CASES_A_CUDA = [(e, "Gauss upwind") for e in ("sensibleEnthalpy", "sensibleInternalEnergy")]


@pytest.mark.parametrize("energy,scheme", CASES_A)
def test_transonic_fixed_point_is_root_host_build(energy, scheme):
    check_fixed_point(HOSTSIM, energy, scheme)


@pytest.mark.gpu
@pytest.mark.parametrize("energy,scheme", CASES_A_CUDA)
def test_transonic_fixed_point_is_root_cuda(energy, scheme):
    check_fixed_point(None, energy, scheme)


# ---- (b) one pressure solve and the coarse inverse ---------------------------------------------------------------------------------
def ell_to_csr(P):
    nC = len(P["diag"])
    rows, cols, vals = [np.arange(nC)], [np.arange(nC)], [P["diag"]]
    for k in range(P["nbr"].shape[0]):
        m = P["nbr"][k] >= 0
        rows.append(np.nonzero(m)[0])
        cols.append(P["nbr"][k][m])
        vals.append(P["off"][k][m])
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(nC, nC))


def check_pressure_solve(lib_path):
    tol = 1e-6  # normalised (about 1e-5 of |b - A p0|): well above where BiCGStab's recursive residual stalls in round-off (p ~ 1e5)
    for scheme in ("Gauss upwind", "Gauss limitedLinear 1.0"):
        mesh, orc, sol, W = transonic_case("sensibleEnthalpy", scheme, lib_path, solvers="    p { tolerance %g; relTol 0; maxIter 5000; }\n" % tol)
        sol.updateOFFields(W)
        W0 = np.zeros(orc.ndof)
        sol.getOFFields(W0)
        rng = np.random.default_rng(3)
        for coarse in (True, False):
            P = sol.getTransonicPressureSystem(coarse=coarse, rc=rng.uniform(-1, 1, 64))
            A = ell_to_csr(P)
            # the equation is not symmetric (convection of p by phid)
            assert abs(A - A.T).max() > 1e-6 * abs(A).max()
            xs = spla.spsolve(A.tocsc(), P["b"])
            x = P["x"]
            # OpenFOAM's normalised residual of the returned solution is within the solver tolerance; the norm factor is the one of
            # the initial guess (the current p), fixed for the solve (lduMatrix::solver::normFactor)
            x0 = W0[3 * mesh.n_cells:4 * mesh.n_cells]
            rs = A @ np.ones(len(x))
            nf = np.abs(A @ x0 - x0.mean() * rs).sum() + np.abs(P["b"] - x0.mean() * rs).sum()
            # (the solver tracks the recursively updated residual: allow the round-off between it and the true one)
            assert np.abs(P["b"] - A @ x).sum() / nf <= 1.2 * tol, (scheme, coarse, np.abs(P["b"] - A @ x).sum() / nf)
            assert np.abs(P["b"] - A @ x0).sum() / nf > 1e3 * tol and P["iterations"] > 0
            # ... and it is spsolve's solution to that tolerance: A (x - xs) is within it, and x - xs itself within what cond(A) ~ 5e7 lets
            # a 1e-6 residual move p (the weakly determined level of p: only outflow faces fix it)
            assert np.abs(A @ (x - xs)).sum() / nf <= 1.2 * tol
            assert np.linalg.norm(x - xs) <= 3e-4 * np.linalg.norm(xs), (scheme, coarse, np.linalg.norm(x - xs) / np.linalg.norm(xs))
            if coarse:
                na = P["n_agg"]
                assert na > 1 and P["agg_of"].min() == 0 and P["agg_of"].max() == na - 1
                Pm = sp.csr_matrix((np.ones(len(x)), (np.arange(len(x)), P["agg_of"])), shape=(len(x), na))
                Ac = (Pm.T @ A @ Pm).toarray()
                rc = rng.uniform(-1, 1, 64)[:na]
                P2 = sol.getTransonicPressureSystem(coarse=True, rc=rc)
                ref, refT = np.linalg.solve(Ac, rc), np.linalg.solve(Ac.T, rc)
                # a check that tells Ac^-1 from Ac^-T: the two differ on this operator
                assert rel_err(refT, ref) > 1e-3
                assert rel_err(P2["yc"], ref) < 1e-9, rel_err(P2["yc"], ref)
            else:
                assert np.all(P["agg_of"] == -1)
        # the probe leaves the states as they were
        W1 = np.zeros(orc.ndof)
        sol.getOFFields(W1)
        assert np.array_equal(W0, W1)


def test_transonic_pressure_solve_host_build():
    check_pressure_solve(HOSTSIM)


@pytest.mark.gpu
def test_transonic_pressure_solve_cuda():
    check_pressure_solve(None)


# ---- (c) the cyclic passage with MRF on one and on two ranks -----------------------------------------------------------------------
def write_transonic_passage(d):
    mesh = cases.annular_passage(nr=5, nt=6, nz=8, n_sectors=7)
    bcs = cases.compressible_bcs(cases.default_bcs_passage(Uin=(0.0, 0.0, 60.0)))
    mrf = dict(cellZone="rotor", cells=list(range(mesh.n_cells)), origin=(0.0, 0.0, 0.0), axis=(0.0, 0.0, 1.0), omega=200.0,
               nonRotatingPatches=["inlet", "outlet", "shroud"])
    cases.write_case(d, mesh, bcs, thermo=cases.default_thermo(energy="sensibleEnthalpy"), mrf=mrf, transonic=True,
                     div_phid_p="Gauss limitedLinear 1.0", relax_p=0.3, relax_p_eqn=1.0)
    return mesh


def check_passage(lib_path):
    from dafoam_b200.pyDASolvers import pyDASolvers
    d = tempfile.mkdtemp(prefix="dab_tpass_")
    write_transonic_passage(d)
    opts = dict(normalizeStates=dict(U=50.0, p=101325.0, T=300.0, nuTilda=1e-3, phi=1.0), primalMinResTol=1e-9, primalMaxIters=3000)
    sol = pyDASolvers("DATurboFoam -python", opts, caseDir=d, _lib_path=lib_path)
    n = sol.getNLocalAdjointStates()
    W0, R = np.zeros(n), np.zeros(n)
    sol.getOFFields(W0)
    sol.getResiduals(R)
    r0 = np.linalg.norm(R)
    assert sol.solvePrimal() == 0, sol.primalStats.max_residual
    sol.getResiduals(R)
    assert np.linalg.norm(R) < 1e-6 * r0, (r0, np.linalg.norm(R))


def test_transonic_passage_host_build():
    check_passage(HOSTSIM)


@pytest.mark.gpu
def test_transonic_passage_cuda():
    check_passage(None)


def run_two_ranks(extra, port):
    d = tempfile.mkdtemp(prefix="dab_tmp_")
    write_transonic_passage(d)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "mp_transonic_worker.py"), d] + extra
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, OMP_NUM_THREADS="1"), cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count(" ok: ") == 2, r.stdout


def test_transonic_passage_two_ranks_host_build():
    run_two_ranks([], 29771)


@pytest.mark.gpu
def test_transonic_passage_two_gpus_cuda():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_two_ranks(["cuda"], 29773)


# ---- (d) primal -> adjoint -> total derivative against re-converged primals --------------------------------------------------------
def check_total_derivative(lib_path):
    from dafoam_b200.pyDASolvers import KSP, Mat
    fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection", "direction": [1.0, 0.0, 0.0],
                 "scale": 1e-3}}
    inp = {"patchV": {"type": "patchVelocity", "patches": ["inout"], "flowAxis": "x", "normalAxis": "y", "components": ["solver"]}}
    mesh, orc, sol, W = transonic_case("sensibleEnthalpy", "Gauss upwind", lib_path, function=fn, inputs=inp)
    # the normalised residuals of this case reach round-off between 1e-10 and 1e-9 (p ~ 1e5)
    sol.updateDAOption(dict(transonicPCOption=1, primalMinResTol=1e-10, primalMaxIters=2500,
                            adjEqnOption=dict(gmresRelTol=1e-12, gmresMaxIters=1500, gmresRestart=1500, pcConLevel=3)))
    mag, aoa = float(np.hypot(U0[0], U0[1])), float(np.degrees(np.arctan2(U0[1], U0[0])))
    x = np.array([mag, aoa])
    sol.setSolverInput("patchV", "patchVelocity", 2, x)
    assert sol.solvePrimal() == 0, sol.primalStats.max_residual
    n = orc.ndof
    W1 = np.zeros(n)
    sol.getOFFields(W1)
    one = np.array([1.0])
    dFdx, dFdW, dRdxTpsi = np.zeros(2), np.zeros(n), np.zeros(2)
    sol.calcJacTVecProduct("patchV", "patchVelocity", x, "CD", "function", one, dFdx)
    sol.calcJacTVecProduct("states", "stateVar", W1, "CD", "function", one, dFdW)
    pc, ksp = Mat(), KSP()
    sol.calcdRdWT(1, pc)
    sol.createMLRKSPMatrixFree(pc, ksp)
    psi = np.zeros(n)
    assert sol.solveLinearEqn(ksp, dFdW, psi) == 0
    sol.calcJacTVecProduct("patchV", "patchVelocity", x, "R", "residual", psi, dRdxTpsi)
    total = dFdx - dRdxTpsi
    # central differences over re-converged transonic primals, each from the converged state
    fd = np.zeros(2)
    for i, h in enumerate((0.5, 0.005)):  # |U| [m/s], angle of attack [deg]: central differences steady to 1e-6 at these steps
        F = []
        for sgn in (1.0, -1.0):
            xi = x.copy()
            xi[i] += sgn * h
            sol.updateOFFields(W1)
            sol.setSolverInput("patchV", "patchVelocity", 2, xi)
            assert sol.solvePrimal() == 0, sol.primalStats.max_residual
            F.append(sol.calcFunction("CD"))
        fd[i] = (F[0] - F[1]) / (2 * h)
    assert np.all(np.abs(fd) > 0)
    assert np.all(np.abs(total - fd) <= 2e-5 * np.abs(fd)), (total, fd)


def test_transonic_total_derivative_host_build():
    check_total_derivative(HOSTSIM)


@pytest.mark.gpu
def test_transonic_total_derivative_cuda():
    check_total_derivative(None)


# ---- out of scope: the other compressible solvers keep their error -----------------------------------------------------------------
def check_other_solvers_refuse(lib_path):
    from dafoam_b200.pyDASolvers import pyDASolvers
    mesh = cases.naca0012_ogrid(ni=24, nj=12, nk=2)
    th = cases.default_thermo()
    bcs = cases.compressible_bcs(cases.default_bcs_naca(U0=U0))
    for solver in ("DARhoSimpleCFoam", "DARhoSimpleFoam"):
        d = tempfile.mkdtemp(prefix="dab_tref_")
        cases.write_case(d, mesh, bcs, thermo=th, transonic=True)
        sol = pyDASolvers("%s -python" % solver, dict(normalizeStates=dict(NS_C, U=float(U0[0]))), caseDir=d, _lib_path=lib_path)
        with pytest.raises(Exception, match="transonic pressure corrector of %s is not built" % solver):
            sol.solvePrimal()


def test_other_solvers_keep_the_error_host_build():
    check_other_solvers_refuse(HOSTSIM)
