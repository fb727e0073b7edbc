"""SIMPLE primal on the GPU: iterations, residuals, seconds; then |R(W)|.
env: PB_CASE = incompressible (default: DASimpleFoam on the NACA0012 O-grid), transonic (DATurboFoam, SIMPLE { transonic yes; }, on
the O-grid with an MRF zone around the aerofoil, freestream about Mach 0.66) or transonic_passage (DATurboFoam transonic on BASELINE
config 5's annular rotor passage: cyclic sides, MRF zone); PB_NI, PB_NJ, PB_NK (default 1400x700x1; the passage takes nr x nt x nz),
PB_ITERS (default 2000), PB_TOL (default 1e-8), PB_OUT (optional: also write the result as a JSON file there)"""
import json, os, sys, tempfile, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import pyDASolvers

kind = os.environ.get("PB_CASE", "incompressible")
ni, nj, nk = int(os.environ.get("PB_NI", 1400)), int(os.environ.get("PB_NJ", 700)), int(os.environ.get("PB_NK", 1))
iters, tol = int(os.environ.get("PB_ITERS", 2000)), float(os.environ.get("PB_TOL", 1e-8))
t0 = time.time()
d = tempfile.mkdtemp(prefix="dab_pb_")
a3 = np.deg2rad(3.0)
if kind == "incompressible":
    mesh = cases.naca0012_ogrid(ni=ni, nj=nj, nk=1)
    cases.write_case(d, mesh, cases.default_bcs_naca(U0=(10.0 * np.cos(a3), 10.0 * np.sin(a3), 0.0)), binary=True)
    fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection",
                 "direction": [float(np.cos(a3)), float(np.sin(a3)), 0.0], "scale": 1.0 / (0.5 * 100 * 0.1)},
          "CL": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection",
                 "direction": [-float(np.sin(a3)), float(np.cos(a3)), 0.0], "scale": 1.0 / (0.5 * 100 * 0.1)}}
    solver, ns = "DASimpleFoam", dict(U=10.0, p=50.0, nuTilda=1e-3, phi=1.0)
else:
    # div(phid,p) upwind; PB_RELAX = fields p, equations p (0: no pEqn.relax()), U, h (default 0.3,1,0.7,0.7)
    th = cases.default_thermo(energy="sensibleEnthalpy")
    rp, rpe, ru, rh = [float(v) for v in os.environ.get("PB_RELAX", "0.3,1,0.7,0.7").split(",")]
    kw = dict(thermo=th, transonic=True, div_phid_p="Gauss upwind", relax_p=rp, relax_p_eqn=rpe if rpe > 0 else None, relax_u=ru,
              relax_he=rh, binary=True, div_u="bounded Gauss linearUpwindV grad(U)")
    solver, ns = "DATurboFoam", dict(U=230.0, p=101325.0, T=300.0, nuTilda=1e-3, phi=1.0)
    if kind == "transonic":
        U0 = (230.0, 8.0, 0.0)
        mesh = cases.naca0012_ogrid(ni=ni, nj=nj, nk=1)
        from tests.common import mrf_zone
        cases.write_case(d, mesh, cases.compressible_bcs(cases.default_bcs_naca(U0=U0)), mrf=mrf_zone(mesh, omega=0.3), **kw)
        fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection",
                     "direction": [1.0, 0.0, 0.0], "scale": 1.0}}
    elif kind == "transonic_passage":
        mesh = cases.annular_passage(nr=ni, nt=nj, nz=nk, r0=0.2, r1=0.35, lz=0.3, n_sectors=36)
        mrf = dict(cellZone="rotor", cells=np.arange(mesh.n_cells), origin=(0.0, 0.0, 0.0), axis=(0.0, 0.0, 1.0), omega=300.0,
                   nonRotatingPatches=["inlet", "outlet", "shroud"])
        cases.write_case(d, mesh, cases.compressible_bcs(cases.default_bcs_passage(Uin=(0.0, 0.0, 100.0))), mrf=mrf, **kw)
        fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["hub"], "directionMode": "fixedDirection",
                     "direction": [0.0, 0.0, 1.0], "scale": 1.0}}
        ns = dict(ns, U=100.0)
    else:
        raise SystemExit("PB_CASE: incompressible, transonic or transonic_passage")
sol = pyDASolvers("%s -python" % solver, dict(normalizeStates=ns, function=fn, primalMinResTol=tol, primalMaxIters=iters, printInterval=100,
                                              adjEqnOption=dict(printInfo=1)), caseDir=d)
n = sol.getNLocalAdjointStates()
R = np.zeros(n)
sol.getResiduals(R)
r0 = float(np.linalg.norm(R))
t1 = time.time()
error = None
try:
    fail = sol.solvePrimal()
except Exception as e:  # noqa: BLE001  (a diverged run still reports what it measured)
    fail, error = 1, str(e)
st = sol.primalStats
sol.getResiduals(R)
out = dict(case=kind, solver=solver, relax=os.environ.get("PB_RELAX", "0.3,1,0.7,0.7") if kind != "incompressible" else None,
           cells=mesh.n_cells, setup_sec=t1 - t0, fail=fail, error=error, iterations=st.iterations, converged=st.converged,
           max_residual=st.max_residual, res_u=list(st.res_u), res_p=st.res_p, res_nutilda=st.res_nutilda, p_iterations=st.p_iterations,
           p_iterations_per_solve=st.p_iterations / max(st.iterations, 1), seconds=st.seconds,
           ms_per_iteration=1e3 * st.seconds / max(st.iterations, 1), R0=r0, R=float(np.linalg.norm(R)),
           **{k: sol.calcFunction(k) for k in fn})
try:
    import subprocess
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True,
                                text=True, timeout=30).stdout.strip()
except Exception:  # noqa: BLE001
    pass
print(json.dumps(out))
if os.environ.get("PB_OUT"):  # optional copy of the result line as a JSON file
    os.makedirs(os.path.dirname(os.path.abspath(os.environ["PB_OUT"])), exist_ok=True)
    json.dump(out, open(os.environ["PB_OUT"], "w"), indent=1)
