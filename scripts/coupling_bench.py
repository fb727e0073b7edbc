"""forceCouplingOutput on one GPU: calcOutput and the stateVar product on the NACA0012 O-grid of bench.py (1440x720x1 = 1 036 800
cells), and the volCoord product on the passage of scripts/volcoord_bench.py, next to the force function's own products.

    python scripts/coupling_bench.py [--reps 20]

Every timed call ends in a device-to-host copy of its result (a device synchronise); each is warmed up first.  Prints the card's
name and power limit, then one JSON line.  env: CB_NI, CB_NJ (O-grid), CB_NR, CB_NT, CB_NZ (passage)."""
import argparse, json, os, subprocess, sys, tempfile, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import pyDASolvers

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
a = ap.parse_args()
FC = "forceCouplingOutput"
NS = dict(U=10.0, p=50.0, nuTilda=1e-3, phi=1.0)


def timed(f, reps, warm=2):
    for _ in range(warm):
        f()
    t = time.perf_counter()
    for _ in range(reps):
        f()
    return (time.perf_counter() - t) / reps * 1e3


def options(patch, direction):
    return dict(normalizeStates=NS,
                function={"CD": {"type": "force", "source": "patchToFace", "patches": [patch], "directionMode": "fixedDirection",
                                 "direction": direction, "scale": 1.0}},
                outputInfo={"f_aero": {"type": FC, "patches": [patch], "pRef": 0.0}})


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
out = dict(card=card)

# NACA0012 O-grid: calcOutput and the state product, against calcFunction and the force function's state product
mesh = cases.naca0012_ogrid(ni=int(os.environ.get("CB_NI", 1440)), nj=int(os.environ.get("CB_NJ", 720)), nk=1)
d = tempfile.mkdtemp(prefix="dab_cb_")
cases.write_case(d, mesh, cases.default_bcs_naca(), binary=True)
sol = pyDASolvers("DASimpleFoam -python", options("wing", [1.0, 0.0, 0.0]), caseDir=d)
y = np.zeros(sol.getNLocalCells())
sol.getOFField("yWall", "scalar", y)
W = cases.boundary_layer_state(mesh, y, noise=0.001)
sol.updateOFFields(W)
n, n3 = sol.getNLocalAdjointStates(), sol.getOutputSize("f_aero", FC)
f, prod = np.zeros(n3), np.zeros(n)
seed = np.random.default_rng(3).uniform(-1, 1, n3)
out.update(naca_cells=mesh.n_cells, naca_nodes=n3 // 3,
           calcOutput_ms=timed(lambda: sol.calcOutput("f_aero", FC, f), a.reps),
           calcFunction_ms=timed(lambda: sol.calcFunction("CD"), a.reps),
           state_product_ms=timed(lambda: sol.calcJacTVecProduct("states", "stateVar", W, "f_aero", FC, seed, prod), a.reps),
           dFdW_ms=timed(lambda: sol.calcJacTVecProduct("states", "stateVar", W, "CD", "function", np.array([1.0]), prod), a.reps),
           state_product_d2h_MB=n * 8 / 1e6)
del sol

# passage: the volCoord product (coloured central differences), against the force function's
pm = cases.annular_passage(nr=int(os.environ.get("CB_NR", 24)), nt=int(os.environ.get("CB_NT", 24)), nz=int(os.environ.get("CB_NZ", 48)), n_sectors=7)
d = tempfile.mkdtemp(prefix="dab_cb_")
cases.write_case(d, pm, cases.default_bcs_passage(Uin=(0.0, 0.0, 10.0)), binary=True)
sol = pyDASolvers("DASimpleFoam -python", options("hub", [0.0, 0.0, 1.0]), caseDir=d)
nP3 = 3 * sol.getNLocalPoints()
pts = np.zeros(nP3)
sol.getOFMeshPoints(pts)
n3 = sol.getOutputSize("f_aero", FC)
seed = np.random.default_rng(5).uniform(-1, 1, n3)
dx = np.zeros(nP3)
reps = max(1, a.reps // 10)
out.update(passage_cells=pm.n_cells, passage_nodes=n3 // 3, volcoord_evaluations=None,
           volCoord_product_ms=timed(lambda: sol.calcJacTVecProduct("x", "volCoord", pts, "f_aero", FC, seed, dx), reps, warm=1),
           volCoord_function_ms=timed(lambda: sol.calcJacTVecProduct("x", "volCoord", pts, "CD", "function", np.array([1.0]), dx), reps, warm=1))
out["volcoord_evaluations"] = sol.getVolCoordEvaluations()
print(json.dumps(out), flush=True)
