"""[dR/dx_v]^T psi and dF/dx_v on the GPU: set-up (colouring) and product seconds.

    python scripts/volcoord_bench.py [--mesh naca|passage] [--solver DASimpleFoam|DATurboFoam]
    python -m torch.distributed.run --nproc-per-node N scripts/volcoord_bench.py --mesh passage --solver DATurboFoam

Under torch.distributed every rank drives one GPU (NCCL between them) and rank 0 prints the times, the maximum over the ranks.
env: VB_NI, VB_NJ (NACA O-grid), VB_NR, VB_NT, VB_NZ (passage)."""
import argparse, json, os, sys, tempfile, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import pyDASolvers

ap = argparse.ArgumentParser()
ap.add_argument("--mesh", default="naca", choices=["naca", "passage"])
ap.add_argument("--solver", default="DASimpleFoam", choices=["DASimpleFoam", "DATurboFoam"])
a = ap.parse_args()
world = int(os.environ.get("WORLD_SIZE", "1"))
rank, uid, dist = 0, None, None
if world > 1:
    import torch.distributed as dist
    from dafoam_b200.pyDASolvers import nccl_unique_id
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    box = [nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    uid = box[0]
turbo = a.solver == "DATurboFoam"
box = [tempfile.mkdtemp(prefix="dab_vb_") if rank == 0 else None]
if dist:
    dist.broadcast_object_list(box, src=0)
d = box[0]
if a.mesh == "naca":
    mesh = cases.naca0012_ogrid(ni=int(os.environ.get("VB_NI", 1400)), nj=int(os.environ.get("VB_NJ", 700)), nk=1)
    bcs, patch, direction = cases.default_bcs_naca(), "wing", [1.0, 0.0, 0.0]
else:
    mesh = cases.annular_passage(nr=int(os.environ.get("VB_NR", 24)), nt=int(os.environ.get("VB_NT", 24)), nz=int(os.environ.get("VB_NZ", 48)), n_sectors=7)
    bcs, patch, direction = cases.default_bcs_passage(Uin=(0.0, 0.0, 60.0 if turbo else 10.0)), "hub", [0.0, 0.0, 1.0]
kw = {}
if turbo:
    bcs = cases.compressible_bcs(bcs)
    kw = dict(thermo=cases.default_thermo(energy="sensibleEnthalpy"))
    if a.mesh == "passage":
        kw["mrf"] = dict(cellZone="rotor", cells=list(range(mesh.n_cells)), origin=(0.0, 0.0, 0.0), axis=(0.0, 0.0, 1.0), omega=200.0,
                         nonRotatingPatches=["inlet", "outlet", "shroud"])
if rank == 0:
    cases.write_case(d, mesh, bcs, binary=True, **kw)
if dist:
    dist.barrier()
fn = {"CD": {"type": "force", "source": "patchToFace", "patches": [patch], "directionMode": "fixedDirection", "direction": direction, "scale": 1.0}}
ns = dict(U=50.0, p=101325.0, T=300.0, nuTilda=1e-3, phi=1.0) if turbo else dict(U=10.0, p=50.0, nuTilda=1e-3, phi=1.0)
opts = dict(normalizeStates=ns, function=fn, adjEqnOption=dict(printInfo=1 if rank == 0 else 0))
sol = pyDASolvers(a.solver + " -python", opts, caseDir=d, device=rank, rank=rank, nRanks=world, ncclUniqueId=uid)
n, nP3 = sol.getNLocalAdjointStates(), 3 * sol.getNLocalPoints()
pts = np.zeros(nP3)
sol.getOFMeshPoints(pts)
psi = np.random.default_rng(7 + rank).uniform(-1, 1, n)
prod = np.zeros(nP3)


def timed(f):
    if dist:
        dist.barrier()
    t = time.time()
    f()
    t = time.time() - t
    if dist:
        box = [None] * world
        dist.all_gather_object(box, t)
        t = max(box)
    return t


t_first = timed(lambda: sol.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", psi, prod))
t_prod = timed(lambda: sol.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", psi, prod))
dFdx = np.zeros(nP3)
t_fn = timed(lambda: sol.calcJacTVecProduct("x", "volCoord", pts, "CD", "function", np.array([1.0]), dFdx))
if rank == 0:
    out = dict(mesh=a.mesh, solver=a.solver, gpus=world, cells=mesh.n_cells, points=nP3 // 3, setup_s=t_first - t_prod, product_s=t_prod,
               function_s=t_fn, residual_evaluations=sol.getVolCoordEvaluations(), norm_rank0=float(np.linalg.norm(prod)), norm_dFdx_rank0=float(np.linalg.norm(dFdx)))
    print(json.dumps(out), flush=True)
if dist:
    dist.barrier()
    dist.destroy_process_group()
