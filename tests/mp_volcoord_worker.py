"""Worker of tests/test_volcoord_partitioned.py (launched through torch.distributed.run): the `volCoord` products and updateOFMesh
on N ranks against one rank on the same case.  Each rank returns the contribution of its owned rows over the full point list; the
sum over the ranks is the one-rank product."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dafoam_b200.pyDASolvers import pyDASolvers, set_comm_callbacks  # noqa: E402
from tests.common import HOSTSIM, NORM_STATES  # noqa: E402
from tests.test_volcoord_partitioned import FN, TURBO_OPTS, periodic_displacement  # noqa: E402


def main():
    case_dir, kind = sys.argv[1], sys.argv[2]
    cuda = len(sys.argv) > 3 and sys.argv[3] == "cuda"
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    lib = None if cuda else HOSTSIM

    def exchange(peers, sends, recvs):
        reqs = []
        for p, s, r in zip(peers, sends, recvs):
            if r.size:
                reqs.append(dist.irecv(torch.from_numpy(r), src=p))
            if s.size:
                reqs.append(dist.isend(torch.from_numpy(np.ascontiguousarray(s)), dst=p))
        for q in reqs:
            q.wait()

    def allreduce(a):
        dist.all_reduce(torch.from_numpy(a))

    uid = None
    if cuda:
        from dafoam_b200.pyDASolvers import nccl_unique_id
        box = [nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        uid = box[0]
    else:
        set_comm_callbacks(exchange, allreduce, HOSTSIM)
    comp = "turbo" in kind
    if kind.startswith("passage"):
        name, opts = ("DATurboFoam -python", dict(TURBO_OPTS)) if comp else ("DASimpleFoam -python", dict(normalizeStates=NORM_STATES, function=FN))
    else:
        name = "DASimpleFoam -python"
        opts = dict(normalizeStates=NORM_STATES, function={"CD": dict(FN["CD"], patches=["wing"], direction=[1.0, 0.0, 0.0])})
    dev = rank if cuda else 0
    one = pyDASolvers(name, opts, caseDir=case_dir, device=dev, _lib_path=lib)
    par = pyDASolvers(name, opts, caseDir=case_dir, device=dev, rank=rank, nRanks=world, ncclUniqueId=uid, _lib_path=lib)
    nCg = one.getNGlobalCells()
    ns = 6 if comp else 5
    nFg = int(one.getLocalToGlobal("faces").max()) + 1

    def maps(sol):
        idx = sol.localStateIndex(nCg, nFg, compressible=comp)
        owned = np.concatenate([np.ones(ns * sol.getNLocalCells(), dtype=bool), sol.getLocalToGlobal("faceOwned").astype(bool)])
        return idx, owned

    i1, o1 = maps(one)
    i2, o2 = maps(par)
    n = ns * nCg + nFg
    W1 = np.zeros(i1.size)
    one.getOFFields(W1)
    rng = np.random.default_rng(5)
    Wg = np.zeros(n)
    Wg[i1[o1]] = W1[o1]
    Wg *= 1.0 + 0.01 * rng.uniform(-1, 1, n)
    Wg[:3 * nCg] += 0.3 * rng.uniform(-1, 1, 3 * nCg)
    one.updateOFFields(np.ascontiguousarray(Wg[i1]))
    par.updateOFFields(np.ascontiguousarray(Wg[i2]))
    nP3 = 3 * one.getNLocalPoints()
    assert par.getNLocalPoints() == one.getNLocalPoints()
    pts = np.zeros(nP3)
    one.getOFMeshPoints(pts)

    def rel(a, b):
        return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)

    # the device geometry at the unmoved points reproduces this rank's slice of the host geometry
    R0, R0b = np.zeros(i2.size), np.zeros(i2.size)
    par.getResiduals(R0)
    par.updateOFMesh(pts)
    par.getResiduals(R0b)
    e0 = rel(R0b[o2], R0[o2])
    assert e0 < 1e-12, e0

    def summed(a):
        t = torch.from_numpy(a.copy())
        dist.all_reduce(t)
        return t.numpy()

    # [dR/dx_v]^T psi and dF/dx_v: the sum over the ranks equals one rank
    psi = rng.uniform(-1, 1, n)
    x1, x2 = np.ascontiguousarray(psi[i1]), np.ascontiguousarray(psi[i2])
    x1[~o1] = 0.0
    x2[~o2] = 0.0
    p1, p2 = np.zeros(nP3), np.zeros(nP3)
    one.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", x1, p1)
    par.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", x2, p2)
    e1 = rel(summed(p2), p1)
    assert e1 < 1e-9, e1
    f1, f2 = np.zeros(nP3), np.zeros(nP3)
    one.calcJacTVecProduct("x", "volCoord", pts, "CD", "function", np.array([1.0]), f1)
    par.calcJacTVecProduct("x", "volCoord", pts, "CD", "function", np.array([1.0]), f2)
    e2 = rel(summed(f2), f1)
    assert e2 < 1e-9, e2
    assert par.getVolCoordEvaluations() == one.getVolCoordEvaluations() > 0  # one colouring on every rank

    # updateOFMesh with a smooth (periodic) displacement: each rank's residual rows and the force are the one-rank values
    if kind.startswith("passage"):
        v = periodic_displacement(pts)
    else:
        X = pts.reshape(-1, 3)
        v = np.stack([np.sin(3.0 * X[:, 1]) * 1e-3, np.cos(2.0 * X[:, 0]) * 1e-3, np.zeros(len(X))], axis=1).ravel()
    one.updateOFMesh(pts + v)
    par.updateOFMesh(pts + v)
    R1, R2 = np.zeros(i1.size), np.zeros(i2.size)
    one.getResiduals(R1)
    par.getResiduals(R2)
    Rg = np.zeros(n)
    Rg[i1[o1]] = R1[o1]
    e3 = rel(R2[o2], Rg[i2][o2])
    assert e3 < 1e-12, e3
    F1, F2 = one.calcFunction("CD"), par.calcFunction("CD")
    assert abs(F1 - F2) <= 1e-12 * abs(F1), (F1, F2)
    print("rank %d ok: unmoved rebuild %.1e, residual product %.1e, dF/dx %.1e, moved residual %.1e" % (rank, e0, e1, e2, e3), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
