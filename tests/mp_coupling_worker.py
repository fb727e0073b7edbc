"""Worker of tests/test_force_coupling.py (launched through torch.distributed.run): forceCouplingOutput on N ranks against one rank
on the same case.  Each rank outputs the nodes of its own faces, so a point on a partition seam is a node of every rank around it;
per global point the sum over the ranks is the one-rank value.  Node seeds are taken per global point, so the state products
(mapped to global states) and the summed volCoord products equal one rank."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dafoam_b200.pyDASolvers import pyDASolvers, set_comm_callbacks  # noqa: E402
from tests.common import HOSTSIM, NORM_STATES  # noqa: E402
from tests.test_volcoord_partitioned import TURBO_OPTS  # noqa: E402

FC = "forceCouplingOutput"


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
    comp = kind == "passageturbo"
    if comp:
        name, opts = "DATurboFoam -python", dict(TURBO_OPTS)
        opts["outputInfo"] = {"f_aero": {"type": FC, "patches": ["hub"], "pRef": 101325.0}}
    else:
        name = "DASimpleFoam -python"
        opts = dict(normalizeStates=NORM_STATES, outputInfo={"f_aero": {"type": FC, "patches": ["wing", "sym1"], "pRef": 0.4}})
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
    W1, W2 = np.ascontiguousarray(Wg[i1]), np.ascontiguousarray(Wg[i2])
    one.updateOFFields(W1)
    par.updateOFFields(W2)
    nP = one.getNLocalPoints()
    pts = np.zeros(3 * nP)
    one.getOFMeshPoints(pts)

    def rel(a, b):
        return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)

    def summed(a):
        t = torch.from_numpy(a.copy())
        dist.all_reduce(t)
        return t.numpy()

    def per_point(sol, f):
        acc = np.zeros((nP, 3))
        np.add.at(acc, sol.getForceCouplingPoints("f_aero"), f.reshape(-1, 3))
        return acc

    # the value: per global point, the ranks' shares add up to the one-rank force
    n1, n2 = one.getOutputSize("f_aero", FC), par.getOutputSize("f_aero", FC)
    f1, f2 = np.zeros(n1), np.zeros(n2)
    one.calcOutput("f_aero", FC, f1)
    par.calcOutput("f_aero", FC, f2)
    e1 = rel(summed(per_point(par, f2)), per_point(one, f1))
    assert e1 < 1e-12, e1
    # state product with one seed per global point
    G = rng.uniform(-1, 1, (nP, 3))
    s1 = np.ascontiguousarray(G[one.getForceCouplingPoints("f_aero")].ravel())
    s2 = np.ascontiguousarray(G[par.getForceCouplingPoints("f_aero")].ravel())
    p1, p2 = np.zeros(i1.size), np.zeros(i2.size)
    one.calcJacTVecProduct("states", "stateVar", W1, "f_aero", FC, s1, p1)
    par.calcJacTVecProduct("states", "stateVar", W2, "f_aero", FC, s2, p2)
    Pg = np.zeros(n)
    Pg[i1[o1]] = p1[o1]
    e2 = rel(p2[o2], Pg[i2][o2])
    assert np.abs(p1).max() > 0 and e2 < 1e-12, e2
    # volCoord product: the sum over the ranks equals one rank
    x1, x2 = np.zeros(3 * nP), np.zeros(3 * nP)
    one.calcJacTVecProduct("x", "volCoord", pts, "f_aero", FC, s1, x1)
    par.calcJacTVecProduct("x", "volCoord", pts, "f_aero", FC, s2, x2)
    e3 = rel(summed(x2), x1)
    assert np.abs(x1).max() > 0 and e3 < 1e-9, e3
    print("rank %d ok: %d nodes (one rank %d), value %.1e, state product %.1e, volCoord product %.1e" % (rank, n2 // 3, n1 // 3, e1, e2, e3),
          flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
