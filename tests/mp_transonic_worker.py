"""Worker of the two-rank transonic primal test (launched by tests/test_transonic_primal.py through torch.distributed.run): DATurboFoam
with SIMPLE { transonic yes; } on the cyclic passage with an MRF zone, cut in two, against the same passage on one rank.  The host
build routes the ghost exchanges and all-reduces of the BiCGStab through gloo; the CUDA build uses NCCL."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dafoam_b200.pyDASolvers import pyDASolvers, set_comm_callbacks  # noqa: E402
from tests.common import HOSTSIM  # noqa: E402


def main():
    case_dir = sys.argv[1]
    cuda = len(sys.argv) > 2 and sys.argv[2] == "cuda"
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
    dev = rank if cuda else 0
    opts = dict(normalizeStates=dict(U=50.0, p=101325.0, T=300.0, nuTilda=1e-3, phi=1.0), primalMinResTol=1e-11, primalMaxIters=4000)
    one = pyDASolvers("DATurboFoam -python", opts, caseDir=case_dir, device=dev, _lib_path=lib)
    two = pyDASolvers("DATurboFoam -python", opts, caseDir=case_dir, device=dev, rank=rank, nRanks=world, ncclUniqueId=uid, _lib_path=lib)
    nCg = one.getNGlobalCells()
    fo1 = one.getLocalToGlobal("faceOwned").astype(bool)
    nFg = int(one.getLocalToGlobal("faces").max()) + 1
    ns = 6
    n = ns * nCg + nFg

    def maps(sol):
        idx = sol.localStateIndex(nCg, nFg, compressible=True)
        owned = np.concatenate([np.ones(ns * sol.getNLocalCells(), dtype=bool), sol.getLocalToGlobal("faceOwned").astype(bool)])
        return idx, owned

    i1, o1 = maps(one)
    i2, o2 = maps(two)
    assert fo1.sum() == nFg
    f1, f2 = one.solvePrimal(), two.solvePrimal()
    assert f1 == 0 and f2 == 0, (f1, f2, one.primalStats.max_residual, two.primalStats.max_residual)
    W1, W2 = np.zeros(i1.size), np.zeros(i2.size)
    one.getOFFields(W1)
    two.getOFFields(W2)
    g1 = np.zeros(n)
    g1[i1[o1]] = W1[o1]
    nCl = two.getNLocalCells()
    errs = []
    for a, b in [(0, 3 * nCl)] + [(k * nCl, (k + 1) * nCl) for k in range(3, ns)]:
        ref = g1[i2][a:b]
        errs.append(np.abs(W2[a:b] - ref).max() / np.abs(ref).max())
    fo = o2[ns * nCl:]
    ref = g1[i2][ns * nCl:][fo]
    errs.append(np.abs(W2[ns * nCl:][fo] - ref).max() / np.abs(ref).max())
    assert max(errs) < 1e-8, errs
    assert two.primalStats.p_iterations > 0
    print("rank %d ok: primal iterations one rank %d, two ranks %d, BiCGStab iterations %d / %d, state difference %.1e"
          % (rank, one.primalStats.iterations, two.primalStats.iterations, one.primalStats.p_iterations, two.primalStats.p_iterations,
             max(errs)), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
