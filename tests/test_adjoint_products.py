"""The transpose products of the adjoint checked entry by entry, not through the convergence of a solve:
  (a) y = diag(s) [dR/dW]^T psi (calcdRdWTPsiAD) against a dense central-difference Jacobian of the oracle's float64 residual, and
      against the oracle's exact tape product as a second witness;
  (b) [dR/dx_v]^T psi (the volCoord input of calcJacTVecProduct) against a dense central-difference Jacobian of the oracle's residual
      over the mesh points;
  (c) the same products on 2 and 3 partitions (ghost-cell halos, cut faces) and on a cyclic passage (partner faces of a coupled pair,
      on one partition and with the pair cut between two), gathered and compared with one partition and with (a) / (b).
s_j is the engine's state scaling (normalizeStates, times |Sf| for phi).  The probes: random psi, the dot-product identity
<psi, J v> = <J^T psi, v> with J v from the engine's own residual and from the oracle's forward tangent, psi = e_i on every residual
row of a cell next to each patch type (wall, inlet, outlet, symmetry, cyclic) -- the boundary-face pass of RevA/RevB/RevC and the
partner contribution of a coupled face -- and psi supported on cells without boundary faces.

Shapes: the product's kernels run one cell per thread in 128-thread CTAs, so the meshes have 6 cells (22 boundary faces: less than a
warp), 129 cells (one CTA plus one) and 140 cells (7 x 5 x 4, the only one with cells that have no boundary face).  The product has
no float32 path (fp32 storage exists only for the preconditioner's factors), and its kernels are gathers without atomics, so
repeated products must be bitwise equal.

Every reference below is plain numpy around the oracle (oracle/oracle.cpp); none of it goes through the engine's kernels.  The file
is also the worker of the partitioned cases: `python -m torch.distributed.run ... tests/test_adjoint_products.py <case dir> <kind>
<host|cuda>`."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from dafoam_b200 import cases  # noqa: E402
from dafoam_b200.pyDASolvers import pyDASolvers  # noqa: E402
from oracle.pyoracle import Oracle, synthetic_state  # noqa: E402
from tests.common import ALL_RES, HOSTSIM, NORM_STATES  # noqa: E402

# ---- steps and tolerances ----------------------------------------------------------------------------------------------------
# Entry errors are |y_j - ref_j| / scale_j (entry_scale, mesh_scale): scale_j sums |psi_i| times the size of the terms of J_ij, so a
# face missed or counted twice moves its entries by O(1) while roundoff and difference error stay far below.  An entry of a cell
# that no row of psi is coupled to must be exactly zero.  Measured: host build (x86-64, no FMA contraction) over every probe.
FD_H = 1e-6          # central-difference step, relative to s_j (states) or in metres (mesh points; cells of 0.03-0.3 m)
FLOOR_REL = 1e-9     # floor of an entry's scale, times |J|max: residual rows that vanish up to roundoff (z-momentum of a 2-D flow)
TOL_FD_CHECK = 1e-6  # J_fd vs the oracle's exact tangent / tape: truncation (h / cell size)^2 plus roundoff eps / h; measured 2e-9
#                      (states), 2.4e-7 of the largest entry (mesh points)
TOL_FD = 1e-6        # product vs J_fd^T psi: the same difference error summed over psi; measured 1.8e-7
TOL_TAPE = 1e-7      # product vs the oracle's tape: both exact float64, so only entries at the floor differ (their 1e-14 roundoff
#                      over a floor of 1e-9 |J|max); measured 2.6e-8
TOL_DOT = 1e-12      # <psi, J v> (exact tangent) vs <y, v>, relative to sum |psi_i (J v)_i|: float64 sums of ~1e3 terms; measured 8e-16
TOL_DOT_FD = 1e-8    # the same with J v from the engine's own residual by central differences (step FD_H); measured 1.6e-10
TOL_X = 1e-6         # volCoord product (the engine's own coloured central differences) vs J_x,fd^T psi; measured 2.2e-8
TOL_PART = 1e-8      # several partitions vs one: halo copies are exact, but a cut face is evaluated from the other side (the same
#                      terms in another order), which entries at the floor see; measured 3.5e-10 (a coupled face's phi)
TOL_PART_X = 1e-8    # the same for the volCoord product, relative to its largest entry: each partition takes its own differences; measured 3.9e-10


# ---- cases ---------------------------------------------------------------------------------------------------------------------
PATCH_TYPE = {"inlet": "inlet", "outlet": "outlet", "walls": "wall", "sym1": "symmetry", "sym2": "symmetry", "hub": "wall",
              "shroud": "wall", "per_lo": "cyclic", "per_hi": "cyclic"}
MESHES = {
    "channel_6": lambda: cases.channel(nx=3, ny=2, nz=1),      # 6 cells, 22 boundary faces: fewer than a warp
    "channel_129": lambda: cases.channel(nx=43, ny=3, nz=1),   # 129 cells: one 128-thread CTA plus one cell
    "channel_140": lambda: cases.channel(nx=7, ny=5, nz=4),    # 140 cells, 30 of them without a boundary face
}
DIV_U = "linearUpwindV"
ENGINE_OPTS = dict(normalizeStates=NORM_STATES, normalizeResiduals=list(ALL_RES))


def kinds_of(n_cells, n_dof):
    k = np.empty(n_dof, dtype=object)
    k[:3 * n_cells] = ["Ux", "Uy", "Uz"] * n_cells
    k[3 * n_cells:4 * n_cells] = "p"
    k[4 * n_cells:5 * n_cells] = "nuTilda"
    k[5 * n_cells:] = "phi"
    return k


def state_scales(n_cells, magSf):
    """s_j: the engine's state scaling (normalizeStates; phi also times |Sf|)"""
    return np.concatenate([np.full(3 * n_cells, NORM_STATES["U"]), np.full(n_cells, NORM_STATES["p"]),
                           np.full(n_cells, NORM_STATES["nuTilda"]), NORM_STATES["phi"] * magSf])


class Plain:
    """a mesh without cyclic patches: the engine's single-partition numbering is the polyMesh one, the oracle's too"""
    cyclic = False

    def __init__(self, name):
        self.name = name
        self.mesh = MESHES[name]()
        self.bcs = cases.default_bcs_channel()
        self.orc = Oracle(self.mesh, self.bcs, normalizeStates=NORM_STATES, divU=DIV_U, normalizeResiduals=ALL_RES)
        self.nC = self.mesh.n_cells
        self.n = self.orc.ndof
        self.W = synthetic_state(self.mesh, self.orc.geometry("C"), self.orc.geometry("Sf"))
        self.scale = state_scales(self.nC, self.orc.geometry("magSf"))
        self.kinds = kinds_of(self.nC, self.n)
        own = self.mesh.owner
        self.cell = np.concatenate([np.repeat(np.arange(self.nC), 3), np.arange(self.nC), np.arange(self.nC), own])
        self.face_patch = [""] * self.mesh.n_internal_faces
        for p in self.mesh.patches:
            self.face_patch += [p["name"]] * p["size"]

    def write(self, d):
        cases.write_case(d, self.mesh, self.bcs, div_u="bounded Gauss %s grad(U)" % DIV_U)

    def solver(self, lib_path):
        d = tempfile.mkdtemp(prefix="dab_prod_")
        self.write(d)
        sol = pyDASolvers("DASimpleFoam -python", dict(ENGINE_OPTS), caseDir=d, _lib_path=lib_path)
        sol.updateOFFields(self.W)
        return Engine(sol, np.arange(self.n), np.ones(self.n, dtype=bool))

    def residual(self, W):
        return self.orc.residual(W)

    def tangent(self, v):
        """J v in scaled states: the oracle's forward-mode dual numbers"""
        return self.orc.jvec(self.W, self.scale * v)

    def tape(self, psi):
        self.orc.record(self.W)  # one tape per process: another case's oracle may have recorded since
        return self.orc.jtvec(psi)

    def boundary_rows(self):
        """patch type -> (cell, phi row of one of its faces on that patch), for the first cell next to each patch type"""
        out = {}
        nIF = self.mesh.n_internal_faces
        for p in self.mesh.patches:
            t = PATCH_TYPE[p["name"]]
            if t not in out:
                f = p["start"] + p["size"] // 2
                out[t] = (int(self.mesh.owner[f]), 5 * self.nC + f)
        assert nIF > 0
        return out

    def describe(self, j):
        if j < 5 * self.nC:
            return "%s of cell %d" % (self.kinds[j], self.cell[j])
        f = j - 5 * self.nC
        return "phi of face %d (%s, owner cell %d)" % (f, self.face_patch[f] or "internal", self.cell[j])


class Cyclic:
    """the annular passage with cyclic sides (tests/test_cyclic.py Pair): the engine on one passage, its reference the oracle on the
    closed ring of passages with a passage-periodic state; vectors in the engine's merged numbering (one face per coupled pair)"""
    cyclic = True

    def __init__(self, name, lib_path=HOSTSIM):
        from tests.test_cyclic import Pair, merged_faces
        self.name = name
        self.P = P = Pair(True, "linearUpwind", lib_path=lib_path)
        self.nC, self.n = P.nCs, P.n_sec()
        self.W = P.state()
        self.Wr = P.to_ring(self.W)
        magSf = np.asarray(P.orc.geometry("magSf"))[P.s2f]
        self.scale = state_scales(self.nC, magSf)
        self.kinds = kinds_of(self.nC, self.n)
        so, sn, pname = merged_faces(P.sec)
        self.so, self.sn, self.pname = so, sn, pname
        self.cell = np.concatenate([np.repeat(np.arange(self.nC), 3), np.arange(self.nC), np.arange(self.nC), so])

    def solver(self, lib_path):
        P = self.P if lib_path == HOSTSIM else type(self.P)(True, "linearUpwind", lib_path=lib_path)
        P.sol.updateOFFields(P.local(self.W))
        return Engine(P.sol, P.idx, P.owned)

    def residual(self, W):
        return self.P.from_ring(self.P.orc.residual(self.P.to_ring(W)))

    def tangent(self, v):
        return self.P.from_ring(self.P.orc.jvec(self.Wr, self.P.to_ring(self.scale * v)))

    def tape(self, psi):
        self.P.orc.record(self.Wr)
        return self.P.from_ring(self.P.orc.jtvec(self.P.to_ring(psi)))

    def boundary_rows(self):
        nIF = self.P.sec.n_internal_faces
        out = {}
        # the coupled faces follow the internal faces; owner = the cell on per_lo, neighbour = its partner on per_hi
        g = nIF + int(np.count_nonzero(self.sn[nIF:] >= 0)) // 2
        out["cyclic (per_lo side)"] = (int(self.so[g]), 5 * self.nC + g)
        out["cyclic (per_hi side)"] = (int(self.sn[g]), 5 * self.nC + g)
        for g in range(nIF, len(self.so)):
            if self.sn[g] < 0 and PATCH_TYPE[self.pname[g]] not in out:
                out[PATCH_TYPE[self.pname[g]]] = (int(self.so[g]), 5 * self.nC + g)
        return out

    def describe(self, j):
        if j < 5 * self.nC:
            return "%s of cell %d" % (self.kinds[j], self.cell[j])
        g = j - 5 * self.nC
        what = "coupled" if self.sn[g] >= 0 and g >= self.P.sec.n_internal_faces else (self.pname[g] or "internal")
        return "phi of face %d (%s, owner cell %d)" % (g, what, self.cell[j])


class Engine:
    """the engine's solver on one partition, vectors in the case's numbering (idx: local -> case numbering, owned: the local slots
    that carry a degree of freedom)"""

    def __init__(self, sol, idx, owned):
        self.sol, self.idx, self.owned = sol, idx, owned

    def local(self, v):
        return np.ascontiguousarray(v[self.idx])

    def merged(self, vloc, n):
        out = np.zeros(n)
        out[self.idx[self.owned]] = vloc[self.owned]
        return out

    def product(self, psi):
        y = np.zeros(self.idx.size)
        self.sol.calcdRdWTPsiAD(self.local(psi), y)
        return self.merged(y, psi.size)

    def residual(self, W):
        self.sol.updateOFFields(self.local(W))
        R = np.zeros(self.idx.size)
        self.sol.getResiduals(R)
        return self.merged(R, W.size)


CASES = {"channel_6": Plain, "channel_129": Plain, "channel_140": Plain, "passage_cyclic": Cyclic}
_REF = {}


def reference(name):
    """the case and its dense Jacobian diag(.) dR/dW diag(s) by central differences of the oracle's residual (cached per session)"""
    if name not in _REF:
        case = CASES[name](name)
        _REF[name] = (case, fd_jacobian(case.residual, case.W, case.scale))
    return _REF[name]


def fd_jacobian(residual, W, scale, h=FD_H):
    """column j: (R(W + h s_j e_j) - R(W - h s_j e_j)) / (2 h), divided by the step actually taken (W_j +- h s_j rounds)"""
    n = W.size
    J = np.empty((residual(W).size, n))
    Wp = W.copy()
    for j in range(n):
        Wp[j] = W[j] + h * scale[j]
        up = Wp[j]
        Rp = residual(Wp)
        Wp[j] = W[j] - h * scale[j]
        step = (up - Wp[j]) / scale[j]
        Rm = residual(Wp)
        Wp[j] = W[j]
        J[:, j] = (Rp - Rm) / step
    return J


def coupled_size(case, J, psi):
    """per entry j: sum of |psi_i| over the rows i of the cells coupled to the cell of j in J (any variable to any variable)"""
    from scipy.sparse import coo_matrix
    r, c = np.nonzero(J)
    C = coo_matrix((np.ones(r.size), (case.cell[r], case.cell[c])), shape=(case.nC, case.nC)).toarray() > 0
    pc = np.zeros(case.nC)
    np.add.at(pc, case.cell, np.abs(psi))
    return (C.T.astype(float) @ pc)[case.cell]


def entry_scale(case, J, psi, fd=False):
    """the size of entry j of J^T psi.  Exact products (fd False): sum_i |J_ij psi_i|, the terms that sum to the entry.  Central
    differences (fd True): the error of J_ij is roundoff of residual terms of the size of the row's and the column's largest entries,
    divided by the step, so the terms are taken at max(row max, column max).  Either way with a floor of FLOOR_REL |J|max times the
    psi of the coupled cells: residual rows that are zero up to roundoff (the z-momentum of a flow without z-velocity) sum terms of a
    few 1e-14 that the differences do not resolve."""
    A = np.abs(J)
    if fd:
        row, col = A.max(axis=1), A.max(axis=0)
        raw = ((J != 0.0) * np.maximum(row[:, None], col[None, :])).T @ np.abs(psi)
    else:
        raw = A.T @ np.abs(psi)
    return np.maximum(raw, FLOOR_REL * A.max() * coupled_size(case, J, psi))


def worst_entry(y, ref, scale):
    """(worst |y - ref| / scale, its index); an entry of a cell that no row of psi couples to (scale 0) must be exactly zero"""
    d = np.abs(y - ref)
    err = np.divide(d, scale, out=np.where(d > 0.0, np.inf, 0.0), where=scale > 0.0)
    j = int(np.argmax(err))
    return float(err[j]), j


def check_entries(case, y, ref, scale, tol, what):
    e, j = worst_entry(y, ref, scale)
    assert e <= tol, "%s: worst entry %s: %r vs %r (|diff| / term size %.2e > %.0e)" % (what, case.describe(j), y[j], ref[j], e, tol)
    return e


# ---- (a) state products --------------------------------------------------------------------------------------------------------
def check_fd_jacobian(name):
    """the finite-difference Jacobian itself against the oracle's exact forward tangent: a bad step would show here first"""
    case, J = reference(name)
    rng = np.random.default_rng(17)
    worst = 0.0
    for _ in range(2):
        v = rng.uniform(-1.0, 1.0, case.n)
        t = case.tangent(v)
        worst = max(worst, worst_entry(J @ v, t, entry_scale(case, J.T, v, fd=True))[0])
    print("\n%s: %d states; |J_fd v - J v| / (|J| |v|) %.2e" % (name, case.n, worst))
    assert worst <= TOL_FD_CHECK, (name, worst)


def check_state_product(name, lib_path):
    case, J = reference(name)
    eng = case.solver(lib_path)
    rng = np.random.default_rng(23)
    report = {}

    def compare(psi, what):
        y = eng.product(psi)
        y2 = eng.product(psi)
        assert np.array_equal(y, y2), "%s: the product is not bitwise reproducible" % what  # gathers, no atomics
        e_fd = check_entries(case, y, J.T @ psi, entry_scale(case, J, psi, fd=True), TOL_FD, what + " vs central differences")
        e_tp = check_entries(case, y, case.tape(psi), entry_scale(case, J, psi, fd=True), TOL_TAPE, what + " vs the oracle's tape")
        report[what] = (e_fd, e_tp)
        return y

    # random psi, and the dot-product identity with J v from the oracle's exact tangent and from the engine's own residual
    psi = rng.uniform(-1.0, 1.0, case.n)
    y = compare(psi, "random psi")
    v = rng.uniform(-1.0, 1.0, case.n)
    Jv = case.tangent(v)
    lhs, rhs = float(psi @ Jv), float(y @ v)
    size = float(np.abs(psi) @ np.abs(Jv))
    assert abs(lhs - rhs) <= TOL_DOT * size, ("<psi, J v> vs <J^T psi, v>", lhs, rhs, size)
    Rp = eng.residual(case.W + FD_H * case.scale * v)
    Rm = eng.residual(case.W - FD_H * case.scale * v)
    eng.residual(case.W)
    lhs_fd = float(psi @ (Rp - Rm)) / (2.0 * FD_H)
    assert abs(lhs_fd - rhs) <= TOL_DOT_FD * size, ("<psi, engine's J v> vs <J^T psi, v>", lhs_fd, rhs, size)

    # psi = e_i on every residual row of a cell next to each patch type, and on the phi row of its face on that patch
    nC = case.nC
    rows = case.boundary_rows()
    for t, (c, frow) in rows.items():
        for r in [3 * c, 3 * c + 1, 3 * c + 2, 3 * nC + c, 4 * nC + c, frow]:
            e = np.zeros(case.n)
            e[r] = 1.0
            compare(e, "psi = e_i on %s (next to %s)" % (case.describe(r), t))

    # psi on the cells without a boundary face (and their internal faces' phi rows) only
    if not case.cyclic:
        bcell = np.zeros(nC, dtype=bool)
        bcell[case.mesh.owner[case.mesh.n_internal_faces:]] = True
        if not bcell.all():
            inner = ~bcell[case.cell]
            nIF = case.mesh.n_internal_faces
            inner[5 * nC:] = False
            inner[5 * nC:5 * nC + nIF] = ~bcell[case.mesh.owner[:nIF]] & ~bcell[case.mesh.neighbour]
            psi = np.where(inner, rng.uniform(-1.0, 1.0, case.n), 0.0)
            compare(psi, "psi on interior cells only")
    worst_fd = max(v[0] for v in report.values())
    worst_tp = max(v[1] for v in report.values())
    print("\n%s (%s): %d probes; worst entry vs central differences %.2e, vs tape %.2e; dot-product identity %.1e (exact J v), %.1e (engine FD)"
          % (name, "host build" if lib_path else "CUDA", len(report), worst_fd, worst_tp, abs(lhs - rhs) / size, abs(lhs_fd - rhs) / size))
    return case, eng


# ---- (b) mesh products ---------------------------------------------------------------------------------------------------------
_REF_X = {}


def mesh_reference(name):
    """dense dR/dx_v by central differences of the oracle's residual on the moved mesh (wall distance frozen, as in the engine)"""
    if name not in _REF_X:
        case, _ = reference(name)
        mesh = case.mesh
        yw = case.orc.geometry("yWall")
        pts = mesh.points.ravel().copy()
        J = np.empty((case.n, pts.size))

        def res(p):
            m = cases.PolyMesh(p.reshape(-1, 3), mesh.faces, mesh.owner, mesh.neighbour, mesh.patches)
            return Oracle(m, case.bcs, normalizeStates=NORM_STATES, divU=DIV_U, normalizeResiduals=ALL_RES, yWall=yw).residual(case.W)

        for k in range(pts.size):
            q = pts.copy()
            q[k] = pts[k] + FD_H
            up = q[k]
            Rp = res(q)
            q[k] = pts[k] - FD_H
            Rm = res(q)
            J[:, k] = (Rp - Rm) / (up - q[k])
        _REF_X[name] = J
    return _REF_X[name]


def mesh_scale(Jx, psi):
    """entry_scale(fd=True) of a product over the mesh points (columns are point coordinates, not states): the floor is taken
    over the whole Jacobian"""
    A = np.abs(Jx)
    row, col = A.max(axis=1), A.max(axis=0)
    raw = ((Jx != 0.0) * np.maximum(row[:, None], col[None, :])).T @ np.abs(psi)
    return np.maximum(raw, FLOOR_REL * A.max() * np.abs(psi).max())


def check_mesh_product(name, lib_path):
    case, _ = reference(name)
    Jx = mesh_reference(name)
    eng = case.solver(lib_path)
    sol = eng.sol
    nP3 = 3 * sol.getNLocalPoints()
    assert nP3 == Jx.shape[1]
    pts = np.zeros(nP3)
    sol.getOFMeshPoints(pts)
    rng = np.random.default_rng(29)
    probes = {"random psi": rng.uniform(-1.0, 1.0, case.n)}
    nC = case.nC
    for t, (c, frow) in case.boundary_rows().items():
        for r in (3 * c, 3 * nC + c, frow):
            e = np.zeros(case.n)
            e[r] = 1.0
            probes["psi = e_i on %s (next to %s)" % (case.describe(r), t)] = e
    # the tape through the geometry checks the difference step (away from the symmetry planes' normal component, where the tape
    # takes the one-sided derivative of |n_z| and central differences the symmetric one)
    sym = np.zeros((nP3 // 3, 3), dtype=bool)
    for p in case.mesh.patches:
        if p["type"] == "symmetry":
            fp = case.mesh.faces[p["start"]:p["start"] + p["size"]]
            sym[np.unique(fp[fp >= 0]), 2] = True
    sym = sym.ravel()
    worst = 0.0
    for what, psi in probes.items():
        prod = np.zeros(nP3)
        sol.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", psi, prod)
        sc = mesh_scale(Jx, psi)
        ref = Jx.T @ psi
        if what == "random psi":
            tp = case.orc.jtvec_xv(case.W, psi)
            e_tp = np.abs(ref - tp)[~sym].max() / np.abs(tp).max()
            assert e_tp <= TOL_FD_CHECK, ("central-difference dR/dx_v vs the tape", e_tp)
            print("central-difference dR/dx_v vs the tape: %.2e of the largest entry" % e_tp)
        e, j = worst_entry(prod, ref, sc)
        assert e <= TOL_X, "%s: worst point coordinate %d (point %d, %s): %r vs %r (%.2e)" % (what, j, j // 3, "xyz"[j % 3], prod[j], ref[j], e)
        worst = max(worst, e)
    print("\n%s (%s): volCoord product, %d probes; worst entry vs central differences %.2e" % (name, "host build" if lib_path else "CUDA",
                                                                                          len(probes), worst))


# ---- (c) partitions ------------------------------------------------------------------------------------------------------------
def partition_probes(case, rng):
    """random psi and e_i on the rows of cells next to each patch type (the coupled pair's two sides on the passage)"""
    P = [rng.uniform(-1.0, 1.0, case.n)]
    for t, (c, frow) in case.boundary_rows().items():
        for r in (3 * c, 3 * case.nC + c, 4 * case.nC + c, frow):
            e = np.zeros(case.n)
            e[r] = 1.0
            P.append(e)
    return np.array(P)


def run_partitioned(name, nproc, port, lib_kind):
    case, J = reference(name)
    if case.cyclic:
        d = case.P.case_dir
    else:
        d = tempfile.mkdtemp(prefix="dab_prod_mp_")
        case.write(d)
    psi = partition_probes(case, np.random.default_rng(31))
    data = dict(W=case.W, psi=psi, ref=psi @ J, scale=np.array([entry_scale(case, J, p, fd=True) for p in psi]))
    if not case.cyclic:
        Jx = mesh_reference(name)
        data.update(ref_x=psi @ Jx, scale_x=np.array([mesh_scale(Jx, p) for p in psi]))
    np.savez(os.path.join(d, "products.npz"), **data)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % nproc, "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.abspath(__file__), d, name, lib_kind]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, OMP_NUM_THREADS="1"), cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert r.stdout.count(" ok: ") == nproc, r.stdout
    print("\n" + r.stdout.strip())


def describe_global(j, nC):
    if j < 5 * nC:
        return "%s of cell %d" % ((["Ux", "Uy", "Uz"][j % 3] if j < 3 * nC else "p" if j < 4 * nC else "nuTilda"), j // 3 if j < 3 * nC else j % nC)
    return "phi of face %d" % (j - 5 * nC)


def worker(case_dir, name, lib_kind):
    import torch
    import torch.distributed as dist
    from dafoam_b200.pyDASolvers import set_comm_callbacks
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    cuda = lib_kind == "cuda"
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
    data = np.load(os.path.join(case_dir, "products.npz"))
    dev = rank if cuda else 0
    one = pyDASolvers("DASimpleFoam -python", dict(ENGINE_OPTS), caseDir=case_dir, device=dev, _lib_path=lib)
    par = pyDASolvers("DASimpleFoam -python", dict(ENGINE_OPTS), caseDir=case_dir, device=dev, rank=rank, nRanks=world, ncclUniqueId=uid,
                      _lib_path=lib)
    nCg = one.getNGlobalCells()
    nFg = int(one.getLocalToGlobal("faces").max()) + 1
    n = 5 * nCg + nFg

    def maps(sol):
        idx = sol.localStateIndex(nCg, nFg)
        owned = np.concatenate([np.ones(5 * sol.getNLocalCells(), dtype=bool), sol.getLocalToGlobal("faceOwned").astype(bool)])
        return Engine(sol, idx, owned)

    e1, e2 = maps(one), maps(par)
    W = data["W"]
    assert W.size == n
    one.updateOFFields(e1.local(W))
    par.updateOFFields(e2.local(W))

    def gathered(v):
        t = torch.from_numpy(v.copy())
        dist.all_reduce(t)
        return t.numpy()

    worst_one = worst_ref = worst_x = 0.0
    for m, psi in enumerate(data["psi"]):
        y1 = e1.product(psi)
        x2 = e2.local(psi)
        x2[~e2.owned] = 0.0
        yl = np.zeros(e2.idx.size)
        par.calcdRdWTPsiAD(x2, yl)
        assert np.all(yl[~e2.owned] == 0.0), "probe %d: foreign slots must be structural zeros" % m
        y2 = gathered(e2.merged(yl, n))
        sc = data["scale"][m]
        for ref, tol, what in ((y1, TOL_PART, "one partition"), (data["ref"][m], TOL_FD, "central differences")):
            e, j = worst_entry(y2, ref, sc)
            assert e <= tol, "rank %d, probe %d: %d partitions vs %s: entry %d (%s): %r vs %r (%.2e)" % (
                rank, m, world, what, j, describe_global(j, nCg), y2[j], ref[j], e)
            if what == "one partition":
                worst_one = max(worst_one, e)
            else:
                worst_ref = max(worst_ref, e)
    pts = np.zeros(3 * one.getNLocalPoints())
    one.getOFMeshPoints(pts)
    for m, psi in enumerate(data["psi"]):
        p1, p2 = np.zeros(pts.size), np.zeros(pts.size)
        x1 = e1.local(psi)
        x1[~e1.owned] = 0.0
        one.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", x1, p1)
        x2 = e2.local(psi)
        x2[~e2.owned] = 0.0
        par.calcJacTVecProduct("x", "volCoord", pts, "R", "residual", x2, p2)
        s2 = gathered(p2)
        # each partition returns the contribution of its own rows over the full point list: their sum is the one-partition product
        big = max(np.abs(p1).max(), 1e-300)
        e = np.abs(s2 - p1).max() / big
        assert e <= TOL_PART_X, ("volCoord: %d partitions vs one" % world, m, e)
        worst_x = max(worst_x, e)
        if "ref_x" in data:
            ex, j = worst_entry(s2, data["ref_x"][m], data["scale_x"][m])
            assert ex <= TOL_X, ("volCoord: %d partitions vs central differences" % world, m, j, ex)
    print("rank %d ok: %d probes; worst entry vs one partition %.1e, vs central differences %.1e; volCoord vs one partition %.1e"
          % (rank, len(data["psi"]), worst_one, worst_ref, worst_x), flush=True)
    dist.barrier()
    dist.destroy_process_group()


# ---- tests ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_fd_jacobian_matches_forward_tangent(name):
    check_fd_jacobian(name)


@pytest.mark.parametrize("name", list(CASES))
def test_state_product_entries_host_build(name):
    check_state_product(name, HOSTSIM)


@pytest.mark.parametrize("name", ["channel_6", "channel_140"])
def test_mesh_product_entries_host_build(name):
    check_mesh_product(name, HOSTSIM)


@pytest.mark.parametrize("name,nproc,port", [("channel_140", 2, 29801), ("channel_140", 3, 29803), ("passage_cyclic", 2, 29805)])
def test_partitioned_products_host_build(name, nproc, port):
    run_partitioned(name, nproc, port, "host")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_state_product_entries_cuda(name):
    check_state_product(name, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["channel_6", "channel_140"])
def test_mesh_product_entries_cuda(name):
    check_mesh_product(name, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name,nproc,port", [("channel_140", 2, 29811), ("channel_140", 3, 29813), ("passage_cyclic", 2, 29815)])
def test_partitioned_products_cuda(name, nproc, port):
    import torch
    if torch.cuda.device_count() < nproc:
        # the CUDA build exchanges halos through NCCL, which takes one device per rank; the same partitioned kernels run as
        # several partitions on one machine in test_partitioned_products_host_build
        pytest.skip("%d partitions of the CUDA build need %d GPUs (NCCL: one device per rank)" % (nproc, nproc))
    run_partitioned(name, nproc, port, "cuda")


if __name__ == "__main__":
    worker(sys.argv[1], sys.argv[2], sys.argv[3])
