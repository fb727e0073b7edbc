"""The compressible transpose product y = diag(s) [dR/dW]^T psi (calcdRdWTPsiAD of DARhoSimpleFoam, DARhoSimpleCFoam and DATurboFoam:
the reverse sweep cRevA / cRevB / cRevE / cRevC of comp_rev_kernels.hpp) checked entry by entry, not through segment norms:
  (a) against the dense Jacobian J taken column by column from the oracle's forward-mode dual numbers (Oracle.jvec, exact), and
      against the oracle's tape (Oracle.jtvec) as a second witness;
  (b) through the dot-product identity <psi, J v> = <J^T psi, v>, with J v from the oracle's tangent and from central differences
      of the engine's own residual (the reverse sweep tied to the engine's forward, independent of the oracle);
  (c) as an operator: bitwise reproducible (gathers, no atomics), linear, and the same with the rolled face loops (DAB_NOHEX6=1)
      as with the unrolled six-face loops of a hex mesh;
  (d) on 2 and 3 partitions and on a cyclic passage cut between two (the T and nuTilda halos, the exchanges between cRevE and
      cRevC), gathered and compared with one partition and with J;
  (e) the function path: [dF/dW] of a force and a moment, seeded into the work arrays and finished by cRevC, against
      Oracle.dforce_dw;
  (f) a 33 792-cell O-grid against the tape (no dense J at that size): thousands of CTAs.
The state layout is [U | p | T | nuTilda | phi] and s_j = (U_ref, 101325, 300, 1e-3, |Sf|): the engine's normalizeStates, times
the face area for phi.  The probes: random psi, the constant psi = 1e-3, psi = e_i on every row of a cell next to each patch type
and on the phi row of its face on that patch, and psi on cells without a boundary face.

Shapes: the product's kernels run one cell per thread in 128-thread CTAs; the channels have 6 cells (fewer boundary faces than a
warp), 129 cells (one CTA plus one) and 140 cells (7 x 5 x 4, with interior cells); they and the O-grids are hex meshes (the
unrolled NF=6 face loops), the prism channel (130 cells, five faces per cell) takes the rolled NF=0 loops.  The physics is spread
over the cases: internal energy and enthalpy, constant and Sutherland viscosity, SA and SA-fv3, every div(phi,U) and div(phi,e|h)
scheme, the Spalding wall function, a wall with fixedValue T, an MRF zone with rotating-wall and relative-flux faces, the transonic
pressure equation with limitedLinear 1.0 / 0.5, and a DATurboFoam cyclic passage.

Every reference is plain numpy around the oracle (oracle/oracle.cpp); none of it goes through the engine's kernels.  The file is
also the worker of the partitioned cases: `python -m torch.distributed.run ... tests/test_compressible_products.py <case dir>
<name> <host|cuda>`."""
import contextlib
import json
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
from tests.common import HOSTSIM, mrf_zone  # noqa: E402
from tests.test_adjoint_products import Engine, check_entries, entry_scale, worst_entry  # noqa: E402

# ---- steps and tolerances ----------------------------------------------------------------------------------------------------
# Entry errors are |y_j - ref_j| / scale_j with scale_j = entry_scale(fd=True) of tests/test_adjoint_products.py: the sum over the
# rows of psi of |psi_i| times max(row max, column max) of J, floored at 1e-9 |J|max times the psi of the coupled cells.  Scaled by
# |J_ij| alone, entries such as d(TRes)/dp with internal energy (p/rho = RT cancels terms ~1e5 times the entry) differ between the
# tape and the dual numbers by 1e-10 of themselves; without the floor, 1e-14 ... 1e-20 roundoff of the dual numbers stands against
# the engine's exact zeros.  An entry of a cell that no row of psi couples to must be exactly zero.
#
# This scale is generous: the row and column maxima of J are dominated by the pressure and energy rows, so a single term missed or
# counted twice moves its entry by far less than O(1) of it.  Measured on the host build, worst entry over the scale across all
# probes, for single-term mistakes planted in comp_rev_kernels.hpp (the smallest and largest case; "-" where the term does not enter):
#   mistake                                               worst entry / scale            <psi, J v> vs <y, v> (see TOL_DOT)
#   drop `ba.sngT -= heA qc aE |S|` (cRevE)               1.2e-8 (transonic) ... 8.6e-5  1e-10 ... 6e-6
#   flip the sign of the Coriolis rho term (cRevA)        3.6e-4 ... 1.8e-3 (MRF cases)  2e-6 ... 5e-6
#   wc for wn in cRevB's muEff interpolation              5.2e-8 (channel_140) ... 5.5e-6 4e-12 ... 2e-10
#   skip the dLimDr block (cRevA)                         3.9e-3 ... 3.2e-2 (transonic)  5e-8 ... 1e-7
#   drop d(nut_b)/d(nu_b) of a `calculated` nut           2.9e-10 (naca_wf) ... 2.6e-7   2e-13 ... 3e-9
#   drop d(nut_b)/d(nu_b) of the Spalding wall function   1.1e-6 (naca_wf only)          3e-9
#   drop the second term of dmuSutherland                 4.3e-9 (naca_wf) ... 1.9e-7    2e-9 ... 8e-9
# Every mistake exceeds the host tolerances below on at least one case, most on several; the dot-product identity (noise 1.2e-15,
# tolerance 1e-13) catches each one too, on most cases it enters (it misses the calculated-nut term on the transonic cases, 3e-14).  So the tolerances sit a few times above
# the measured roundoff and no further: loosening them hides real mistakes.  Measured on the host build (x86-64, no FMA contraction) over every
# probe and case:
TOL_J = 3e-9         # product vs J^T psi (J from the oracle's dual numbers): both exact float64, different operation orders; measured
#                      6.9e-10: d(TRes)/d(phi) of an outflow face of channel_6 (internal energy), where Ek_b - Ek_c carries
#                      p_b/rho_b - p_c/rho_c = R (T_b - T_c) = 0: the engine sums terms of ~1e5 to 2e-11, the oracle gets an exact zero
TOL_TAPE = 3e-9      # product vs the oracle's tape; measured 6.9e-10 (the same entry)
TOL_DOT = 1e-13      # <psi, J v> (dual numbers) vs <y, v>, relative to sum |psi_i (J v)_i|; measured 1.2e-15 (1.2e-15 on the H100)
FD_H = 1e-6          # central-difference step of the engine's residual, relative to s_j
TOL_DOT_FD = 1e-9    # the same with J v from the engine's residual (step FD_H): roundoff of rows that sum pressures of 1e5, over
#                      the step; measured 8.9e-11
TOL_LINEAR = 1e-12   # y(2a - 3b) vs 2 y(a) - 3 y(b), per entry of the entry scale; measured 8.4e-17
TOL_PART = 1e-12     # several partitions vs one: halo copies are exact, a cut face is evaluated from the other side (the same terms
#                      in another order); measured 2.4e-16
TOL_F = 1e-11        # dF/dW vs Oracle.dforce_dw per entry, relative to max(|entry|, FLOOR_F of the largest); measured 2.7e-13
FLOOR_F = 1e-9
# CUDA: nvcc contracts a*b + c into fused multiply-adds, which changes the rounding of every term, and the terms of an entry
# cancel: the energy and pressure rows carry p ~ 1e5, rho*T and p/rho products whose sums are 1e4 ... 1e5 times the entry, and
# the entries at the floor (1e-9 |J|max) see the roundoff of their row's largest terms.  Measured on an H100 80GB HBM3 (700 W
# power limit):
TOL_J_CUDA = 1.5e-8  # product vs dual numbers / tape; measured 4.6e-9 (channel_6, the outflow entry of TOL_J above), 2.5e-9
#                      (naca_wf), 6.5e-10 (channel_140), 3.9e-10 (transonic), below 1e-11 elsewhere.  Three times the worst: the
#                      planted mistakes above still fail on the channels (sngT, muEff, calculated nut, Sutherland) and on naca_wf
#                      (sngT 4.7e-8, wall function); the dot-product identity keeps its host tolerance.
TOL_F_CUDA = 1e-10   # dF/dW; measured 6.7e-13
TOL_HEX_CUDA = 1e-12  # rolled vs unrolled face loops: contraction may differ between the two instantiations; measured 1.2e-19


# ---- cases ---------------------------------------------------------------------------------------------------------------------
NRES = ("URes", "pRes", "TRes", "nuTildaRes", "phiRes")
PATCH_TYPE = {"inlet": "inlet", "outlet": "outlet (inletOutlet)", "walls": "wall", "sym1": "symmetry", "sym2": "symmetry",
              "wing": "wall", "inout": "farfield (inletOutlet / outletInlet)", "hub": "wall", "shroud": "wall", "per_lo": "cyclic",
              "per_hi": "cyclic"}
TRANSONIC = {"upwind": 0, "linear": 2, "limitedLinear": 4}

# mesh, solver, energy, transport, RAS model, div(phi,U), div(phi,e|h); optional: wall function, fixedValue T on the walls, MRF
# zone, transonic limitedLinear k
SPECS = {
    "channel_6": dict(mesh=lambda: cases.channel(nx=3, ny=2, nz=1), solver="DARhoSimpleFoam", energy="sensibleInternalEnergy",
                      transport="const", ras="SpalartAllmaras", divU="upwind", divE="upwind"),
    "channel_129": dict(mesh=lambda: cases.channel(nx=43, ny=3, nz=1), solver="DARhoSimpleFoam", energy="sensibleEnthalpy",
                        transport="sutherland", ras="SpalartAllmarasFv3", divU="linear", divE="linear"),
    "channel_140": dict(mesh=lambda: cases.channel(nx=7, ny=5, nz=4), solver="DARhoSimpleFoam", energy="sensibleInternalEnergy",
                        transport="sutherland", ras="SpalartAllmaras", divU="linearUpwind", divE="linearUpwind"),
    "prism_130": dict(mesh=lambda: cases.prism_channel(nx=13, ny=5), solver="DARhoSimpleFoam", energy="sensibleEnthalpy",
                      transport="const", ras="SpalartAllmarasFv3", divU="linearUpwindV", divE="upwind"),
    "channel_wallT": dict(mesh=lambda: cases.channel(nx=9, ny=4, nz=1), solver="DARhoSimpleFoam", energy="sensibleEnthalpy",
                          transport="sutherland", ras="SpalartAllmaras", divU="linearUpwindV", divE="linearUpwind", wallT=320.0),
    "naca_wf": dict(mesh=lambda: cases.naca0012_ogrid(ni=12, nj=6, nk=1), solver="DARhoSimpleFoam", energy="sensibleInternalEnergy",
                    transport="sutherland", ras="SpalartAllmarasFv3", divU="linearUpwindV", divE="linearUpwind", wf=True),
    "naca_mrf_turbo": dict(mesh=lambda: cases.naca0012_ogrid(ni=12, nj=6, nk=1), solver="DATurboFoam", energy="sensibleEnthalpy",
                           transport="const", ras="SpalartAllmaras", divU="linearUpwindV", divE="upwind", mrf=40.0),
    "transonic_ll1": dict(mesh=lambda: cases.naca0012_ogrid(ni=12, nj=6, nk=1), solver="DARhoSimpleCFoam", energy="sensibleInternalEnergy",
                          transport="const", ras="SpalartAllmaras", divU="linearUpwindV", divE="upwind", transonic=1.0),
    "transonic_ll05": dict(mesh=lambda: cases.naca0012_ogrid(ni=12, nj=6, nk=1), solver="DARhoSimpleCFoam", energy="sensibleInternalEnergy",
                           transport="const", ras="SpalartAllmaras", divU="linearUpwindV", divE="upwind", transonic=0.5),
    "transonic_turbo_mrf": dict(mesh=lambda: cases.naca0012_ogrid(ni=12, nj=6, nk=1), solver="DATurboFoam", energy="sensibleEnthalpy",
                                transport="const", ras="SpalartAllmaras", divU="linearUpwindV", divE="upwind", transonic=0.5, mrf=40.0),
}


def kinds_of(n_cells, n_dof):
    k = np.empty(n_dof, dtype=object)
    k[:3 * n_cells] = ["Ux", "Uy", "Uz"] * n_cells
    for i, name in enumerate(("p", "T", "nuTilda")):
        k[(3 + i) * n_cells:(4 + i) * n_cells] = name
    k[6 * n_cells:] = "phi"
    return k


def state_scales(n_cells, magSf, ns):
    """s_j: the engine's state scaling (normalizeStates; phi also times |Sf|)"""
    return np.concatenate([np.full(3 * n_cells, ns["U"]), np.full(n_cells, ns["p"]), np.full(n_cells, ns["T"]),
                           np.full(n_cells, ns["nuTilda"]), ns["phi"] * magSf])


def norm_states(U_ref):
    return dict(U=float(U_ref), p=101325.0, T=300.0, nuTilda=1e-3, phi=1.0)


class Plain:
    """a mesh without cyclic patches: the engine's single-partition numbering is the polyMesh one, the oracle's too"""
    cyclic = False

    def __init__(self, name):
        self.name = name
        sp = self.spec = SPECS[name]
        self.mesh = mesh = sp["mesh"]()
        naca = any(p["name"] == "wing" for p in mesh.patches)
        self.U0 = U0 = (230.0, 8.0, 0.0) if "transonic" in sp else (50.0, 2.0, 0.0)
        base = cases.default_bcs_naca(U0=U0, wall_function=sp.get("wf", False)) if naca else cases.default_bcs_channel(U0=U0)
        self.bcs = cases.compressible_bcs(base)
        if "wallT" in sp:  # a heated wall: compressible_bcs gives walls a zeroGradient T
            self.bcs["T"][3]["walls"] = dict(type="fixedValue", value=sp["wallT"])
        self.thermo = cases.default_thermo(energy=sp["energy"], transport=sp["transport"], divE=sp["divE"],
                                           divEkp="linear" if sp["divE"] == "linear" else "upwind")
        self.ns = norm_states(U0[0])
        self.orc = orc = Oracle(mesh, self.bcs, normalizeStates=self.ns, normalizeResiduals=NRES, thermo=self.thermo, rasModel=sp["ras"],
                                divU=sp["divU"])
        orc.set_turbo(sp["solver"] == "DATurboFoam")
        if "transonic" in sp:
            orc.set_transonic(True, TRANSONIC["limitedLinear"], sp["transonic"], -1)
        self.mrf = None
        if "mrf" in sp:
            self.mrf = mrf_zone(mesh, omega=sp["mrf"])
            orc.set_mrf(mesh, self.mrf)
        self.nC = mesh.n_cells
        self.n = orc.ndof
        assert self.n == 6 * self.nC + mesh.n_faces
        self.W = synthetic_state(mesh, orc.geometry("C"), orc.geometry("Sf"), U0=U0, thermo=self.thermo)
        self.scale = state_scales(self.nC, orc.geometry("magSf"), self.ns)
        self.kinds = kinds_of(self.nC, self.n)
        self.cell = np.concatenate([np.repeat(np.arange(self.nC), 3)] + [np.arange(self.nC)] * 3 + [mesh.owner])
        self.face_patch = [""] * mesh.n_internal_faces
        for p in mesh.patches:
            self.face_patch += [p["name"]] * p["size"]
        self.options = dict(normalizeStates=self.ns, normalizeResiduals=list(NRES))

    def write(self, d):
        sp = self.spec
        div_u = "bounded Gauss %s%s" % (sp["divU"], " grad(U)" if sp["divU"].startswith("linearUpwind") else "")
        kw = dict(thermo=self.thermo, ras_model=sp["ras"])
        if self.mrf is not None:
            kw["mrf"] = self.mrf
        if "transonic" in sp:
            # DARhoSimpleCFoam is transonic whatever fvSolution says; DATurboFoam reads SIMPLE { transonic yes; }
            kw.update(transonic=sp["solver"] == "DATurboFoam", div_phid_p="Gauss limitedLinear %g" % sp["transonic"])
        cases.write_case(d, self.mesh, self.bcs, div_u=div_u, **kw)

    def solver(self, lib_path, nohex6=False):
        d = tempfile.mkdtemp(prefix="dab_cprod_")
        self.write(d)
        sol = make_solver(self.spec["solver"], self.options, d, lib_path, nohex6=nohex6)
        sol.updateOFFields(self.W)
        return Engine(sol, np.arange(self.n), np.ones(self.n, dtype=bool))

    def tangent(self, v):
        """J v in scaled states: the oracle's forward-mode dual numbers"""
        return self.orc.jvec(self.W, self.scale * v)

    def tape(self, psi):
        self.orc.record(self.W)  # one tape per process: another case's oracle may have recorded since
        return self.orc.jtvec(psi)

    def boundary_rows(self):
        """patch type -> (cell, phi row of one of its faces on that patch): the face in the middle of the first patch of each type,
        and on a patch that switches between inflow and outflow (inletOutlet / outletInlet) one face of each direction"""
        out = {}
        nC = self.nC
        for p in self.mesh.patches:
            t = PATCH_TYPE[p["name"]]
            faces = np.arange(p["start"], p["start"] + p["size"])
            phi = self.W[6 * nC + faces]
            if "inletOutlet" in t:
                for what, sel in (("inflow", phi < 0.0), ("outflow", phi > 0.0)):
                    if sel.any():
                        f = int(faces[sel][sel.sum() // 2])
                        out.setdefault("%s, %s face" % (t, what), (int(self.mesh.owner[f]), 6 * nC + f))
            elif t not in out:
                f = int(faces[p["size"] // 2])
                out[t] = (int(self.mesh.owner[f]), 6 * nC + f)
        return out

    def interior_psi(self, rng):
        """psi on the cells without a boundary face and the phi rows of the faces between them, or None"""
        nC, nIF = self.nC, self.mesh.n_internal_faces
        bcell = np.zeros(nC, dtype=bool)
        bcell[self.mesh.owner[nIF:]] = True
        if bcell.all():
            return None
        inner = ~bcell[self.cell]
        inner[6 * nC:] = False
        inner[6 * nC:6 * nC + nIF] = ~bcell[self.mesh.owner[:nIF]] & ~bcell[self.mesh.neighbour]
        return np.where(inner, rng.uniform(-1.0, 1.0, self.n), 0.0)

    def describe(self, j):
        if j < 6 * self.nC:
            return "%s of cell %d" % (self.kinds[j], self.cell[j])
        f = j - 6 * self.nC
        return "phi of face %d (%s, owner cell %d)" % (f, self.face_patch[f] or "internal", self.cell[j])


class Cyclic:
    """DATurboFoam on the annular passage with cyclic sides and an MRF zone over every cell (tests/test_cyclic.py Pair): the engine
    on one passage, its reference the oracle on the closed ring of passages with a passage-periodic state; vectors in the engine's
    merged numbering (one face per coupled pair)"""
    cyclic = True
    SOLVER = "DATurboFoam"

    def __init__(self, name, lib_path=HOSTSIM):
        from tests.test_cyclic import merged_faces
        self.name = name
        self.P = P = self.pair(lib_path)
        self.nC, self.n = P.nCs, P.n_sec()
        self.W = P.state()
        self.Wr = P.to_ring(self.W)
        self.ns = norm_states(50.0)
        magSf = np.asarray(P.orc.geometry("magSf"))[P.s2f]
        self.scale = state_scales(self.nC, magSf, self.ns)
        self.kinds = kinds_of(self.nC, self.n)
        self.so, self.sn, self.pname = merged_faces(P.sec)
        self.cell = np.concatenate([np.repeat(np.arange(self.nC), 3)] + [np.arange(self.nC)] * 3 + [self.so])
        self.options = dict(normalizeStates=self.ns, normalizeResiduals=list(NRES))

    @classmethod
    def pair(cls, lib_path):
        from tests.test_cyclic import Pair
        return Pair(True, "linearUpwind", lib_path=lib_path, solver=cls.SOLVER, mrf_omega=300.0)

    def solver(self, lib_path, nohex6=False):
        if lib_path == HOSTSIM and not nohex6:
            P = self.P
        else:
            with rolled_face_loops(nohex6):
                P = self.pair(lib_path)
        P.sol.updateOFFields(P.local(self.W))
        return Engine(P.sol, P.idx, P.owned)

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
        out["cyclic (per_lo side)"] = (int(self.so[g]), 6 * self.nC + g)
        out["cyclic (per_hi side)"] = (int(self.sn[g]), 6 * self.nC + g)
        for g in range(nIF, len(self.so)):
            if self.sn[g] < 0 and self.pname[g] not in out:
                out[self.pname[g]] = (int(self.so[g]), 6 * self.nC + g)
        return out

    def interior_psi(self, rng):
        return None  # every cell of the 4 x 4 x 6 passage touches a wall, a cyclic side, the inlet or the outlet

    def describe(self, j):
        if j < 6 * self.nC:
            return "%s of cell %d" % (self.kinds[j], self.cell[j])
        g = j - 6 * self.nC
        what = "coupled" if self.sn[g] >= 0 and g >= self.P.sec.n_internal_faces else (self.pname[g] or "internal")
        return "phi of face %d (%s, owner cell %d)" % (g, what, self.cell[j])


@contextlib.contextmanager
def rolled_face_loops(on):
    """DAB_NOHEX6=1 while a solver is constructed: it reads the variable once, when it uploads its mesh, and then runs the rolled
    face loops (NF=0) even on a hex mesh"""
    prev = os.environ.get("DAB_NOHEX6")
    if on:
        os.environ["DAB_NOHEX6"] = "1"
    try:
        yield
    finally:
        if on and prev is None:
            del os.environ["DAB_NOHEX6"]
        elif on:
            os.environ["DAB_NOHEX6"] = prev


def make_solver(solver, options, case_dir, lib_path, nohex6=False, **kw):
    with rolled_face_loops(nohex6):
        return pyDASolvers("%s -python" % solver, dict(options), caseDir=case_dir, _lib_path=lib_path, **kw)


CASES = {name: Plain for name in SPECS}
CASES["passage_cyclic"] = Cyclic
_REF = {}


def reference(name):
    """the case and its dense Jacobian diag(.) dR/dW diag(s) from the oracle's dual numbers, one column per state (cached per
    session)"""
    if name not in _REF:
        case = CASES[name](name)
        J = np.empty((case.n, case.n))
        e = np.zeros(case.n)
        for j in range(case.n):
            e[j] = 1.0
            J[:, j] = case.tangent(e)
            e[j] = 0.0
        _REF[name] = (case, J)
    return _REF[name]


# ---- (a)-(c) state products ----------------------------------------------------------------------------------------------------
def probes(case, rng):
    """what -> psi"""
    out = {"random psi": rng.uniform(-1.0, 1.0, case.n), "psi = 1e-3": np.full(case.n, 1e-3)}
    nC = case.nC
    for t, (c, frow) in case.boundary_rows().items():
        for r in [3 * c, 3 * c + 1, 3 * c + 2, 3 * nC + c, 4 * nC + c, 5 * nC + c, frow]:
            e = np.zeros(case.n)
            e[r] = 1.0
            out["psi = e_i on %s (next to %s)" % (case.describe(r), t)] = e
    inner = case.interior_psi(rng)
    if inner is not None:
        out["psi on interior cells only"] = inner
    return out


def check_state_product(name, lib_path):
    case, J = reference(name)
    eng = case.solver(lib_path)
    # the prism channel runs the rolled face loops (NF=0), every other case the unrolled six-face loops (NF=6)
    assert eng.sol.getFaceLoopWidth() == (0 if name == "prism_130" else 6), (name, eng.sol.getFaceLoopWidth())
    cuda = lib_path is None
    tol_j, tol_tp = (TOL_J_CUDA, TOL_J_CUDA) if cuda else (TOL_J, TOL_TAPE)
    rng = np.random.default_rng(23)
    worst_j = worst_tp = 0.0
    P = probes(case, rng)
    for what, psi in P.items():
        y = eng.product(psi)
        assert np.array_equal(y, eng.product(psi)), "%s: the product is not bitwise reproducible" % what  # gathers, no atomics
        sc = entry_scale(case, J, psi, fd=True)
        worst_j = max(worst_j, check_entries(case, y, J.T @ psi, sc, tol_j, "%s: %s vs the oracle's dual numbers" % (name, what)))
        worst_tp = max(worst_tp, check_entries(case, y, case.tape(psi), sc, tol_tp, "%s: %s vs the oracle's tape" % (name, what)))

    # the dot-product identity, with J v from the oracle's dual numbers and from the engine's own residual
    psi, v = rng.uniform(-1.0, 1.0, case.n), rng.uniform(-1.0, 1.0, case.n)
    y = eng.product(psi)
    Jv = case.tangent(v)
    lhs, rhs = float(psi @ Jv), float(y @ v)
    size = float(np.abs(psi) @ np.abs(Jv))
    e_dot = abs(lhs - rhs) / size
    assert e_dot <= TOL_DOT, ("<psi, J v> vs <J^T psi, v>", lhs, rhs, size)
    Rp = eng.residual(case.W + FD_H * case.scale * v)
    Rm = eng.residual(case.W - FD_H * case.scale * v)
    eng.residual(case.W)
    e_fd = abs(float(psi @ (Rp - Rm)) / (2.0 * FD_H) - rhs) / size
    assert e_fd <= TOL_DOT_FD, ("<psi, engine's J v> vs <J^T psi, v>", e_fd)

    # linearity, per entry
    a, b = rng.uniform(-1.0, 1.0, case.n), rng.uniform(-1.0, 1.0, case.n)
    ya, yb, yab = eng.product(a), eng.product(b), eng.product(2.0 * a - 3.0 * b)
    e_lin = check_entries(case, yab, 2.0 * ya - 3.0 * yb, 2.0 * entry_scale(case, J, a, fd=True) + 3.0 * entry_scale(case, J, b, fd=True),
                          TOL_LINEAR, "%s: y(2a - 3b) vs 2 y(a) - 3 y(b)" % name)
    print("\n%s (%s): %d states, %d probes; worst entry vs dual numbers %.2e, vs tape %.2e; dot-product identity %.1e (dual numbers), "
          "%.1e (engine FD); linearity %.1e" % (name, "CUDA" if cuda else "host build", case.n, len(P), worst_j, worst_tp, e_dot, e_fd, e_lin))
    return case, J, eng, P


def check_rolled_loops(name, lib_path):
    """DAB_NOHEX6=1: the same product from the rolled face loops (NF=0) as from the unrolled six-face loops (NF=6) of a hex mesh"""
    case, J = reference(name)
    e6, e0 = case.solver(lib_path), case.solver(lib_path, nohex6=True)
    # otherwise the comparison is of the rolled loops with themselves
    assert e6.sol.getFaceLoopWidth() == 6 and e0.sol.getFaceLoopWidth() == 0, (name, e6.sol.getFaceLoopWidth(), e0.sol.getFaceLoopWidth())
    rng = np.random.default_rng(41)
    worst = 0.0
    for what, psi in probes(case, rng).items():
        y6, y0 = e6.product(psi), e0.product(psi)
        if lib_path is not None:
            assert np.array_equal(y6, y0), "%s: %s: the rolled and unrolled face loops differ on the host build" % (name, what)
        else:
            worst = max(worst, check_entries(case, y0, y6, entry_scale(case, J, psi, fd=True), TOL_HEX_CUDA,
                                             "%s: %s: rolled vs unrolled face loops" % (name, what)))
    print("\n%s (%s): rolled vs unrolled face loops, worst entry %.1e" % (name, "CUDA" if lib_path is None else "host build", worst))


def limiter_fractions(case):
    """the limitedLinear limiter of each internal face from the oracle alone: the phi row of face f carries phid (w_f p_o +
    (1 - w_f) p_n) with w_f = lim w + (1 - lim) upwind, so lim = (R_ll - R_upwind) / (R_linear - R_upwind) on faces where
    p_o != p_n"""
    orc, sp = case.orc, case.spec
    nIF = case.mesh.n_internal_faces
    R = {}
    for what, code in TRANSONIC.items():
        orc.set_transonic(True, code, sp["transonic"], -1)
        R[what] = orc.residual(case.W)[6 * case.nC:6 * case.nC + nIF]
    orc.set_transonic(True, TRANSONIC["limitedLinear"], sp["transonic"], -1)
    den = R["linear"] - R["upwind"]
    ok = np.abs(den) > 1e-9 * np.abs(R["upwind"]).max()
    return (R["limitedLinear"] - R["upwind"])[ok] / den[ok]


# ---- (d) partitions ------------------------------------------------------------------------------------------------------------
def run_partitioned(name, nproc, port, lib_kind):
    case, J = reference(name)
    if case.cyclic:
        d = case.P.case_dir
        solver = Cyclic.SOLVER
    else:
        d = tempfile.mkdtemp(prefix="dab_cprod_mp_")
        case.write(d)
        solver = case.spec["solver"]
    rng = np.random.default_rng(31)
    psi = [rng.uniform(-1.0, 1.0, case.n)]
    for t, (c, frow) in case.boundary_rows().items():
        for r in (3 * c, 3 * c + 1, 3 * c + 2, 3 * case.nC + c, 4 * case.nC + c, 5 * case.nC + c, frow):
            e = np.zeros(case.n)
            e[r] = 1.0
            psi.append(e)
    psi = np.array(psi)
    np.savez(os.path.join(d, "cproducts.npz"), W=case.W, psi=psi, ref=psi @ J, scale=np.array([entry_scale(case, J, p, fd=True) for p in psi]))
    with open(os.path.join(d, "cproducts.json"), "w") as f:
        json.dump(dict(solver=solver, options=case.options), f)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=%d" % nproc, "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.abspath(__file__), d, name, lib_kind]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, OMP_NUM_THREADS="1"), cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert r.stdout.count(" ok: ") == nproc, r.stdout
    print("\n" + r.stdout.strip())


def describe_global(j, nC):
    if j < 6 * nC:
        return "%s of cell %d" % (kinds_of(nC, 6 * nC)[j], j // 3 if j < 3 * nC else j % nC)
    return "phi of face %d" % (j - 6 * nC)


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
    data = np.load(os.path.join(case_dir, "cproducts.npz"))
    with open(os.path.join(case_dir, "cproducts.json")) as f:
        spec = json.load(f)
    dev = rank if cuda else 0
    one = make_solver(spec["solver"], spec["options"], case_dir, lib, device=dev)
    par = make_solver(spec["solver"], spec["options"], case_dir, lib, device=dev, rank=rank, nRanks=world, ncclUniqueId=uid)
    nCg = one.getNGlobalCells()
    nFg = int(one.getLocalToGlobal("faces").max()) + 1
    n = 6 * nCg + nFg

    def maps(sol):
        idx = sol.localStateIndex(nCg, nFg, compressible=True)
        owned = np.concatenate([np.ones(6 * sol.getNLocalCells(), dtype=bool), sol.getLocalToGlobal("faceOwned").astype(bool)])
        return Engine(sol, idx, owned)

    e1, e2 = maps(one), maps(par)
    W = data["W"]
    assert W.size == n
    one.updateOFFields(e1.local(W))
    par.updateOFFields(e2.local(W))
    worst_one = worst_ref = 0.0
    for m, psi in enumerate(data["psi"]):
        y1 = e1.product(psi)
        x2 = e2.local(psi)
        x2[~e2.owned] = 0.0
        yl = np.zeros(e2.idx.size)
        par.calcdRdWTPsiAD(x2, yl)
        assert np.all(yl[~e2.owned] == 0.0), "probe %d: foreign slots must be structural zeros" % m
        t = torch.from_numpy(e2.merged(yl, n))
        dist.all_reduce(t)
        y2 = t.numpy()
        sc = data["scale"][m]
        for ref, tol, what in ((y1, TOL_PART, "one partition"), (data["ref"][m], TOL_J_CUDA if cuda else TOL_J, "dual numbers")):
            e, j = worst_entry(y2, ref, sc)
            assert e <= tol, "rank %d, probe %d: %d partitions vs %s: entry %d (%s): %r vs %r (%.2e)" % (
                rank, m, world, what, j, describe_global(j, nCg), y2[j], ref[j], e)
            if what == "one partition":
                worst_one = max(worst_one, e)
            else:
                worst_ref = max(worst_ref, e)
    print("rank %d ok: %d probes; worst entry vs one partition %.1e, vs dual numbers %.1e" % (rank, len(data["psi"]), worst_one, worst_ref),
          flush=True)
    dist.barrier()
    dist.destroy_process_group()


# ---- (e) function seeding ------------------------------------------------------------------------------------------------------
def check_function_seeding(name, lib_path):
    """dF/dW of a force and a moment on the wing: cForceRevA seeds the work arrays, cRevC finishes the sweep"""
    case, _ = reference(name)
    wing = [p["name"] for p in case.mesh.patches].index("wing")
    d, ctr = [0.6, 0.8, 0.0], [0.25, 0.0, 0.05]
    fn = {"CD": {"type": "force", "source": "patchToFace", "patches": ["wing"], "directionMode": "fixedDirection", "direction": d, "scale": 0.01},
          "CM": {"type": "moment", "source": "patchToFace", "patches": ["wing"], "axis": [0.0, 0.0, 1.0], "center": ctr, "scale": 0.02}}
    eng = case.solver(lib_path)
    eng.sol.updateDAOption(dict(case.options, function=fn))
    eng.sol.updateOFFields(case.W)
    tol = TOL_F if lib_path is not None else TOL_F_CUDA
    p = case.mesh.patches[wing]
    wall = np.zeros(case.nC, dtype=bool)
    wall[case.mesh.owner[p["start"]:p["start"] + p["size"]]] = True
    nIF = case.mesh.n_internal_faces
    support = wall.copy()  # the wall cells and, through their velocity gradient, their neighbours
    support[case.mesh.owner[:nIF][wall[case.mesh.neighbour]]] = True
    support[case.mesh.neighbour[wall[case.mesh.owner[:nIF]]]] = True
    support = support[case.cell]
    worst = 0.0
    for fname, dirv, scale, c_ in (("CD", d, 0.01, None), ("CM", [0.0, 0.0, 1.0], 0.02, ctr)):
        g = np.zeros(case.n)
        eng.sol.calcJacTVecProduct("states", "stateVar", case.W, fname, "function", np.array([1.0]), g)
        go = case.orc.dforce_dw(case.W, wing, dirv, scale, center=c_)
        assert np.abs(go).max() > 0
        # the derivative lives on those cells (and the faces they own) only: every other entry must be an exact zero
        sc = np.where(support, np.maximum(np.abs(go), FLOOR_F * np.abs(go).max()), 0.0)
        worst = max(worst, check_entries(case, g, go, sc, tol, "%s: d%s/dW vs Oracle.dforce_dw" % (name, fname)))
    print("\n%s (%s): dF/dW of a force and a moment, worst entry %.1e" % (name, "CUDA" if lib_path is None else "host build", worst))


# ---- (f) GPU at size -----------------------------------------------------------------------------------------------------------
# |y_j - tape_j| over the largest tape entry of the state block of j.  Measured: 9.8e-14 on the host build, 1.2e-12 on the H100
# (the nuTilda block: the SA source's products of gradients in the wall cells, where FMA contraction rounds differently).  Ten
# times the H100's worst, so a missed term that reaches 1e-11 of the block's largest entry fails; smaller entries (the O-grid's
# cell volumes span eight orders) are the dense-J cases' job.
TOL_BIG = 1e-11


def check_large(lib_path):
    """DARhoSimpleFoam on the 256 x 132 tile-numbered O-grid (the NACA tutorial's linearUpwindV + wall-function variant) against the
    oracle's tape, per entry relative to the largest entry of its state block"""
    mesh = cases.naca0012_ogrid(ni=256, nj=132, nk=1, tile=(16, 12))
    assert mesh.n_cells == 33792
    th = cases.default_thermo(energy="sensibleEnthalpy", transport="sutherland", divE="linearUpwind")
    U0 = (50.0, 2.0, 0.0)
    bcs = cases.compressible_bcs(cases.default_bcs_naca(U0=U0, wall_function=True))
    ns = norm_states(U0[0])
    d = tempfile.mkdtemp(prefix="dab_cbig_")
    cases.write_case(d, mesh, bcs, binary=True, div_u="bounded Gauss linearUpwindV grad(U)", thermo=th)
    orc = Oracle(mesh, bcs, normalizeStates=ns, normalizeResiduals=NRES, thermo=th, divU="linearUpwindV")
    sol = pyDASolvers("DARhoSimpleFoam -python", dict(normalizeStates=ns, normalizeResiduals=list(NRES)), caseDir=d, _lib_path=lib_path)
    W = synthetic_state(mesh, orc.geometry("C"), orc.geometry("Sf"), U0=U0, thermo=th)
    sol.updateOFFields(W)
    orc.record(W)
    nC = mesh.n_cells
    rng = np.random.default_rng(4321)
    out = {}
    for what, psi in (("random psi", rng.uniform(-1.0, 1.0, orc.ndof)), ("psi = 1e-3", np.full(orc.ndof, 1e-3))):
        y, y2 = np.zeros(orc.ndof), np.zeros(orc.ndof)
        sol.calcdRdWTPsiAD(psi, y)
        sol.calcdRdWTPsiAD(psi, y2)
        assert np.array_equal(y, y2), "%s: the product is not bitwise reproducible" % what
        yo = orc.jtvec(psi)
        for blk, a, b in (("U", 0, 3 * nC), ("p", 3 * nC, 4 * nC), ("T", 4 * nC, 5 * nC), ("nuTilda", 5 * nC, 6 * nC), ("phi", 6 * nC, orc.ndof)):
            big = np.abs(yo[a:b]).max()
            err = np.abs(y[a:b] - yo[a:b]) / big
            j = int(np.argmax(err))
            out[(what, blk)] = float(err[j])
            assert err[j] <= TOL_BIG, "%s, %s block: entry %d: %r vs %r (%.2e of the block's largest)" % (what, blk, a + j, y[a + j], yo[a + j], err[j])
    print("\n33 792 cells (%s): worst entry over its block's largest, %s" % ("CUDA" if lib_path is None else "host build",
                                                                          ", ".join("%s %s %.1e" % (k[0], k[1], v) for k, v in out.items())))


# ---- tests ---------------------------------------------------------------------------------------------------------------------
HEX = ["channel_6", "channel_140", "naca_wf", "passage_cyclic"]


@pytest.mark.parametrize("name", list(CASES))
def test_state_product_entries_host_build(name):
    check_state_product(name, HOSTSIM)


def test_values_match_the_tape_on_a_34k_cell_mesh_host_build():
    check_large(HOSTSIM)


def test_limited_linear_limiter_is_active_and_clipped():
    """the transonic cases exercise the limiter's slope (0 < lim < 1, the dLimDr block) and both clipped ends"""
    for name in ("transonic_ll1", "transonic_ll05", "transonic_turbo_mrf"):
        case, _ = reference(name)
        lim = limiter_fractions(case)
        active = np.count_nonzero((lim > 1e-6) & (lim < 1.0 - 1e-6))
        clipped = np.count_nonzero(np.abs(lim) < 1e-9) + np.count_nonzero(np.abs(lim - 1.0) < 1e-9)
        print("\n%s: limitedLinear on %d faces: %d with 0 < lim < 1, %d clipped" % (name, lim.size, active, clipped))
        assert active > 0 and clipped > 0, (name, active, clipped)


def test_mrf_cases_have_rotating_wall_and_relative_flux_faces():
    """MRFZoneDF::setMRFFaces: boundary faces of zone cells on a rotating patch (type 1, the wall velocity and zero relative flux)
    and on a nonRotatingPatch (type 2, minus rho_b (Omega x r).Sf)"""
    for name in ("naca_mrf_turbo", "transonic_turbo_mrf"):
        case, _ = reference(name)
        zone = np.zeros(case.nC, dtype=bool)
        zone[case.mrf["cells"]] = True
        nIF = case.mesh.n_internal_faces
        inz = zone[case.mesh.owner[nIF:]]
        rot = np.array([case.face_patch[f] not in case.mrf["nonRotatingPatches"] for f in range(nIF, case.mesh.n_faces)])
        assert np.count_nonzero(inz & rot) > 0 and np.count_nonzero(inz & ~rot) > 0, name


@pytest.mark.parametrize("name", HEX)
def test_rolled_and_unrolled_face_loops_agree_host_build(name):
    check_rolled_loops(name, HOSTSIM)


@pytest.mark.parametrize("name,nproc,port", [("channel_140", 2, 29821), ("channel_140", 3, 29823), ("passage_cyclic", 2, 29825)])
def test_partitioned_products_host_build(name, nproc, port):
    run_partitioned(name, nproc, port, "host")


@pytest.mark.parametrize("name", ["naca_wf", "naca_mrf_turbo"])
def test_function_seeding_host_build(name):
    check_function_seeding(name, HOSTSIM)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_state_product_entries_cuda(name):
    check_state_product(name, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", HEX)
def test_rolled_and_unrolled_face_loops_agree_cuda(name):
    check_rolled_loops(name, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name,nproc,port", [("channel_140", 2, 29831), ("channel_140", 3, 29833), ("passage_cyclic", 2, 29835)])
def test_partitioned_products_cuda(name, nproc, port):
    import torch
    if torch.cuda.device_count() < nproc:
        # the CUDA build exchanges halos through NCCL, which takes one device per rank; the same partitioned kernels run as
        # several partitions on one machine in test_partitioned_products_host_build
        pytest.skip("%d partitions of the CUDA build need %d GPUs (NCCL: one device per rank)" % (nproc, nproc))
    run_partitioned(name, nproc, port, "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["naca_wf", "naca_mrf_turbo"])
def test_function_seeding_cuda(name):
    check_function_seeding(name, None)


@pytest.mark.gpu
def test_values_match_the_tape_on_a_34k_cell_mesh_cuda():
    check_large(None)


if __name__ == "__main__":
    worker(sys.argv[1], sys.argv[2], sys.argv[3])
