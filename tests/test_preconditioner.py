"""The adjoint preconditioner checked directly, not through the iteration count of a solve:
  (a) every stored entry of the assembled dRdWTPC against a per-column forward difference of the oracle's first-order
      residual (same step and state scaling as the engine) and, loosely, against the oracle's exact isPC Jacobian;
  (b) the ILU(0) factors against a plain row-by-row ILU(0) of that matrix in the engine's factorisation order, and the
      ordering invariant that makes the per-colour kernels race-free;
  (c) M^-1 v (applyPC) against forward/backward substitution with those factors;
  (d) the two-level (pressure coarse space) and Richardson (globalPCIters) wrappers against their definitions.
The references below are plain numpy/Python; none of them goes through the engine's ordering, pattern or kernels."""
import tempfile

import numpy as np
import pytest

from dafoam_b200 import cases
from dafoam_b200.pyDASolvers import Mat, pyDASolvers
from tests.common import HOSTSIM, NORM_STATES, setup

FD_STEP = 1e-6     # adjPartDerivFDStep.State default
PIVOT_SHIFT = 1e-10  # relative pivot guard of the factorisation
KEEP = dict(writeJacobians=["dRdWTPC"])

# ---- tolerances, each set from the worst deviation measured over every case of this file (host build: x86-64 without fused
# multiply-adds; CUDA: one H100 80GB HBM3 SXM).  (a) and (b) are relative to the largest entry of the row (and of the column, for
# (a)); (c) and (d) to the largest entry of the reference vector.
TOL_FD = 2e-8      # (a) stored entry vs the oracle's per-state forward difference: measured 3.1e-9 (host and H100)
TOL_EXACT = 1e-4   # (a) stored entry vs the exact isPC Jacobian (forward-FD truncation at h = 1e-6): measured 1.5e-5 (host and H100)
TOL_ILU = {HOSTSIM: 0.0, None: 1e-11}        # (b) fp64 factors vs ref_ilu0: host bitwise, H100 5.1e-13 (contracted FMAs)
TOL_ILU_F32 = {HOSTSIM: 0.0, None: 1.2e-7}   # (b) fp32 copy vs ref_ilu0 rounded to fp32: host bitwise, H100 4e-25; allows one flip
TOL_APPLY = {HOSTSIM: 1e-12, None: 1e-12}    # (c) applyPC vs substitution: measured host 6.4e-15, H100 2.5e-14
TOL_TWO_LEVEL = {HOSTSIM: 1e-9, None: 1e-9}  # (d) measured host 6.8e-12, H100 5.3e-12 (12 aggregates, cond(Ac) 2e5)


# ---- cases -------------------------------------------------------------------------------------------------------------
def kinds_of(n_cells, n_dof, names):
    """state / residual kind of every external index: U, p, [T], [nuTilda], phi"""
    k = np.empty(n_dof, dtype=object)
    k[:3 * n_cells] = "U"
    off = 3 * n_cells
    for name in names:
        k[off:off + n_cells] = name
        off += n_cells
    k[off:] = "phi"
    return k


def state_scales(kinds, magSf, norm):
    """the engine's FD perturbation per state: normalizeStates value, times |Sf| for phi"""
    s = np.array([norm[k] if k != "phi" else 0.0 for k in kinds])
    phi = kinds == "phi"
    s[phi] = norm["phi"] * magSf
    return s


def incompressible(kind, turbulent, divU, nk, adj=None, lib_path=HOSTSIM):
    mesh, bcs, orc, sol, W, _ = setup(kind, turbulent, divU, nk, lib_path=lib_path,
                                      extra_options=dict(KEEP, adjEqnOption=dict(adj or {})))
    names = ["p", "nuTilda"] if turbulent else ["p"]
    return mesh, orc, sol, W, kinds_of(mesh.n_cells, orc.ndof, names), NORM_STATES


def compressible(lib_path=HOSTSIM):
    from tests.test_compressible import CONFIGS, NS, setup_comp
    mesh, orc, sol, W = setup_comp(CONFIGS[2], lib_path)  # channel, sensibleInternalEnergy, Sutherland, SA
    sol.updateDAOption(KEEP)
    return mesh, orc, sol, W, kinds_of(mesh.n_cells, orc.ndof, ["p", "T", "nuTilda"]), NS


ASSEMBLY_CASES = {
    "naca_sa": lambda lib: incompressible("naca", True, "linearUpwind", 1, lib_path=lib),
    "channel_laminar": lambda lib: incompressible("channel", False, "upwind", 1, lib_path=lib),  # 4 cell slots
    "prism": lambda lib: incompressible("prism", True, "linearUpwind", 1, lib_path=lib),       # 5 faces per cell
    "wing_nk3": lambda lib: incompressible("wing", True, "linearUpwindV", 3, lib_path=lib),    # skewed hexahedra: most slots
    "rhosimple_channel": compressible,                                                         # T state: 6 cell slots
    "naca_stateinfo": lambda lib: incompressible("naca", True, "linearUpwind", 1, dict(pcPattern="stateInfo", pcConLevel=3), lib),
    "naca_level1": lambda lib: incompressible("naca", True, "linearUpwind", 1, dict(pcConLevel=1), lib),
    "naca_level3": lambda lib: incompressible("naca", True, "linearUpwind", 1, dict(pcConLevel=3), lib),
}


def naca_adjoint_case(lib_path, ni, nj, adj=None):
    """an O-grid with a boundary-layer state (no oracle needed): the variants of (b)-(d)"""
    mesh = cases.naca0012_ogrid(ni=ni, nj=nj, nk=1)
    d = tempfile.mkdtemp(prefix="dab_pc_")
    cases.write_case(d, mesh, cases.default_bcs_naca())
    sol = pyDASolvers("DASimpleFoam -python", dict(KEEP, normalizeStates=NORM_STATES, adjEqnOption=dict(adj or {})), caseDir=d,
                      _lib_path=lib_path)
    y = np.zeros(sol.getNLocalCells())
    sol.getOFField("yWall", "scalar", y)
    W = cases.boundary_layer_state(mesh, y)
    sol.updateOFFields(W)
    return mesh, sol, W


def passage_case(lib_path):
    """one-rank cyclic passage as in test_cyclic.solve_on_passage: a partitioned local mesh with identity rows for cut faces"""
    mesh = cases.annular_passage(nr=6, nt=6, nz=12, n_sectors=36)
    bcs = cases.default_bcs_passage(Uin=(0.0, 0.0, 100.0))
    th = cases.default_thermo(energy="sensibleEnthalpy")
    mrf = dict(cellZone="rotor", cells=np.arange(mesh.n_cells), origin=(0.0, 0.0, 0.0), axis=(0.0, 0.0, 1.0), omega=300.0,
               nonRotatingPatches=["inlet", "outlet", "shroud"])
    d = tempfile.mkdtemp(prefix="dab_pc_cyc_")
    cases.write_case(d, mesh, cases.compressible_bcs(bcs), mrf=mrf, thermo=th)
    ns = dict(U=100.0, p=101325.0, T=300.0, nuTilda=1e-3, phi=1.0)
    sol = pyDASolvers("DATurboFoam -python", dict(KEEP, normalizeStates=ns), caseDir=d, _lib_path=lib_path)
    Wg = cases.passage_state(mesh, Uax=100.0, thermo=th, n_sectors=36)
    idx = sol.localStateIndex(mesh.n_cells, cases.merged_face_order(mesh).size, compressible=True)
    sol.updateOFFields(np.ascontiguousarray(Wg[idx]))
    return sol


def assemble(sol):
    sol.calcdRdWT(1, Mat())
    return sol.getPCMatrix(), sol.getPCFactors()


# ---- (a) assembly ------------------------------------------------------------------------------------------------------
def check_assembly(name, lib_path):
    mesh, orc, sol, W, kinds, norm = ASSEMBLY_CASES[name](lib_path)
    sol.updateOFFields(W)
    (rp, cl, vl), _ = assemble(sol)
    n = orc.ndof
    assert len(rp) == n + 1
    scale = state_scales(kinds, orc.geometry("magSf"), norm)
    R0 = orc.residual(W, 1)
    # one oracle residual per state: row j of dRdWTPC is (R(W + h s_j e_j) - R(W)) / h, the engine's coloured difference done
    # one state at a time
    ref_vals, row_max, dropped = np.empty(len(vl)), np.empty(n), {}
    Wp = W.copy()
    for j in range(n):
        Wp[j] = W[j] + FD_STEP * scale[j]
        ref = (orc.residual(Wp, 1) - R0) / FD_STEP
        Wp[j] = W[j]
        c = cl[rp[j]:rp[j + 1]]
        assert j in c, ("no diagonal", name, j)
        ref_vals[rp[j]:rp[j + 1]] = ref[c]
        row_max[j] = np.abs(ref).max()
        out = np.ones(n, dtype=bool)
        out[c] = False
        for r in np.nonzero(out & (ref != 0.0))[0]:
            key = (kinds[j], kinds[r])
            dropped[key] = max(dropped.get(key, 0.0), abs(ref[r]) / row_max[j])
    # Both differences carry the roundoff of their residual evaluation amplified by 1/h, and that roundoff scales with the size of
    # the residual's terms, i.e. with the largest entry of the residual's column as much as with the state's row: the deviation is
    # measured against the larger of the two.
    col_max = np.zeros(n)
    np.maximum.at(col_max, cl, np.abs(ref_vals))
    row = np.repeat(np.arange(n), np.diff(rp))
    err = np.abs(vl - ref_vals) / np.maximum(np.maximum(row_max[row], col_max[cl]), 1e-300)
    at = int(np.argmax(err))
    worst_fd, worst_row = float(err[at]), int(row[at])
    # exact isPC Jacobian on a sample of the rows (one tape product per row), same scale as above
    worst_ex = 0.0
    e_j = np.zeros(n)
    for j in range(0, n, max(1, n // 300)):
        e_j[:] = 0.0
        e_j[j] = scale[j]
        ref = orc.jvec(W, e_j, isPC=1)
        c, v = cl[rp[j]:rp[j + 1]], vl[rp[j]:rp[j + 1]]
        worst_ex = max(worst_ex, (np.abs(v - ref[c]) / np.maximum(np.abs(ref).max(), col_max[c])).max())
    print("\n%s: %d rows, %.1f entries/row; worst |stored - oracle FD| / max(row max, column max) %.2e (row %d, %s), |stored - exact| %.2e"
          % (name, n, len(cl) / n, worst_fd, worst_row, kinds[worst_row], worst_ex))
    print("  largest dropped coupling / row max, per (state, residual):",
          ", ".join("%s->%sRes %.1e" % (k[0], k[1], dropped[k]) for k in sorted(dropped)))
    assert worst_fd <= TOL_FD, (name, "row %d (%s state) column %d (%s residual): %r vs %r" % (worst_row, kinds[worst_row], cl[at], kinds[cl[at]], vl[at], ref_vals[at]))
    assert worst_ex <= TOL_EXACT, (name, worst_ex)
    return mesh, sol, kinds


# ---- (b) ILU(0) factors ------------------------------------------------------------------------------------------------
def permuted(rp, cl, vl, perm):
    """the assembled matrix (external numbering) in the factorisation order: row i = external row perm[i], sorted columns"""
    n = len(perm)
    iperm = np.empty(n, dtype=np.int64)
    iperm[perm] = np.arange(n)
    prp = np.zeros(n + 1, dtype=np.int64)
    lens = (rp[1:] - rp[:-1])[perm]
    prp[1:] = np.cumsum(lens)
    pcl = np.empty(len(cl), dtype=np.int64)
    pvl = np.empty(len(vl))
    for i in range(n):
        a, b = rp[perm[i]], rp[perm[i] + 1]
        c = iperm[cl[a:b]]
        o = np.argsort(c, kind="stable")
        pcl[prp[i]:prp[i + 1]] = c[o]
        pvl[prp[i]:prp[i + 1]] = vl[a:b][o]
    return prp, pcl, pvl


def ref_ilu0(rp, cl, vl):
    """ILU(0) row by row in the given order on the given pattern.  Pivot rule: rowMax over the row before its elimination; a
    pivot with |d| <= 1e-10 rowMax becomes sign(d) 1e-10 rowMax (+-1 for a zero row); the reciprocal 1/d is stored, and the
    multipliers are formed with it.  Returns the factor values and the number of guarded pivots."""
    n = len(rp) - 1
    rp, cl, v = rp.tolist(), cl.tolist(), [float(x) for x in vl]
    diag = [0] * n
    for i in range(n):
        diag[i] = rp[i] + cl[rp[i]:rp[i + 1]].index(i)
    guarded = 0
    for i in range(n):
        a, b, di = rp[i], rp[i + 1], diag[i]
        pos = {cl[e]: e for e in range(a, b)}
        row_max = max(abs(v[e]) for e in range(a, b))
        for e in range(a, di):
            k = cl[e]
            lik = v[e] * v[diag[k]]
            v[e] = lik
            if lik == 0.0:
                continue
            for q in range(diag[k] + 1, rp[k + 1]):
                p = pos.get(cl[q])
                if p is not None:
                    v[p] -= lik * v[q]
        d = v[di]
        if not abs(d) > PIVOT_SHIFT * row_max:
            guarded += 1
            d = (-1.0 if d < 0.0 else 1.0) * (PIVOT_SHIFT * row_max if row_max > 0.0 else 1.0)
        v[di] = 1.0 / d
    return np.array(v), guarded


def cell_of_external(mesh, n_cell_states, n_dof):
    """cell of every external state: its own cell, or the owner of a face (the block a face's row belongs to)"""
    nC = mesh.n_cells
    c = np.empty(n_dof, dtype=np.int64)
    c[:3 * nC] = np.arange(3 * nC) // 3
    c[3 * nC:n_cell_states * nC] = np.arange((n_cell_states - 3) * nC) % nC
    c[n_cell_states * nC:] = mesh.owner[:n_dof - n_cell_states * nC]
    return c


def check_ordering(F, cell_ext):
    """factorisation order is colour-major, and within a colour a row's off-diagonal columns of the same colour belong to its own
    cell: the rows one kernel launch factorises or solves in parallel never read each other"""
    rp, cl, _, perm, colour = F
    assert np.array_equal(np.sort(perm), np.arange(len(perm))), "perm is not a permutation"
    assert np.all(np.diff(colour) >= 0), "rows are not grouped by colour"
    cell = cell_ext[perm]
    row = np.repeat(np.arange(len(perm)), np.diff(rp))
    same = (colour[cl] == colour[row]) & (cl != row)
    bad = np.nonzero(same & (cell[cl] != cell[row]))[0]
    assert bad.size == 0, ("same-colour coupling across cells", int(row[bad[0]]), int(cl[bad[0]]))


def check_factors(sol, A, F, lib_path, f32=False, label=""):
    rp, cl, vl = A
    frp, fcl, fvl, perm, colour = F
    prp, pcl, pvl = permuted(rp, cl, vl, perm)
    assert np.array_equal(prp, frp) and np.array_equal(pcl, fcl), (label, "factor pattern differs from the assembled pattern")
    ref, guarded = ref_ilu0(prp, pcl, pvl)
    if f32:
        ref = ref.astype(np.float32).astype(np.float64)
    rmax = np.maximum.reduceat(np.abs(ref), frp[:-1])
    err = np.abs(fvl - ref) / np.repeat(rmax, np.diff(frp))
    worst = float(err.max())
    at = int(np.argmax(err))
    i = int(np.searchsorted(frp, at, side="right") - 1)
    where = "L" if fcl[at] < i else ("1/u_ii" if fcl[at] == i else "U")
    print("\n%s ILU(0)%s: %d rows, %d colours, %d guarded pivots; worst |factor - ref| / row max %.2e (row %d, %s entry, column %d)"
          % (label, " fp32" if f32 else "", len(perm), colour.max() + 1, guarded, worst, i, where, fcl[at]))
    tol = (TOL_ILU_F32 if f32 else TOL_ILU)[lib_path]
    assert worst <= tol, (label, "factor row %d (colour %d), %s entry at column %d: %r vs %r" % (i, colour[i], where, fcl[at], fvl[at], ref[at]))
    return ref


# ---- (c) application ---------------------------------------------------------------------------------------------------
def ref_apply(F, V):
    """M^-1 V for the columns of V: gather by perm, unit-lower forward substitution, backward substitution multiplying by the
    stored reciprocal, scatter"""
    rp, cl, vals, perm = F[0], F[1], F[2], F[3]
    n = len(perm)
    Y = np.array(V, dtype=np.float64).reshape(n, -1)[perm].copy()
    diag = np.empty(n, dtype=np.int64)
    for i in range(n):
        diag[i] = rp[i] + np.searchsorted(cl[rp[i]:rp[i + 1]], i)
    for i in range(n):
        a, d = rp[i], diag[i]
        if d > a:
            Y[i] -= vals[a:d] @ Y[cl[a:d]]
    for i in range(n - 1, -1, -1):
        d, b = diag[i], rp[i + 1]
        Y[i] = (Y[i] - vals[d + 1:b] @ Y[cl[d + 1:b]]) * vals[d]
    Z = np.empty_like(Y)
    Z[perm] = Y
    return Z


def probe_vectors(F, cell_ext, n_cells, seed=7):
    """random, constant, unit spikes on the first and last row of every colour and on the first and last row of the last slot of
    every colour whose last slot has fewer rows than the colour has cells (cells sorted by owned-face count)"""
    rp, cl, _, perm, colour = F
    n = len(perm)
    rows = set()
    for k in range(colour.max() + 1):
        r = np.nonzero(colour == k)[0]
        rows.update((int(r[0]), int(r[-1])))
        if cell_ext is None:
            continue
        # slots: runs in which the cells appear in the colour's cell order, which slot 0 (the x-velocity rows) lists in full
        cells = cell_ext[perm[r]]
        slot0 = (perm[r] < 3 * n_cells) & (perm[r] % 3 == 0)
        order = {int(c): q for q, c in enumerate(cells[slot0])}
        q = np.array([order[int(c)] for c in cells])
        starts = np.concatenate([[0], np.nonzero(np.diff(q) <= 0)[0] + 1])
        last = r[starts[-1]:]
        if len(last) < slot0.sum():
            rows.update((int(last[0]), int(last[-1])))
    V = [np.random.default_rng(seed).uniform(-1.0, 1.0, n), np.ones(n)]
    for i in sorted(rows):
        e = np.zeros(n)
        e[perm[i]] = 1.0
        V.append(e)
    return np.array(V).T.copy(), len(rows)


def check_apply(sol, F, cell_ext, n_cells, lib_path, label=""):
    V, n_spikes = probe_vectors(F, cell_ext, n_cells)
    Zref = ref_apply(F, V)
    n = V.shape[0]
    worst, which = 0.0, -1
    z, z2 = np.zeros(n), np.zeros(n)
    for m in range(V.shape[1]):
        v = np.ascontiguousarray(V[:, m])
        sol.applyPC(v, z)
        sol.applyPC(v, z2)
        assert np.array_equal(z, z2), (label, "applyPC is not deterministic", m)
        e = np.abs(z - Zref[:, m]).max() / np.abs(Zref[:, m]).max()
        if e > worst:
            worst, which = e, m
    kind = "random" if which == 0 else "constant" if which == 1 else "spike"
    print("%s applyPC: %d vectors (%d spikes); worst |z - ref|inf / |ref|inf %.2e (%s vector %d)" % (label, V.shape[1], n_spikes, worst, kind, which))
    assert worst <= TOL_APPLY[lib_path], (label, kind, which, worst)


def check_case_pc(sol, mesh, n_cell_states, lib_path, label, f32=False):
    """(b) and (c) on an assembled case"""
    A, F = assemble(sol)
    cell_ext = cell_of_external(mesh, n_cell_states, len(F[3])) if mesh is not None else None
    if cell_ext is not None:
        check_ordering(F, cell_ext)
    check_factors(sol, A, F, lib_path, f32=f32, label=label)
    check_apply(sol, F, cell_ext, mesh.n_cells if mesh is not None else 0, lib_path, label=label)
    return A, F


# ---- (d) two-level and Richardson --------------------------------------------------------------------------------------
def operator_columns(sol, X):
    out = np.zeros_like(X)
    y = np.zeros(X.shape[0])
    for a in range(X.shape[1]):
        sol.calcdRdWTPsiAD(np.ascontiguousarray(X[:, a]), y)
        out[:, a] = y
    return out


def check_two_level(lib_path, n_agg, sparse_ap):
    mesh, sol, W = naca_adjoint_case(lib_path, 48, 24, dict(coarseAggregates=n_agg, coarseSparseAP=sparse_ap))
    _, F = assemble(sol)
    agg = sol.getPCAggregates()
    nC = mesh.n_cells
    n = len(F[3])
    K = int(agg.max()) + 1
    assert np.array_equal(np.unique(agg), np.arange(K))
    P = np.zeros((n, K))
    P[3 * nC + np.arange(nC), agg] = 1.0
    AP = operator_columns(sol, P)
    Ac = P.T @ AP
    V = np.random.default_rng(11).uniform(-1.0, 1.0, (n, 2))
    V[:, 1] = 1.0
    Yc = np.linalg.solve(Ac, P.T @ V)
    Zref = P @ Yc + ref_apply(F, V - AP @ Yc)
    worst = 0.0
    z = np.zeros(n)
    for m in range(V.shape[1]):
        sol.applyPC(np.ascontiguousarray(V[:, m]), z)
        worst = max(worst, np.abs(z - Zref[:, m]).max() / np.abs(Zref[:, m]).max())
    print("\ntwo-level, %d aggregates (asked %d), coarseSparseAP %d: cond(Ac) %.1e, worst |z - ref|inf / |ref|inf %.2e"
          % (K, n_agg, sparse_ap, np.linalg.cond(Ac), worst))
    assert worst <= TOL_TWO_LEVEL[lib_path], (n_agg, sparse_ap, worst)


def check_richardson(lib_path, sweeps=2):
    mesh, sol, W = naca_adjoint_case(lib_path, 40, 20, dict(globalPCIters=sweeps))
    _, F = assemble(sol)
    n = len(F[3])
    v = np.random.default_rng(5).uniform(-1.0, 1.0, n)
    z = ref_apply(F, v)[:, 0]
    Az = np.zeros(n)
    for _ in range(sweeps):
        sol.calcdRdWTPsiAD(np.ascontiguousarray(z), Az)
        z = z + ref_apply(F, v - Az)[:, 0]
    out = np.zeros(n)
    sol.applyPC(v, out)
    worst = np.abs(out - z).max() / np.abs(z).max()
    print("\nRichardson, %d sweeps: worst |z - ref|inf / |ref|inf %.2e" % (sweeps, worst))
    assert worst <= TOL_TWO_LEVEL[lib_path], worst


# ---- the variants of (b) and (c) ---------------------------------------------------------------------------------------
VARIANTS = {
    "multicolour": {},
    "block64": dict(pcBlockCells=64),   # 800 cells: a partial last block (TRI_LANES = 4 solves)
    "block50": dict(pcBlockCells=50),   # 800 cells: whole blocks
    "multicolour_fp32": dict(pcStorage="fp32"),
    "block64_fp32": dict(pcBlockCells=64, pcStorage="fp32"),
    "colour_radius2": dict(pcColourRadius=2),  # many colours, launches of fewer than 32 cells
    "stateinfo": dict(pcPattern="stateInfo"),  # uneven row lengths: -1 padding inside the ELL groups
}


def check_variant(name, lib_path, ni=40, nj=20):
    adj = VARIANTS[name]
    mesh, sol, W = naca_adjoint_case(lib_path, ni, nj, adj)
    check_case_pc(sol, mesh, 5, lib_path, "%s %dx%d" % (name, ni, nj), f32=adj.get("pcStorage") == "fp32")


# ---- tests --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(ASSEMBLY_CASES))
def test_pc_assembly_and_factors_host_build(name):
    mesh, sol, kinds = check_assembly(name, HOSTSIM)
    ns = 3 + len(set(kinds) - {"U", "phi"})
    check_case_pc(sol, mesh, ns, HOSTSIM, name)


@pytest.mark.parametrize("name", list(VARIANTS))
def test_pc_factors_and_apply_host_build(name):
    check_variant(name, HOSTSIM)


def test_pc_factors_and_apply_cyclic_passage_host_build():
    check_case_pc(passage_case(HOSTSIM), None, 6, HOSTSIM, "cyclic passage")


@pytest.mark.parametrize("n_agg,sparse_ap", [(12, 0), (12, 1), (100, 0), (100, 1)])
def test_two_level_apply_host_build(n_agg, sparse_ap):
    check_two_level(HOSTSIM, n_agg, sparse_ap)


def test_richardson_apply_host_build():
    check_richardson(HOSTSIM)


def test_pc_aggregates_need_a_coarse_space():
    from dafoam_b200.pyDASolvers import DAB200Error
    mesh, sol, W = naca_adjoint_case(HOSTSIM, 24, 12)
    with pytest.raises(DAB200Error, match="no ILU"):
        sol.getPCFactors()
    sol.calcdRdWT(1, Mat())
    with pytest.raises(DAB200Error, match="coarse space"):
        sol.getPCAggregates()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ASSEMBLY_CASES))
def test_pc_assembly_and_factors_cuda(name):
    mesh, sol, kinds = check_assembly(name, None)
    ns = 3 + len(set(kinds) - {"U", "phi"})
    check_case_pc(sol, mesh, ns, None, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VARIANTS))
def test_pc_factors_and_apply_cuda(name):
    check_variant(name, None)


@pytest.mark.gpu
def test_pc_factors_and_apply_medium_ogrid_cuda():
    """128 x 64 cells: every colour launch spans many CTAs and ends in a partial warp"""
    check_variant("multicolour", None, 128, 64)


@pytest.mark.gpu
def test_pc_factors_and_apply_cyclic_passage_cuda():
    check_case_pc(passage_case(None), None, 6, None, "cyclic passage")


@pytest.mark.gpu
@pytest.mark.parametrize("n_agg,sparse_ap", [(12, 0), (12, 1), (100, 0), (100, 1)])
def test_two_level_apply_cuda(n_agg, sparse_ap):
    check_two_level(None, n_agg, sparse_ap)


@pytest.mark.gpu
def test_richardson_apply_cuda():
    check_richardson(None)
