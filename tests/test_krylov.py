"""The Krylov loops of the adjoint solve checked iterate by iterate, not only through their converged answer:
  (a) GMRES(m) (Solver::solveLinearEqn): x_k after k operator applications against a restarted, right-preconditioned Arnoldi
      process in long double (modified Gram-Schmidt run twice, one least-squares solve per cycle), with every restart length and
      both orthogonalisation branches; final_residual and n_matvec of the capped stop; the iteration count to a tolerance and the
      relative-versus-absolute stopping rule;
  (b) IDR(s) (Solver::solveIdrs): x_k against the textbook bi-orthogonal IDR(s) of van Gijzen & Sonneveld (ACM TOMS Algorithm 913)
      in long double -- one alpha_i at a time instead of the engine's batched forward substitution, omega "maintaining the
      convergence" with kappa = 0.7 -- on the engine's own shadow space, regenerated here from its xorshift64 seeds;
  (c) the fixed-point sweep psi <- psi + omega ILU^-1 (b - A psi) of runFPAdj;
  (d) edges: b = 0, b an eigenvector of A M^-1, and one handle that switches between the solvers (grow-only workspaces).
The reference operator is the engine's own: A column by column from calcdRdWTPsiAD(e_i) and M^-1 from applyPC(e_i).  Both were checked
entry by entry against float64 references (test_adjoint_products.py, test_preconditioner.py); taking them from the engine makes the
Krylov loop the only difference between the two sides.  An iterate is capped with gmresMaxIters = k and gmresRelTol = 1e-14: the
solver stops with converged_reason -3 and reports the true residual of x_k.

Shapes: the dot products of the CUDA build are a two-pass multi-dot over tiles of 8 vectors (DOT_TILE) on 528 x 256 threads; GMRES
step k dots k + 2 vectors, so k = 6, 7, 14, 15 land on and just past a tile edge, and IDR(9) and IDR(16) dot 9 and 16 shadow vectors.
The meshes have n = 59 (channel_6: less than one 256-thread CTA), 679 (channel_129), 2616 (NACA 24 x 12 O-grid) and a DARhoSimpleFoam
channel (6 states per cell); on the GPU also a 250 x 140 O-grid with n > 2 x 528 x 256 and n % 256 != 0, whose grid-stride loop
wraps more than once (too large for a dense operator: its reference runs the same GMRES in float64 through the engine's products).

The file is also the worker of the two-partition case: `python -m torch.distributed.run ... tests/test_krylov.py <case dir>
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
from dafoam_b200.pyDASolvers import KSP, pyDASolvers  # noqa: E402
from tests.common import HOSTSIM, NORM_STATES  # noqa: E402

LD = np.longdouble

# ---- tolerances ----------------------------------------------------------------------------------------------------------
# Iterates are compared as |x_k - x_ref| / |x_ref|.  Both sides apply the same float64 operator; what differs is rounding in the
# loop (classical Gram-Schmidt with refinement and float64 Givens rotations against long double modified Gram-Schmidt), times
# the conditioning of the small least-squares problems.  Measured values: host build (x86-64, no FMA contraction) / one H100.
TOL_GMRES = 1e-10   # GMRES x_k, k <= 60, every restart length: measured 1.2e-13 host
TOL_IDR = 1e-8      # IDR(s) x_k for k <= s + 2: measured 1.8e-9 host (channel_129, IDR(9), k = 11).  The engine takes P^T g once from
#                     the unmodified g (a forward substitution, like classical Gram-Schmidt), which rounds up to ~100x worse than
#                     the textbook's one alpha_i at a time; at k = 2s + 3 see ROUND_FACTOR
TOL_FP = 1e-12      # fixed-point psi_k, k <= 10: a contraction, rounding does not grow; measured 1.6e-15 host
TOL_RES = 1e-12     # final_residual vs |b - A x_k| in long double, relative to |b|: one product's rounding; measured 1e-14 host
TOL_SOLVE = 1e-6    # converged psi (relative tolerance 1e-8) vs the dense direct solve: tolerance times cond; measured 4.4e-9 host
TOL_BIG = 1e-9      # 250 x 140 O-grid, x_k (GMRES k <= 20, IDR(9) k <= 11) vs float64 references through the engine's products (GPU only)
IDR_MARGIN = 0.10   # IDR to 1e-8: |its - its_ref| <= 10 % of its_ref + 3.  Rounding changes the iterates beyond 2s + 3 (see
#                     TOL_IDR), so the count moves by a few applications either way; measured +1 to +3 host, 0 to +5 H100
ROUND_FACTOR = 30   # where rounding alone moves an iterate by more than the floors above (IDR at k = 2s + 3: 1e-5 to 3e-2;
#                     GMRES on the DARhoSimpleFoam channel: 5e-6), the tolerance is this factor times the distance
#                     of the same reference run in float64 from its long double iterate (for IDR the larger of the textbook and the
#                     engine's batched variant); measured engine / float64 ratio <= 4.7 host
GMRES_KS = (1, 2, 6, 7, 14, 15, 30, 60)
FULL = 1000          # gmresRestart larger than any k: one cycle


# ---- cases ---------------------------------------------------------------------------------------------------------------
def kinds_of(nC, n, names):
    k = np.empty(n, dtype=object)
    k[:3 * nC] = ["Ux", "Uy", "Uz"] * nC
    off = 3 * nC
    for name in names:
        k[off:off + nC] = name
        off += nC
    k[off:] = "phi"
    return k


class Case:
    """one solver and the dense operator of its adjoint (A: calcdRdWTPsiAD columns; M^-1: applyPC columns per preconditioner)"""

    def __init__(self, name, sol, nC, names):
        self.name, self.sol = name, sol
        self.n = sol.getNLocalAdjointStates()
        self.kinds = kinds_of(nC, self.n, names)
        self.A = dense(sol.calcdRdWTPsiAD, self.n)
        self._M = {}
        self.b = np.random.default_rng(7).uniform(-1.0, 1.0, self.n)

    def minv(self, pc):
        key = tuple(sorted(pc.items()))
        if key not in self._M:
            self.sol.updateDAOption(dict(adjEqnOption=dict(pc)))
            self._M[key] = dense(self.sol.applyPC, self.n)
        return self._M[key]

    def op(self, pc, dtype=LD):
        return Dense(self.A, self.minv(pc), dtype)


def dense(apply, n):
    M = np.empty((n, n))
    e, col = np.zeros(n), np.zeros(n)
    for i in range(n):
        e[:] = 0.0
        e[i] = 1.0
        apply(e, col)
        M[:, i] = col
    return M


def naca_case(lib, ni=24, nj=12):
    from tests.test_adjoint_solve import adjoint_case
    mesh, sol, W = adjoint_case(lib, ni=ni, nj=nj)
    return Case("naca_%dx%d" % (ni, nj), sol, mesh.n_cells, ["p", "nuTilda"])


def channel_case(name, lib):
    from tests.test_adjoint_products import Plain
    c = Plain(name)
    return Case(name, c.solver(lib).sol, c.nC, ["p", "nuTilda"])


def rhosimple_case(lib):
    """2-norm cond(A M^-1) 2.3e15 (cond(A) 1.1e14): a spread of row scales (largest singular value 1.4e8) and one isolated
    near-null mode of A on nuTilda (smallest singular value 1.3e-6, the next 4.2e-3) -- a property of the operator at this
    synthetic state, not of the Krylov loop, which is why its GMRES iterates are compared at ROUND_FACTOR"""
    from tests.test_compressible import CONFIGS, setup_comp
    mesh, orc, sol, W = setup_comp(CONFIGS[2], lib)  # channel, sensibleInternalEnergy, Sutherland, SA
    sol.updateOFFields(W)
    return Case("rhosimple_channel", sol, mesh.n_cells, ["p", "T", "nuTilda"])


BUILDERS = {"channel_6": lambda lib: channel_case("channel_6", lib), "channel_129": lambda lib: channel_case("channel_129", lib),
            "naca": naca_case, "rhosimple": rhosimple_case}
_CASES = {}


def case_of(name, lib):
    if (name, lib) not in _CASES:
        _CASES[(name, lib)] = BUILDERS[name](lib)
    return _CASES[(name, lib)]


BASE_PC = dict(coarseAggregates=0, coarseSparseAP=1, pcStorage="fp64", globalPCIters=0)


# ---- references ----------------------------------------------------------------------------------------------------------
class Dense:
    """the engine's operator as dense matrices: long double, or float64 to measure how much rounding moves an iterate"""

    def __init__(self, A, Mi, dtype=LD):
        self.dtype = dtype
        self.Al, self.Ml = A.astype(dtype), Mi.astype(dtype)

    def A(self, v):
        return self.Al @ v

    def M(self, v):
        return self.Ml @ v


class Products:
    """the engine's operator as callbacks (a mesh too large for a dense matrix): float64"""
    dtype = np.float64

    def __init__(self, sol):
        self.sol = sol
        self.n = sol.getNLocalAdjointStates()

    def _call(self, f, v):
        y = np.zeros(self.n)
        f(np.ascontiguousarray(v, dtype=np.float64), y)
        return y

    def A(self, v):
        return self._call(self.sol.calcdRdWTPsiAD, v)

    def M(self, v):
        return self._call(self.sol.applyPC, v)


def norm(v):
    return np.sqrt(v @ v)


def back_solve(R, g):
    y = np.zeros(g.size, dtype=R.dtype)
    for i in range(g.size - 1, -1, -1):
        y[i] = (g[i] - R[i, i + 1:g.size] @ y[i + 1:]) / R[i, i]
    return y


def ref_gmres(op, b, ks, m, tol=None):
    """restarted right-preconditioned GMRES(m) from x = 0: {k: (x_k, cycles started)} for k in ks, and the residual estimate
    after every application.  Arnoldi with modified Gram-Schmidt run twice; each cycle solves its least-squares problem with
    Givens rotations.  With tol, stops at the first application whose residual is <= tol."""
    dt = op.dtype
    b = b.astype(dt)
    n, kmax = b.size, max(ks)
    x = np.zeros(n, dt)
    its, cycles, out, hist = 0, 0, {}, []
    while its < kmax:
        r = b - op.A(x)
        beta = norm(r)
        V = np.zeros((m + 1, n), dt)
        V[0] = r / beta
        R = np.zeros((m + 1, m), dt)
        cs, sn, g = np.zeros(m, dt), np.zeros(m, dt), np.zeros(m + 1, dt)
        g[0] = beta
        cycles += 1
        j = 0
        while j < m and its < kmax:
            w = op.A(op.M(V[j]))
            h = np.zeros(j + 2, dt)
            for _ in range(2):
                for i in range(j + 1):
                    d = V[i] @ w
                    h[i] += d
                    w = w - d * V[i]
            h[j + 1] = norm(w)
            V[j + 1] = w / h[j + 1]
            for i in range(j):
                h[i], h[i + 1] = cs[i] * h[i] + sn[i] * h[i + 1], -sn[i] * h[i] + cs[i] * h[i + 1]
            dd = np.sqrt(h[j] * h[j] + h[j + 1] * h[j + 1])
            cs[j], sn[j] = h[j] / dd, h[j + 1] / dd
            h[j] = dd
            g[j + 1], g[j] = -sn[j] * g[j], cs[j] * g[j]
            R[:j + 1, j] = h[:j + 1]
            j += 1
            its += 1
            hist.append(abs(g[j]))
            if its in ks:
                out[its] = (x + op.M(V[:j].T @ back_solve(R[:j, :j], g[:j])), cycles)
            if tol is not None and abs(g[j]) <= tol:
                return out, hist
        x = x + op.M(V[:j].T @ back_solve(R[:j, :j], g[:j]))
    return out, hist


def shadow_space(ns, s):
    """the engine's IDR shadow vectors (solver_krylov.hpp, solveIdrs): per rank r and vector j, xorshift64 from the seed
    0x9E3779B97F4A7C15 (j + 1) + 0xD1B54A32D192ED03 (r + 1), uniform in [-0.5, 0.5); then modified Gram-Schmidt over the
    rank-concatenated vectors.  ns: local vector length of each rank."""
    mask = (1 << 64) - 1
    P = np.empty((s, sum(ns)), dtype=LD)
    for j in range(s):
        parts = []
        for rank, n in enumerate(ns):
            x = (0x9E3779B97F4A7C15 * (j + 1) + 0xD1B54A32D192ED03 * (rank + 1)) & mask
            h = np.empty(n)
            for i in range(n):
                x ^= (x << 13) & mask
                x ^= x >> 7
                x ^= (x << 17) & mask
                h[i] = float(x >> 11) * (1.0 / 9007199254740992.0) - 0.5
            parts.append(h)
        P[j] = np.concatenate(parts)
        for i in range(j):
            P[j] = P[j] - (P[i] @ P[j]) * P[i]
        P[j] = P[j] / norm(P[j])
    return P


def ref_idrs(op, b, P, ks, tol=None, kappa=0.7, batched=False):
    """IDR(s) with bi-orthogonalisation (van Gijzen & Sonneveld, ACM TOMS Algorithm 913), right preconditioning, x = 0: {k: x_k}
    after k operator applications, and the number of applications to |r| <= tol.  The bi-orthogonalisation of g against
    P_0..P_{k-1} runs one alpha_i at a time on the updated g.  batched: the engine's forward substitution instead (P^T g from the
    unmodified g), used only in float64 to measure how much that variant's rounding moves an iterate."""
    s, dt = P.shape[0], op.dtype
    P, b = P.astype(dt), b.astype(dt)
    kmax = max(ks) if ks else 10 ** 9
    x, r = np.zeros(b.size, dt), b.copy()
    G, U = np.zeros((s, b.size), dt), np.zeros((s, b.size), dt)
    Mm = np.eye(s, dtype=dt)
    om, its, out = dt(1.0), 0, {}

    def done():
        return its >= kmax or (tol is not None and norm(r) <= tol)

    while not done():
        f = P @ r
        for k in range(s):
            if done():
                break
            c = np.zeros(s, dt)
            for i in range(k, s):
                c[i] = (f[i] - Mm[i, k:i] @ c[k:i]) / Mm[i, i]
            z = op.M(r - c[k:] @ G[k:])
            u = c[k:] @ U[k:] + om * z
            g = op.A(u)
            if batched:
                d, al = P @ g, np.zeros(k, dt)
                for i in range(k):
                    al[i] = (d[i] - Mm[i, :i] @ al[:i]) / Mm[i, i]
                g, u = g - al @ G[:k], u - al @ U[:k]
                Mm[k:, k] = d[k:] - Mm[k:, :k] @ al
            else:
                for i in range(k):
                    alpha = (P[i] @ g) / Mm[i, i]
                    g = g - alpha * G[i]
                    u = u - alpha * U[i]
                Mm[k:, k] = P[k:] @ g
            G[k], U[k] = g, u
            beta = f[k] / Mm[k, k]
            r = r - beta * g
            x = x + beta * u
            f[k + 1:] -= beta * Mm[k + 1:, k]
            its += 1
            out[its] = x.copy() if its in ks else None
        if done():
            break
        z = op.M(r)
        t = op.A(z)
        its += 1
        tr, tt = t @ r, t @ t
        om = tr / tt
        rho = tr / (np.sqrt(tt) * norm(r))
        if abs(rho) < kappa:
            om = om * kappa / abs(rho)
        r = r - om * t
        x = x + om * z
        out[its] = x.copy() if its in ks else None
    return {k: v for k, v in out.items() if v is not None}, its


# ---- the engine ----------------------------------------------------------------------------------------------------------
def run(sol, b, pc=BASE_PC, **adj):
    """one solve with every Krylov option spelled out (options persist on a handle); returns x, stats, fail flag"""
    opts = dict(kspType="gmres", idrS=4, gmresRestart=FULL, gmresMaxIters=60, gmresRelTol=1e-14, gmresAbsTol=1e-300, useMGSO=0)
    opts.update(pc)
    opts.update(adj)
    sol.updateDAOption(dict(adjEqnOption=opts))
    x = np.zeros(b.size)
    ksp = KSP()
    fail = sol.solveLinearEqn(ksp, np.ascontiguousarray(b), x)
    return x, ksp.stats, fail


def pc_extras(pc):
    """operator products inside one applyPC: the matrix-free coarse correction and the Richardson sweeps"""
    return (1 if pc.get("coarseAggregates", 0) > 0 and not pc.get("coarseSparseAP", 1) else 0) + pc.get("globalPCIters", 0)


def rel(x, ref):
    ref = np.asarray(ref, dtype=LD)
    return float(norm(np.asarray(x, dtype=LD) - ref) / norm(ref))


def rounding_tol(ref, ref64, floor):
    """floor, or ROUND_FACTOR times how far float64 runs (the same reference; for IDR also the engine's batched variant) land
    from the long double iterate"""
    return max([floor] + [ROUND_FACTOR * rel(r, ref) for r in (ref64 if isinstance(ref64, list) else [ref64])])


def idr_float64(op64, b, P, ks):
    """{k: [textbook x_k, batched x_k]} in float64"""
    t, _ = ref_idrs(op64, b, P, ks)
    u, _ = ref_idrs(op64, b, P, ks, batched=True)
    return {k: [t[k], u[k]] for k in ks}


def check_iterate(case, x, ref, tol, what):
    ref = np.asarray(ref, dtype=LD)
    d = np.abs(x.astype(LD) - ref)
    e = float(norm(d) / norm(ref))
    j = int(np.argmax(d))
    assert e <= tol, "%s on %s: |x_k - x_ref| / |x_ref| = %.2e > %.1e; worst entry %d (%s): %r vs %r" % (
        what, case.name, e, tol, j, case.kinds[j], x[j], float(ref[j]))
    return e


def kind_name(lib):
    return "host build" if lib else "CUDA"


# ---- (a) GMRES -----------------------------------------------------------------------------------------------------------
def check_gmres_iterates(name, lib):
    case = case_of(name, lib)
    op = case.op(BASE_PC)
    ks = [k for k in GMRES_KS if k <= case.n // 2]
    Al = op.Al
    worst = worst_res = 0.0
    for m in (FULL, 5, 8):
        ref, _ = ref_gmres(op, case.b, ks, min(m, max(ks)))
        ref64, _ = ref_gmres(case.op(BASE_PC, np.float64), case.b, ks, min(m, max(ks)))
        for mgso in (0, 1):
            for k in ks:
                x, st, fail = run(case.sol, case.b, gmresRestart=m, gmresMaxIters=k, useMGSO=mgso)
                what = "GMRES(%s) useMGSO %d, k = %d" % ("full" if m == FULL else m, mgso, k)
                assert st.converged_reason == -3 and st.iterations == k and fail == 1, (what, st.converged_reason, st.iterations, fail)
                xr, cycles = ref[k]
                assert cycles == -(-k // min(m, k)), (what, cycles)
                assert st.n_matvec == k + cycles, "%s: %d operator products, expected k + cycles = %d" % (what, st.n_matvec, k + cycles)
                tol = rounding_tol(xr, ref64[k][0], TOL_GMRES)
                worst = max(worst, check_iterate(case, x, xr, tol, what) / tol)
                rt = float(norm(case.b.astype(LD) - Al @ x.astype(LD)))
                e = abs(st.final_residual - rt) / np.linalg.norm(case.b)
                assert e <= TOL_RES, "%s: final_residual %r vs |b - A x_k| %r" % (what, st.final_residual, rt)
                worst_res = max(worst_res, e)
    print("\n%s (%s, n = %d): GMRES iterates k in %s, restart full/5/8, useMGSO 0/1: worst %.2f of the tolerance; final_residual %.1e"
          % (name, kind_name(lib), case.n, ks, worst, worst_res))


def check_gmres_convergence(lib):
    case = case_of("naca", lib)
    op = case.op(BASE_PC)
    tol = 1e-8 * np.linalg.norm(case.b)
    _, hist = ref_gmres(op, case.b, [400], 400, tol=tol)
    k_ref = len(hist)
    x, st, fail = run(case.sol, case.b, gmresMaxIters=400, gmresRelTol=1e-8)
    its = st.iterations
    # the engine stops on its Givens recurrence, which agrees with the reference's residual only to rounding: when |r_k| lies
    # within that rounding of the tolerance, the two sides may cross it one application apart
    assert fail == 0 and st.converged_reason == 2 and abs(st.iterations - k_ref) <= 1, (st.iterations, k_ref, hist[-3:])
    psi = np.linalg.solve(case.A, case.b)
    e = np.linalg.norm(x - psi) / np.linalg.norm(psi)
    assert e <= TOL_SOLVE, e
    # |b| ~ 1e-12: the absolute tolerance (gmresAbsTol 1e-14) is the larger one and decides
    bs = case.b * 1e-12
    x, st, fail = run(case.sol, bs, gmresMaxIters=400, gmresRelTol=1e-8, gmresAbsTol=1e-14)
    assert st.converged_reason == 3 and fail == 0 and st.final_residual <= 1e-14 * 1.0000001, (st.converged_reason, fail, st.final_residual)
    assert st.iterations < k_ref, (st.iterations, k_ref)
    print("\nGMRES to 1e-8 (%s): %d iterations, reference %d; psi vs dense solve %.1e; |b| 1e-12: %d iterations" % (kind_name(lib), its, k_ref, e, st.iterations))


# ---- (b) IDR(s) ----------------------------------------------------------------------------------------------------------
def idr_ks(s):
    return sorted({1, s, s + 1, s + 2, 2 * s + 3})


def check_idrs_iterates(name, lib, svals=(1, 4, 8, 9, 16)):
    case = case_of(name, lib)
    op = case.op(BASE_PC)
    worst = 0.0
    for s in svals:
        P = shadow_space([case.n], s)
        ks = idr_ks(s)
        ref, _ = ref_idrs(op, case.b, P, ks)
        ref64 = idr_float64(case.op(BASE_PC, np.float64), case.b, P, ks)
        for k in ks:
            x, st, fail = run(case.sol, case.b, kspType="idrs", idrS=s, gmresMaxIters=k)
            what = "IDR(%d), k = %d" % (s, k)
            assert st.converged_reason == -3 and st.iterations == k and st.n_matvec == k + 1, (what, st.converged_reason, st.iterations, st.n_matvec)
            tol = rounding_tol(ref[k], ref64[k], TOL_IDR)
            worst = max(worst, check_iterate(case, x, ref[k], tol, what) / tol)
            if k == ks[-1]:
                x2, _, _ = run(case.sol, case.b, kspType="idrs", idrS=s, gmresMaxIters=k)
                assert np.array_equal(x, x2), "%s: two solves on one handle differ" % what
    print("\n%s (%s, n = %d): IDR(s) iterates, s in %s, k <= 2s + 3: worst %.2f of the tolerance" % (name, kind_name(lib), case.n, list(svals), worst))


def check_idrs_convergence(lib, svals=(1, 4, 8, 9, 16)):
    case = case_of("naca", lib)
    op = case.op(BASE_PC)
    psi = np.linalg.solve(case.A, case.b)
    tol = 1e-8 * np.linalg.norm(case.b)
    for s in svals:
        _, its_ref = ref_idrs(op, case.b, shadow_space([case.n], s), [], tol=tol)
        x, st, fail = run(case.sol, case.b, kspType="idrs", idrS=s, gmresMaxIters=1500, gmresRelTol=1e-8)
        assert fail == 0 and st.converged_reason == 2, (s, st.converged_reason)
        assert abs(st.iterations - its_ref) <= IDR_MARGIN * its_ref + 3, (s, st.iterations, its_ref)
        e = np.linalg.norm(x - psi) / np.linalg.norm(psi)
        assert e <= TOL_SOLVE, (s, e)
        print("IDR(%d) to 1e-8 (%s): %d applications, reference %d; psi vs dense solve %.1e" % (s, kind_name(lib), st.iterations, its_ref, e))


# ---- preconditioner variants, edges, fixed point ---------------------------------------------------------------------------
PC_VARIANTS = {
    # 12 aggregates: A P has 2.4 entries per row on this mesh, so the sparse path is kept (the engine drops it above 3 per row,
    # which 24 aggregates exceed); n_matvec tells the two paths apart: the matrix-free one takes one product per application
    "coarse 12, sparse A P": dict(BASE_PC, coarseAggregates=12, coarseSparseAP=1),
    "coarse 12, matrix-free A P": dict(BASE_PC, coarseAggregates=12, coarseSparseAP=0),
    "fp32 factors": dict(BASE_PC, pcStorage="fp32"),
    "globalPCIters 2": dict(BASE_PC, globalPCIters=2),
}
BENCH_PC = dict(BASE_PC, coarseAggregates=12, pcStorage="fp32")  # bench.py: IDR(8), coarse space with sparse A P, fp32 factors


def check_pc_variants(lib):
    case = case_of("naca", lib)
    worst = 0.0
    for what, pc in PC_VARIANTS.items():
        op = case.op(pc)
        ks = [7, 15, 30]
        ref, _ = ref_gmres(op, case.b, ks, 30)
        ref64, _ = ref_gmres(case.op(pc, np.float64), case.b, ks, 30)
        for k in ks:
            x, st, fail = run(case.sol, case.b, pc=pc, gmresMaxIters=k)
            assert st.converged_reason == -3 and st.n_matvec == (k + 1) * (1 + pc_extras(pc)), (what, k, st.n_matvec)
            tol = rounding_tol(ref[k][0], ref64[k][0], TOL_GMRES)
            worst = max(worst, check_iterate(case, x, ref[k][0], tol, "GMRES, %s, k = %d" % (what, k)) / tol)
    op = case.op(BENCH_PC)
    ks = idr_ks(8)
    P = shadow_space([case.n], 8)
    ref, _ = ref_idrs(op, case.b, P, ks)
    ref64 = idr_float64(case.op(BENCH_PC, np.float64), case.b, P, ks)
    for k in ks:
        x, st, fail = run(case.sol, case.b, pc=BENCH_PC, kspType="idrs", idrS=8, gmresMaxIters=k)
        assert st.converged_reason == -3 and st.n_matvec == k + 1, (k, st.n_matvec)  # the sparse A P path: no extra product
        tol = rounding_tol(ref[k], ref64[k], TOL_IDR)
        worst = max(worst, check_iterate(case, x, ref[k], tol, "IDR(8), coarse 12 + fp32 factors, k = %d" % k) / tol)
    print("\npreconditioner variants (%s): worst %.2f of the tolerance" % (kind_name(lib), worst))


def check_zero_rhs(lib):
    case = case_of("channel_129", lib)
    for ksp in ("gmres", "idrs"):
        x, st, fail = run(case.sol, np.zeros(case.n), kspType=ksp, gmresMaxIters=50)
        assert st.converged_reason == 3 and fail == 0 and st.iterations == 0 and np.all(x == 0.0), (ksp, st.converged_reason, fail, st.iterations)


def check_eigenvector(lib):
    """b = a real eigenvector of A M^-1: the Krylov space is one-dimensional, GMRES converges in one step with x = M^-1 b / lambda"""
    case = case_of("channel_6", lib)
    Mi = case.minv(BASE_PC)
    lam, vec = np.linalg.eig(case.A @ Mi)
    real = np.nonzero(np.abs(lam.imag) == 0.0)[0]
    gap = np.array([np.delete(np.abs(lam - lam[i]), i).min() / abs(lam[i]) for i in real])
    i = real[int(np.argmax(gap))]  # the best separated real eigenvalue: its eigenvector is accurate to rounding
    b = np.ascontiguousarray(vec[:, i].real)
    x, st, fail = run(case.sol, b, gmresMaxIters=50, gmresRelTol=1e-10)
    assert st.converged_reason == 2 and fail == 0 and st.iterations == 1, (st.converged_reason, fail, st.iterations)
    xr = Mi @ b / lam[i].real
    check_iterate(case, x, xr, 1e-10, "eigenvector rhs (lambda %.3g)" % lam[i].real)


def check_shared_handle(lib):
    """one handle that switches between the solvers gives the iterates of fresh handles.  GMRES and IDR(s) share the dot-product
    workspace and the coefficient buffer (GMRES: m + 1 values per cycle, IDR(s): s), and the handle keeps IDR's workspace while s
    is unchanged: IDR(9), then GMRES(5), then IDR(9) again reuses IDR's workspace after GMRES sized the shared buffer for 7"""
    from tests.test_adjoint_solve import adjoint_case
    seq = [dict(gmresRestart=8, gmresMaxIters=20), dict(kspType="idrs", idrS=4, gmresMaxIters=11),
           dict(gmresRestart=30, gmresMaxIters=25), dict(kspType="idrs", idrS=9, gmresMaxIters=21),
           dict(gmresRestart=5, gmresMaxIters=5), dict(kspType="idrs", idrS=9, gmresMaxIters=12),
           dict(gmresRestart=5, gmresMaxIters=12), dict(kspType="idrs", idrS=16, gmresMaxIters=20)]
    _, shared, _ = adjoint_case(lib)  # a handle of its own: what it has been through is this sequence only
    b = np.random.default_rng(7).uniform(-1.0, 1.0, shared.getNLocalAdjointStates())
    for opts in seq:
        x, _, _ = run(shared, b, **opts)
        _, fresh, _ = adjoint_case(lib)
        xf, _, _ = run(fresh, b, **opts)
        assert np.array_equal(x, xf), ("shared handle vs fresh handle", opts, np.abs(x - xf).max())


def check_fixed_point(lib):
    case = case_of("naca", lib)
    Ilu = case.minv(BASE_PC).astype(LD)  # ILU(0) only: no coarse space, no Richardson sweeps, as solveFixedPoint applies it
    Al, b = case.A.astype(LD), case.b.astype(LD)
    worst = 0.0
    for omega in (0.5, 0.8):
        psi = np.zeros(case.n, LD)
        ref = {}
        for k in range(1, 11):
            psi = psi + LD(omega) * (Ilu @ (b - Al @ psi))
            ref[k] = psi.copy()
        for k in (1, 2, 10):
            case.sol.updateDAOption(dict(adjEqnOption=dict(BASE_PC, fpMaxIters=k, fpOmega=omega, fpRelTol=1e-300, fpMinResTolDiff=1.0)))
            x = np.zeros(case.n)
            case.sol.runFPAdj(np.ascontiguousarray(case.b), x)
            assert case.sol.fpStats.iterations == k and case.sol.fpStats.n_matvec == k + 1, (omega, k, case.sol.fpStats.iterations)
            worst = max(worst, check_iterate(case, x, ref[k], TOL_FP, "fixed point, omega %g, k = %d" % (omega, k)))
    print("\nfixed point (%s): worst %.2e" % (kind_name(lib), worst))


# ---- a mesh too large for a dense operator (GPU) ---------------------------------------------------------------------------
BIG_PC = dict(BASE_PC, coarseAggregates=200)


def check_big_mesh(lib):
    """250 x 140 O-grid, n = 315 250 > 2 x 528 x 256 and n % 256 = 114: the grid-stride loop of the multi-dot wraps twice and its
    last pass is partial.  The reference is the same GMRES (and IDR(9)) in float64 with the engine's products as callbacks."""
    from types import SimpleNamespace
    mesh = cases.naca0012_ogrid(ni=250, nj=140, nk=1, tile=(10, 14))
    d = tempfile.mkdtemp(prefix="dab_kry_big_")
    cases.write_case(d, mesh, cases.default_bcs_naca(wall_function=True), binary=True, div_u="bounded Gauss linearUpwindV grad(U)")
    sol = pyDASolvers("DASimpleFoam -python", dict(normalizeStates=NORM_STATES), caseDir=d, _lib_path=lib)
    yw = np.zeros(mesh.n_cells)
    sol.getOFField("yWall", "scalar", yw)
    sol.updateOFFields(cases.boundary_layer_state(mesh, yw, noise=0.01))
    n = sol.getNLocalAdjointStates()
    print("\n250 x 140 O-grid: n = %d (n %% 256 = %d, 2 x 528 x 256 = %d)" % (n, n % 256, 2 * 528 * 256))
    assert n > 2 * 528 * 256 and n % 256 != 0, n
    case = SimpleNamespace(name="naca_250x140", kinds=kinds_of(mesh.n_cells, n, ["p", "nuTilda"]))
    sol.updateDAOption(dict(adjEqnOption=BIG_PC))
    op = Products(sol)
    b = np.random.default_rng(7).uniform(-1.0, 1.0, n)
    ks = [1, 6, 7, 14, 15, 20]
    ref, _ = ref_gmres(op, b, ks, 20)
    worst = 0.0
    for k in ks:
        x, st, _ = run(sol, b, pc=BIG_PC, gmresMaxIters=k)
        assert st.converged_reason == -3 and st.iterations == k, (k, st.converged_reason, st.iterations)
        worst = max(worst, check_iterate(case, x, ref[k][0], TOL_BIG, "GMRES, k = %d" % k))
    ks = idr_ks(9)[:-1]
    ref, _ = ref_idrs(op, b, shadow_space([n], 9), ks)
    for k in ks:
        x, st, _ = run(sol, b, pc=BIG_PC, kspType="idrs", idrS=9, gmresMaxIters=k)
        worst = max(worst, check_iterate(case, x, ref[k], TOL_BIG, "IDR(9), k = %d" % k))
    print("GMRES k <= 20 and IDR(9) k <= 11 vs float64 references through the engine's products: worst %.2e" % worst)


# ---- two partitions ------------------------------------------------------------------------------------------------------
def run_partitioned(lib_kind, port):
    """the 7 x 5 x 4 channel on two partitions: the reference operator is built over the rank-concatenated local vectors"""
    from tests.test_adjoint_products import Plain
    c = Plain("channel_140")
    d = tempfile.mkdtemp(prefix="dab_kry_mp_")
    c.write(d)
    np.save(os.path.join(d, "W.npy"), c.W)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.abspath(__file__), d, lib_kind]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=dict(os.environ, OMP_NUM_THREADS="1"), cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert " ok: " in r.stdout, r.stdout
    print("\n" + r.stdout.strip())


def worker(case_dir, lib_kind):
    import torch
    import torch.distributed as dist
    from types import SimpleNamespace
    from dafoam_b200.pyDASolvers import set_comm_callbacks
    from tests.test_adjoint_products import ENGINE_OPTS
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
    dev = rank if cuda else 0
    one = pyDASolvers("DASimpleFoam -python", dict(ENGINE_OPTS), caseDir=case_dir, device=dev, _lib_path=lib)
    nCg = one.getNGlobalCells()
    nFg = int(one.getLocalToGlobal("faces").max()) + 1
    par = pyDASolvers("DASimpleFoam -python", dict(ENGINE_OPTS), caseDir=case_dir, device=dev, rank=rank, nRanks=world, ncclUniqueId=uid,
                      _lib_path=lib)
    idx = par.localStateIndex(nCg, nFg)
    par.updateOFFields(np.ascontiguousarray(np.load(os.path.join(case_dir, "W.npy"))[idx]))
    nl = idx.size
    owned = np.concatenate([np.ones(5 * par.getNLocalCells(), dtype=bool), par.getLocalToGlobal("faceOwned").astype(bool)])

    def gather(v):
        out = [None] * world
        dist.all_gather_object(out, v)
        return out

    sizes = gather(nl)
    N, off = sum(sizes), sum(sizes[:rank])
    # the operator over the concatenated rank-local vectors, column by column (collective products on every rank)
    A, Mi = np.empty((nl, N)), np.empty((nl, N))
    e, y = np.zeros(nl), np.zeros(nl)
    par.updateDAOption(dict(adjEqnOption=dict(BASE_PC)))
    for i in range(N):
        e[:] = 0.0
        if off <= i < off + nl:
            e[i - off] = 1.0
        par.calcdRdWTPsiAD(e, y)
        A[:, i] = y
        par.applyPC(e, y)
        Mi[:, i] = y
    A, Mi = np.vstack(gather(A)), np.vstack(gather(Mi))
    own = np.concatenate(gather(owned))
    b = np.where(own, np.random.default_rng(7).uniform(-1.0, 1.0, N), 0.0)  # no right-hand side on slots another rank owns
    runs = [("GMRES(full), k = %d" % k, dict(gmresMaxIters=k)) for k in (1, 7, 15, 30)]
    runs += [("GMRES(8), k = %d" % k, dict(gmresRestart=8, gmresMaxIters=k)) for k in (15, 30)]
    for s in (4, 9):
        runs += [("IDR(%d), k = %d" % (s, k), dict(kspType="idrs", idrS=s, gmresMaxIters=k)) for k in idr_ks(s)]
    xs = {}
    for what, opts in runs:
        x, st, _ = run(par, np.ascontiguousarray(b[off:off + nl]), **opts)
        xs[what] = np.concatenate(gather(x))
        assert st.converged_reason == -3, (what, st.converged_reason)
    if rank == 0:
        op = Dense(A, Mi)
        slots = ["rank %d, local slot %d" % (r, j) for r, m in enumerate(sizes) for j in range(m)]
        case = SimpleNamespace(name="channel_140 on 2 partitions", kinds=np.array(slots, dtype=object))
        op64 = Dense(A, Mi, np.float64)
        gm = {m: (ref_gmres(op, b, [1, 7, 15, 30], m)[0], ref_gmres(op64, b, [1, 7, 15, 30], m)[0]) for m in (30, 8)}
        idr = {}
        for s in (4, 9):
            P = shadow_space(sizes, s)
            idr[s] = (ref_idrs(op, b, P, idr_ks(s))[0], idr_float64(op64, b, P, idr_ks(s)))
        worst = 0.0
        for what, opts in runs:
            k = opts["gmresMaxIters"]
            if "idrS" in opts:
                ref, ref64 = idr[opts["idrS"]]
                ref, tol = ref[k], rounding_tol(ref[k], ref64[k], TOL_IDR)
            else:
                ref, ref64 = gm[opts.get("gmresRestart", 30)]
                ref, tol = ref[k][0], rounding_tol(ref[k][0], ref64[k][0], TOL_GMRES)
            worst = max(worst, check_iterate(case, xs[what], ref, tol, what) / tol)
        print("rank 0 ok: n = %s; %d capped solves (GMRES, IDR(4), IDR(9)) vs the concatenated reference: worst %.2f of the tolerance"
              % ("+".join(map(str, sizes)), len(runs), worst), flush=True)
    dist.barrier()
    dist.destroy_process_group()


# ---- tests: host build ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["channel_6", "channel_129", "naca", "rhosimple"])
def test_gmres_iterates_host_build(name):
    check_gmres_iterates(name, HOSTSIM)


def test_gmres_convergence_host_build():
    check_gmres_convergence(HOSTSIM)


@pytest.mark.parametrize("name", ["channel_129", "naca"])
def test_idrs_iterates_host_build(name):
    check_idrs_iterates(name, HOSTSIM)


def test_idrs_convergence_host_build():
    check_idrs_convergence(HOSTSIM)


def test_pc_variants_host_build():
    check_pc_variants(HOSTSIM)


def test_zero_rhs_host_build():
    check_zero_rhs(HOSTSIM)


def test_eigenvector_rhs_host_build():
    check_eigenvector(HOSTSIM)


def test_shared_handle_host_build():
    check_shared_handle(HOSTSIM)


def test_fixed_point_iterates_host_build():
    check_fixed_point(HOSTSIM)


@pytest.mark.parametrize("port", [29821])
def test_two_partitions_host_build(port):
    run_partitioned("host", port)


# ---- tests: CUDA ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["channel_6", "channel_129", "naca", "rhosimple"])
def test_gmres_iterates_cuda(name):
    check_gmres_iterates(name, None)


@pytest.mark.gpu
def test_gmres_convergence_cuda():
    check_gmres_convergence(None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["channel_129", "naca"])
def test_idrs_iterates_cuda(name):
    check_idrs_iterates(name, None)


@pytest.mark.gpu
def test_idrs_convergence_cuda():
    check_idrs_convergence(None)


@pytest.mark.gpu
def test_pc_variants_cuda():
    check_pc_variants(None)


@pytest.mark.gpu
def test_zero_rhs_cuda():
    check_zero_rhs(None)


@pytest.mark.gpu
def test_eigenvector_rhs_cuda():
    check_eigenvector(None)


@pytest.mark.gpu
def test_shared_handle_cuda():
    check_shared_handle(None)


@pytest.mark.gpu
def test_fixed_point_iterates_cuda():
    check_fixed_point(None)


@pytest.mark.gpu
def test_multidot_grid_stride_cuda():
    check_big_mesh(None)


@pytest.mark.gpu
@pytest.mark.parametrize("port", [29823])
def test_two_partitions_cuda(port):
    import torch
    if torch.cuda.device_count() < 2:
        # NCCL takes one device per rank; the same partitioned Krylov loop runs on one machine in test_two_partitions_host_build
        pytest.skip("2 partitions of the CUDA build need 2 GPUs (NCCL: one device per rank)")
    run_partitioned("cuda", port)


if __name__ == "__main__":
    worker(sys.argv[1], sys.argv[2])
