// Device kernels of the SIMPLE primal solver (reference src/adjoint/DASolver/DASimpleFoam/DASimpleFoam.C:123-185,
// UEqnSimple.H, pEqnSimple.H; turbulence: DASpalartAllmaras::correct = calcResiduals with solveTurbState_ = 1,
// DASpalartAllmaras.C:407-470).  Each equation is assembled by one cell-parallel gather into a per-cell ELL row
// (one coefficient per face slot of the cell -> the same ELL shape as cellFaces/cellNbr), with exactly the
// discretisation of the residual kernels in fwd_kernels.hpp, so the fixed point of the iteration is R(W) = 0.
#pragma once
#include "backend.hpp"
#include "views.hpp"
#include "fwd_kernels.hpp"
#include "krylov.hpp"
#include <cmath>

namespace dab
{

// one segregated equation: (diag_j x_j)_c + sum_k off_k x_j,nbr(k) = b_j
struct EqnView
{
    int nC, maxCF, nc;      // nc: components sharing the off-diagonals (U: 3)
    double* off;            // [maxCF][nC]
    double* diag;           // [nc][nC]
    double* b;              // [nc][nC]
    const int32_t* cellNbr; // [maxCF][nC]
};

// momentum matrix: fvm::div(phi,U) + divDevReff(U), relaxed (fvMatrix::relax), boundary coefficients folded into
// the per-component diagonal/source the way fvMatrix::solveSegregated does (addBoundaryDiag / addBoundarySource);
// rAU = 1/A() is written to the record.  The pressure gradient is NOT part of b (UEqn == -grad(p) at solve time).
template <int NF, int FEAT>
struct UEqnAssemble
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    EqnView e;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const int schU = q.divU;
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double nuEc = r.nut[c] + q.nu;
        double gUc[9];
        for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
        const double trc = gUc[0] + gUc[4] + gUc[8];
        double D0 = 0.0, sumOff = 0.0, X[3] = {0.0, 0.0, 0.0}; // X = explicit part of V*(UEqn & U)
        double icMax = 0.0, icMin = 0.0, icAvg = 0.0, icS[3] = {0.0, 0.0, 0.0};
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0)
            {
                for (int kk = k; kk < m.maxCF; kk++) e.off[(size_t)kk * nC + c] = 0.0;
                break;
            }
            const int f = fr.f;
            const double mf = fr.s * s.phi[f];
            const double Sv[3] = {m.Sx[f], m.Sy[f], m.Sz[f]};
            const double mS = m.magSf[f], dl = m.delta[f];
            if (!fr.bnd)
            {
                const int n = fr.n;
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f], wn = 1.0 - wc;
                const bool pos0 = s.phi[f] >= 0.0;
                const double wup = fr.s > 0 ? (pos0 ? 1.0 : 0.0) : (pos0 ? 0.0 : 1.0);
                const double Un[3] = {s.U[3 * n], s.U[3 * n + 1], s.U[3 * n + 2]};
                const double nuEn = r.nut[n] + q.nu;
                const double wp = schU == DIV_LINEAR ? wc : wup;
                const double a = wp * mf;
                const double gf = (wc * nuEc + wn * nuEn) * mS;
                const double g = gf * dl;
                const double off = mf - a - g;
                e.off[(size_t)k * nC + c] = off;
                D0 += a + g - mf;
                sumOff += fabs(off);
                double gUn[9];
                for (int i = 0; i < 9; i++) gUn[i] = r.gU[(size_t)i * nT + n];
                if (schU == DIV_LINEAR_UPWIND || ((FEAT & 1) && schU == DIV_LINEAR_UPWIND_V))
                {
                    const bool ownUp = s.phi[f] > 0.0;
                    const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                    double gu[9]; // per-element selects: a pointer into either array would put both in local memory
                    for (int i = 0; i < 9; i++) gu[i] = cUp ? gUc[i] : gUn[i];
                    const int u = cUp ? c : n;
                    const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                    double corr[3];
                    for (int j = 0; j < 3; j++) corr[j] = d[0] * gu[j * 3 + 0] + d[1] * gu[j * 3 + 1] + d[2] * gu[j * 3 + 2];
                    if ((FEAT & 1) && schU == DIV_LINEAR_UPWIND_V)
                    {
                        const double wo_ = m.w[f];
                        const double cf = ownUp ? (1.0 - wo_) : -wo_;
                        double maxCorr[3];
                        for (int j = 0; j < 3; j++) maxCorr[j] = cf * fr.s * (Un[j] - Uc[j]);
                        luvLimit(corr, maxCorr, corr);
                    }
                    for (int j = 0; j < 3; j++) X[j] += mf * corr[j];
                }
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                const double wo = m.w[f];
                const bool own = fr.s > 0; // value selects: a pointer into either gradient array would put both in local memory
                for (int j = 0; j < 3; j++)
                {
                    double cg = 0.0;
                    for (int i = 0; i < 3; i++)
                    {
                        const double gO = own ? gUc[j * 3 + i] : gUn[j * 3 + i], gN_ = own ? gUn[j * 3 + i] : gUc[j * 3 + i];
                        cg += kv[i] * (wo * gO + (1.0 - wo) * gN_);
                    }
                    X[j] -= fr.s * gf * cg;
                }
                const double trn = gUn[0] + gUn[4] + gUn[8];
                for (int j = 0; j < 3; j++)
                {
                    const double tc = nuEc * (Sv[0] * gUc[0 * 3 + j] + Sv[1] * gUc[1 * 3 + j] + Sv[2] * gUc[2 * 3 + j] - (2.0 / 3.0) * trc * Sv[j]);
                    const double tn = nuEn * (Sv[0] * gUn[0 * 3 + j] + Sv[1] * gUn[1 * 3 + j] + Sv[2] * gUn[2 * 3 + j] - (2.0 / 3.0) * trn * Sv[j]);
                    X[j] -= fr.s * (wc * tc + wn * tn);
                }
            }
            else
            {
                e.off[(size_t)k * nC + c] = 0.0;
                const int b = f - m.nIF, pa = m.bPatch[b];
                const double im = frcp(mS);
                const double nh[3] = {Sv[0] * im, Sv[1] * im, Sv[2] * im};
                BCv bu;
                double uw[3];
                mrfWallRef(m, f, q.bcVal[F_U][pa], uw);
                bcVector(q.bcKind[F_U][pa], uw, Uc, mf, dl, nh, bu);
                double ntb = 0.0, sngN = 0.0, frN;
                const double ntc = q.turb ? s.nt[c] : 0.0;
                if (q.turb) bcScalar(q.bcKind[F_NUTILDA][pa], q.bcVal[F_NUTILDA][pa][0], ntc, mf, dl, ntb, sngN, frN);
                double dP, dNb, dUn[3];
                double nutb = 0.0;
                if (q.turb)
                    nutb = (FEAT & 2) ? nutBoundary<true>(q.bcKind[F_NUT][pa], q.bcVal[F_NUT][pa][0], r.nut[c], ntb, q.nu, Uc, bu.val, dl, dP, dNb, dUn)
                                      : nutBoundaryBasic(q.bcKind[F_NUT][pa], q.bcVal[F_NUT][pa][0], r.nut[c], ntb, q.nu, dP, dNb);
                const double G = (nutb + q.nu) * mS;
                D0 -= mf; // bounded
                double mx = 0.0, mn = 0.0, av = 0.0;
                for (int j = 0; j < 3; j++)
                {
                    const double ic = mf * bu.vic[j] - G * bu.gic[j];
                    const double aic = fabs(ic);
                    if (j == 0) { mx = aic; mn = ic; }
                    else { mx = aic > mx ? aic : mx; mn = ic < mn ? ic : mn; }
                    av += ic;
                    icS[j] += ic;
                    // explicit remainder of the boundary contribution: mf*val - G*sng - ic*U_P
                    X[j] += mf * bu.val[j] - G * bu.sng[j] - ic * Uc[j];
                }
                icMax += mx; icMin += mn; icAvg += av / 3.0;
                double Gb[9];
                for (int j = 0; j < 3; j++)
                {
                    const double nG = nh[0] * gUc[j * 3 + 0] + nh[1] * gUc[j * 3 + 1] + nh[2] * gUc[j * 3 + 2];
                    for (int i = 0; i < 3; i++) Gb[j * 3 + i] = gUc[j * 3 + i] + nh[i] * (bu.sng[j] - nG);
                }
                const double trb = Gb[0] + Gb[4] + Gb[8];
                for (int j = 0; j < 3; j++)
                {
                    const double x = Sv[0] * Gb[0 * 3 + j] + Sv[1] * Gb[1 * 3 + j] + Sv[2] * Gb[2 * 3 + j] - (2.0 / 3.0) * trb * Sv[j];
                    X[j] -= (nutb + q.nu) * x;
                }
            }
        }
        const double V = m.V[c];
        const double D1 = D0 + icMax;
        const double aD1 = fabs(D1);
        const double D2 = aD1 > sumOff ? aD1 : sumOff;
        const double Dn = D2 * frcp(q.alphaU) - icMin;
        r.rAU[c] = V * frcp(Dn + icAvg);
        double cor[3] = {0.0, 0.0, 0.0}; // MRF.DDt(U), explicit
        if (m.mrfCell && m.mrfCell[c])
        {
            const double* w = m.mrfOmega;
            cor[0] = w[1] * Uc[2] - w[2] * Uc[1];
            cor[1] = w[2] * Uc[0] - w[0] * Uc[2];
            cor[2] = w[0] * Uc[1] - w[1] * Uc[0];
        }
        for (int j = 0; j < 3; j++)
        {
            e.diag[(size_t)j * nC + c] = Dn + icS[j];
            e.b[(size_t)j * nC + c] = -X[j] + (Dn - D0) * Uc[j] + (m.fvS ? V * m.fvS[(size_t)j * nC + c] : 0.0) - V * cor[j];
        }
    }
};

// one Jacobi sweep of a segregated equation on an AoS (stride nc) or SoA field; rhs_j = b_j - V*g_j (g: optional
// gradient record, SoA [nc][nT])
template <int NC>
struct JacobiSweep
{
    EqnView e;
    const double* x;  // [nc*nT] AoS (stride nc)
    double* xn;       // same layout
    const double* g;  // nullable: [nc][nT] subtracted as V*g
    const double* V;
    int nT;
    DAB_HD void operator()(int c) const
    {
        const int nC = e.nC;
        double acc[3] = {0.0, 0.0, 0.0};
        for (int k = 0; k < e.maxCF; k++)
        {
            const int n = e.cellNbr[(size_t)k * nC + c];
            if (n < 0) continue;
            const double o = e.off[(size_t)k * nC + c];
            for (int j = 0; j < NC; j++) acc[j] += o * x[(size_t)NC * n + j];
        }
        for (int j = 0; j < NC; j++)
        {
            double rhs = e.b[(size_t)j * nC + c];
            if (g) rhs -= V[c] * g[(size_t)j * nT + c];
            xn[(size_t)NC * c + j] = (rhs - acc[j]) * frcp(e.diag[(size_t)j * nC + c]);
        }
    }
};

// residual pieces of a segregated equation for OpenFOAM's normalised L1 residual (lduMatrix::solver::normFactor):
// out[j][c] = |b - A x|, out[nc+j][c] = |A x - xRef*rowSum| + |b - xRef*rowSum|
template <int NC>
struct EqnResidual
{
    EqnView e;
    const double* x;
    const double* g;
    const double* V;
    int nT;
    double xRef[3];
    double* out; // [2*nc][nC]
    DAB_HD void operator()(int c) const
    {
        const int nC = e.nC;
        double acc[3] = {0.0, 0.0, 0.0}, so = 0.0;
        for (int k = 0; k < e.maxCF; k++)
        {
            const int n = e.cellNbr[(size_t)k * nC + c];
            if (n < 0) continue;
            const double o = e.off[(size_t)k * nC + c];
            so += o;
            for (int j = 0; j < NC; j++) acc[j] += o * x[(size_t)NC * n + j];
        }
        for (int j = 0; j < NC; j++)
        {
            double rhs = e.b[(size_t)j * nC + c];
            if (g) rhs -= V[c] * g[(size_t)j * nT + c];
            const double d = e.diag[(size_t)j * nC + c];
            const double Ax = d * x[(size_t)NC * c + j] + acc[j];
            const double xa = xRef[j] * (d + so);
            out[(size_t)j * nC + c] = fabs(rhs - Ax);
            out[(size_t)(NC + j) * nC + c] = fabs(Ax - xa) + fabs(rhs - xa);
        }
    }
};

// SoA copy of a strided component (for the reductions)
struct StridedCopy
{
    const double* src;
    int stride, nc, nC;
    double* dst; // [nc][nC]
    DAB_HD void operator()(int c) const
    {
        for (int j = 0; j < nc; j++) dst[(size_t)j * nC + c] = src[(size_t)stride * c + j];
    }
};

// HbyA = rAU*H = U - rAU*(UEqn & U) with the matrix frozen and U the solution of the momentum predictor
// SIMPLEC (fvSolution SIMPLE { consistent yes; }, reference pEqnSimple.H:27-33): rAtU = 1/(1/rAU - H1) replaces rAU in the
// pressure laplacian and the correctors; phiHbyA and HbyA carry the (rAtU - rAU) part of the old pressure gradient.
// rAt == nullptr: plain SIMPLE.
struct Simplec
{
    const double* rAt = nullptr;   // [nT]
    const double* pOld = nullptr;  // [nT] p at the start of the iteration
    const double* gPOld = nullptr; // [3*nT] its gradient
};

// H1 = -(sum of the off-diagonal coefficients)/V of the relaxed momentum matrix (fvMatrix::H1), rAtU from it
struct RAtKernel
{
    EqnView e;
    const double *rAU, *V;
    double* rAt;
    DAB_HD void operator()(int c) const
    {
        double h1 = 0.0;
        for (int k = 0; k < e.maxCF; k++) h1 -= e.off[(size_t)k * e.nC + c];
        rAt[c] = frcp(1.0 / rAU[c] - h1 / V[c]);
    }
};

struct HbyAKernel
{
    EqnView e;
    StateView s;
    RecordView r;
    const double* V;
    int nT;
    DAB_HD void operator()(int c) const
    {
        const int nC = e.nC;
        double acc[3] = {0.0, 0.0, 0.0};
        for (int k = 0; k < e.maxCF; k++)
        {
            const int n = e.cellNbr[(size_t)k * nC + c];
            if (n < 0) continue;
            const double o = e.off[(size_t)k * nC + c];
            for (int j = 0; j < 3; j++) acc[j] += o * s.U[3 * n + j];
        }
        const double rAU = r.rAU[c], iV = frcp(V[c]);
        for (int j = 0; j < 3; j++)
        {
            const double M = (e.diag[(size_t)j * nC + c] * s.U[3 * c + j] + acc[j] - e.b[(size_t)j * nC + c]) * iV;
            r.HbyA[(size_t)j * nT + c] = s.U[3 * c + j] - rAU * M;
        }
    }
};

// phiHbyA on a boundary face (constrainHbyA rule, reference pEqnSimple.H:8-19)
DAB_HD double phiHbyABoundary(const MeshView& m, const Params& q, const StateView& s, const RecordView& r, int f, int c)
{
    const int nT = m.nCtot;
    const int b = f - m.nIF, pa = m.bPatch[b];
    const int kU = q.bcKind[F_U][pa];
    const bool assignable = (kU == BC_INLET_OUTLET || kU == BC_OUTLET_INLET || kU == BC_ZERO_GRADIENT);
    if (q.constrainHbyA && !assignable)
    {
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double im = frcp(m.magSf[f]);
        const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
        BCv bu;
        double uw[3];
        mrfWallRef(m, f, q.bcVal[F_U][pa], uw);
        bcVector(kU, uw, Uc, s.phi[f], m.delta[f], nh, bu);
        return mrfBoundaryFlux(m, f, m.Sx[f] * bu.val[0] + m.Sy[f] * bu.val[1] + m.Sz[f] * bu.val[2], 1.0);
    }
    return mrfBoundaryFlux(m, f, m.Sx[f] * r.HbyA[c] + m.Sy[f] * r.HbyA[(size_t)nT + c] + m.Sz[f] * r.HbyA[(size_t)2 * nT + c], 1.0);
}

// pressure equation laplacian(rAU, p) == div(phiHbyA), assembled with the sign flipped (symmetric positive definite):
//   (sum_f g_f + sum_b g_b fr_b) p_c - sum_f g_f p_n = -sum_f s (phiHbyA_f - gf cg_f) + sum_b (g_b fr_b ref_b - phiHbyA_b)
// with g = rAU_f |S_f| delta_f and cg the non-orthogonal correction from the recorded grad(p)
template <int NF>
struct PEqnAssemble
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    EqnView e;
    Simplec sc;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        double D = 0.0, B = 0.0;
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0)
            {
                for (int kk = k; kk < m.maxCF; kk++) e.off[(size_t)kk * nC + c] = 0.0;
                break;
            }
            const int f = fr.f;
            const double mS = m.magSf[f], dl = m.delta[f];
            if (!fr.bnd)
            {
                const int o = fr.s > 0 ? c : fr.n, n = fr.s > 0 ? fr.n : c;
                const double w = m.w[f];
                double ph = 0.0, cg = 0.0;
                const double Sv[3] = {m.Sx[f], m.Sy[f], m.Sz[f]};
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                for (int j = 0; j < 3; j++)
                {
                    ph += Sv[j] * (w * r.HbyA[(size_t)j * nT + o] + (1.0 - w) * r.HbyA[(size_t)j * nT + n]);
                    cg += kv[j] * (w * r.gP[(size_t)j * nT + o] + (1.0 - w) * r.gP[(size_t)j * nT + n]);
                }
                if (m.mrfFlux) ph -= m.mrfFlux[f];
                double gam = (w * r.rAU[o] + (1.0 - w) * r.rAU[n]) * mS;
                if (sc.rAt)
                {
                    const double gamT = (w * sc.rAt[o] + (1.0 - w) * sc.rAt[n]) * mS;
                    double cgOld = 0.0;
                    for (int j = 0; j < 3; j++) cgOld += kv[j] * (w * sc.gPOld[(size_t)j * nT + o] + (1.0 - w) * sc.gPOld[(size_t)j * nT + n]);
                    ph += (gamT - gam) * (dl * (sc.pOld[n] - sc.pOld[o]) + cgOld);
                    gam = gamT;
                }
                e.off[(size_t)k * nC + c] = -gam * dl;
                D += gam * dl;
                B -= fr.s * (ph - gam * cg);
            }
            else
            {
                e.off[(size_t)k * nC + c] = 0.0;
                const int b = f - m.nIF, pa = m.bPatch[b];
                const double frp = bcFrac(q.bcKind[F_P][pa], s.phi[f]);
                double ph = phiHbyABoundary(m, q, s, r, f, c), gU = r.rAU[c] * mS;
                if (sc.rAt)
                {
                    double pv, snOld, fr_;
                    bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], sc.pOld[c], s.phi[f], dl, pv, snOld, fr_);
                    ph += (sc.rAt[c] * mS - gU) * snOld;
                    gU = sc.rAt[c] * mS;
                }
                const double gb = gU * dl * frp;
                D += gb;
                B += gb * q.bcVal[F_P][pa][0] - ph;
            }
        }
        e.diag[c] = D;
        e.b[c] = B;
    }
};

// phi = phiHbyA - pEqn.flux() (reference pEqnSimple.H:60-63): the same face flux F_f as the residual kernel FwdC
template <int NF>
struct PhiUpdate
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    double* phi;
    Simplec sc;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot;
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            if (fr.s < 0) continue;
            const int f = fr.f;
            if (!fr.bnd)
            {
                double F = faceF(m, s, r, f, c, fr.n);
                if (sc.rAt)
                {
                    // + (rAtU - rAU)_f snGrad(pOld) |Sf| of phiHbyA, - (rAtU - rAU)_f snGrad(p) |Sf| of the flux
                    const int n = fr.n;
                    const double w = m.w[f], dl = m.delta[f];
                    const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                    double cg = 0.0, cgOld = 0.0;
                    for (int j = 0; j < 3; j++)
                    {
                        cg += kv[j] * (w * r.gP[(size_t)j * nT + c] + (1.0 - w) * r.gP[(size_t)j * nT + n]);
                        cgOld += kv[j] * (w * sc.gPOld[(size_t)j * nT + c] + (1.0 - w) * sc.gPOld[(size_t)j * nT + n]);
                    }
                    const double dg = (w * (sc.rAt[c] - r.rAU[c]) + (1.0 - w) * (sc.rAt[n] - r.rAU[n])) * m.magSf[f];
                    F += dg * ((dl * (sc.pOld[n] - sc.pOld[c]) + cgOld) - (dl * (s.p[n] - s.p[c]) + cg));
                }
                phi[f] = F;
            }
            else
            {
                const int b = f - m.nIF, pa = m.bPatch[b];
                double ph = phiHbyABoundary(m, q, s, r, f, c), gU = r.rAU[c] * m.magSf[f];
                double pv, sn, fr_;
                if (sc.rAt)
                {
                    bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], sc.pOld[c], s.phi[f], m.delta[f], pv, sn, fr_);
                    ph += (sc.rAt[c] * m.magSf[f] - gU) * sn;
                    gU = sc.rAt[c] * m.magSf[f];
                }
                bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], s.p[c], s.phi[f], m.delta[f], pv, sn, fr_);
                phi[f] = ph - gU * sn;
            }
        }
    }
};

struct RelaxField // x = xOld + alpha*(x - xOld)
{
    double* x;
    const double* xOld;
    double alpha;
    DAB_HD void operator()(int c) const { x[c] = xOld[c] + alpha * (x[c] - xOld[c]); }
};

struct UCorrect // U = HbyA - rAU*grad(p); SIMPLEC: HbyA - (rAU - rAtU)*grad(pOld) - rAtU*grad(p)
{
    RecordView r;
    double* U;
    int nT;
    Simplec sc;
    DAB_HD void operator()(int c) const
    {
        if (sc.rAt)
        {
            const double a = r.rAU[c] - sc.rAt[c];
            for (int j = 0; j < 3; j++)
                U[3 * c + j] = r.HbyA[(size_t)j * nT + c] - a * sc.gPOld[(size_t)j * nT + c] - sc.rAt[c] * r.gP[(size_t)j * nT + c];
            return;
        }
        for (int j = 0; j < 3; j++) U[3 * c + j] = r.HbyA[(size_t)j * nT + c] - r.rAU[c] * r.gP[(size_t)j * nT + c];
    }
};

// nuTilda equation (DASpalartAllmaras.C:452-462): div(phi,nt) - laplacian(DnuTildaEff,nt) - Cb2/sigma |grad nt|^2
// == Cb1 Stilda nt - Sp(Cw1 fw nt/y^2, nt), relaxed
template <int NF>
struct NutEqnAssemble
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    EqnView e;
    double alphaN;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const int schN = q.divNut;
        const double ntc = s.nt[c];
        const double Gc = (ntc + q.nu) * (1.0 / SA::sigma);
        double gUc[9], gNc[3];
        for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
        for (int i = 0; i < 3; i++) gNc[i] = r.gNt[(size_t)i * nT + c];
        double D0 = 0.0, sumOff = 0.0, X = 0.0, ic = 0.0, aic = 0.0;
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0)
            {
                for (int kk = k; kk < m.maxCF; kk++) e.off[(size_t)kk * nC + c] = 0.0;
                break;
            }
            const int f = fr.f;
            const double mf = fr.s * s.phi[f];
            const double mS = m.magSf[f], dl = m.delta[f];
            if (!fr.bnd)
            {
                const int n = fr.n;
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f], wn = 1.0 - wc;
                const bool pos0 = s.phi[f] >= 0.0;
                const double wup = fr.s > 0 ? (pos0 ? 1.0 : 0.0) : (pos0 ? 0.0 : 1.0);
                const double ntn = s.nt[n];
                const double wp = schN == DIV_LINEAR ? wc : wup;
                const double a = wp * mf;
                const double gf = (wc * Gc + wn * (ntn + q.nu) * (1.0 / SA::sigma)) * mS;
                const double g = gf * dl;
                const double off = mf - a - g;
                e.off[(size_t)k * nC + c] = off;
                D0 += a + g - mf;
                sumOff += fabs(off);
                if (schN == DIV_LINEAR_UPWIND)
                {
                    const bool ownUp = s.phi[f] > 0.0;
                    const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                    const int u = cUp ? c : n;
                    const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                    double corr = 0.0;
                    for (int i = 0; i < 3; i++) corr += d[i] * r.gNt[(size_t)i * nT + u];
                    X += mf * corr;
                }
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                double cg = 0.0;
                for (int i = 0; i < 3; i++) cg += kv[i] * (wc * gNc[i] + wn * r.gNt[(size_t)i * nT + n]);
                X -= fr.s * gf * cg;
            }
            else
            {
                e.off[(size_t)k * nC + c] = 0.0;
                const int b = f - m.nIF, pa = m.bPatch[b];
                double ntb, sngN, frN;
                bcScalar(q.bcKind[F_NUTILDA][pa], q.bcVal[F_NUTILDA][pa][0], ntc, mf, dl, ntb, sngN, frN);
                const double Gs = (ntb + q.nu) * (1.0 / SA::sigma) * mS;
                const double icf = mf * (1.0 - frN) + Gs * frN * dl;
                ic += icf;
                aic += fabs(icf);
                D0 -= mf; // bounded
                X += mf * ntb - Gs * sngN - icf * ntc;
            }
        }
        const double V = m.V[c], y = m.yWall[c];
        // cell-local sources: the destruction term is implicit (fvm::Sp), the rest explicit
        const double P = saSource(ntc, q.nu, y, gUc, gNc, q.saFv3); // -Cb2/sigma|grad nt|^2 - Cb1 St nt + Cw1 fw nt^2/y^2
        const double St = saStilda(ntc, q.nu, y, gUc, q.saFv3);
        const double mg2 = gNc[0] * gNc[0] + gNc[1] * gNc[1] + gNc[2] * gNc[2];
        const double expl = -(SA::Cb2 * (1.0 / SA::sigma)) * mg2 - SA::Cb1 * St * ntc; // explicit part of P
        const double sp = ntc != 0.0 ? (P - expl) / ntc : 0.0;                  // Cw1 fw nt / y^2
        D0 += V * sp;
        X += V * expl;
        // fvMatrix::relax (scalar)
        const double D1 = D0 + aic;
        const double aD1 = fabs(D1);
        const double D2 = aD1 > sumOff ? aD1 : sumOff;
        const double Dn = D2 * frcp(alphaN) - ic;
        e.diag[c] = Dn + ic;
        e.b[c] = -X + (Dn - D0) * ntc;
    }
};

struct BoundField // DAUtility::boundVar
{
    double* x;
    double lo, hi;
    DAB_HD void operator()(int c) const
    {
        const double v = x[c];
        x[c] = v < lo ? lo : (v > hi ? hi : v);
    }
};

// ---- pressure solver: PCG with a multicolour symmetric Gauss-Seidel preconditioner -----------------------------
struct SpmvEll // y = A x (A = diag + off)
{
    EqnView e;
    const double* x;
    double* y;
    DAB_HD void operator()(int c) const
    {
        const int nC = e.nC;
        double acc = e.diag[c] * x[c];
        for (int k = 0; k < e.maxCF; k++)
        {
            const int n = e.cellNbr[(size_t)k * nC + c];
            if (n >= 0) acc += e.off[(size_t)k * nC + c] * x[n];
        }
        y[c] = acc;
    }
};

// one colour of the forward ((D+L) y = r) or backward ((D+U) z = D y) sweep; cells of the colour are list[0..n)
struct SgsColour
{
    EqnView e;
    const int32_t* list;
    const int32_t* colourOf;
    int colour, backward;
    const double* rhs; // forward: r; backward: unused
    double* z;         // forward: y written; backward: updated in place
    DAB_HD void operator()(int t) const
    {
        const int c = list[t], nC = e.nC;
        double acc = 0.0;
        for (int k = 0; k < e.maxCF; k++)
        {
            const int n = e.cellNbr[(size_t)k * nC + c];
            if (n < 0 || n >= nC) continue;
            const int cn = colourOf[n];
            if (backward ? cn > colour : cn < colour) acc += e.off[(size_t)k * nC + c] * z[n];
        }
        if (backward) z[c] -= acc * frcp(e.diag[c]);
        else z[c] = (rhs[c] - acc) * frcp(e.diag[c]);
    }
};

// PCG scalars live on the device (no host round trip per iteration): S[0] rz, S[1] rzOld, S[2] dq, S[3] sum|r|, S[4] alpha, S[5] beta
struct PcgScalarBeta
{
    double* S;
    int first;
    DAB_HD void operator()(int) const
    {
        S[5] = first ? 0.0 : S[0] / S[1];
        S[1] = S[0];
    }
};
struct PcgScalarAlpha
{
    double* S;
    DAB_HD void operator()(int) const { S[4] = S[2] > 0.0 ? S[0] / S[2] : 0.0; }
};
struct PcgUpdate1 // x += alpha d; r -= alpha q; absr = |r|
{
    const double* S;
    const double *d, *q;
    double *x, *r, *absr;
    DAB_HD void operator()(int c) const
    {
        const double a = S[4];
        x[c] += a * d[c];
        const double v = r[c] - a * q[c];
        r[c] = v;
        absr[c] = fabs(v);
    }
};
struct PcgUpdate2 // d = z + beta d
{
    const double* S;
    const double* z;
    double* d;
    DAB_HD void operator()(int c) const
    {
        const double beta = S[5];
        d[c] = beta == 0.0 ? z[c] : z[c] + beta * d[c];
    }
};
struct SpmvEllProd // y = A x, prod = x*y
{
    EqnView e;
    const double* x;
    double *y, *prod;
    DAB_HD void operator()(int c) const
    {
        const int nC = e.nC;
        double acc = e.diag[c] * x[c];
        for (int k = 0; k < e.maxCF; k++)
        {
            const int n = e.cellNbr[(size_t)k * nC + c];
            if (n >= 0) acc += e.off[(size_t)k * nC + c] * x[n];
        }
        y[c] = acc;
        prod[c] = acc * x[c];
    }
};

// ---- aggregation coarse space of the pressure preconditioner: z += P (P^T A P)^-1 P^T r ------------------------
// Galerkin operator, one thread per aggregate (the thread owns its row: deterministic, no atomics)
struct CoarseGalerkin
{
    EqnView e;
    const int32_t* aggOf;
    const int32_t* cells;    // cells sorted by aggregate
    const int32_t* aggStart; // [nAgg+1]
    int nAgg;
    double* Ac;              // [nAgg][nAgg], zeroed
    DAB_HD void operator()(int a) const
    {
        const int nC = e.nC;
        double* row = Ac + (size_t)a * nAgg;
        for (int i = aggStart[a]; i < aggStart[a + 1]; i++)
        {
            const int c = cells[i];
            row[a] += e.diag[c];
            for (int k = 0; k < e.maxCF; k++)
            {
                const int n = e.cellNbr[(size_t)k * nC + c];
                if (n >= 0 && n < nC) row[aggOf[n]] += e.off[(size_t)k * nC + c];
            }
        }
    }
};
// in-place Gauss-Jordan inversion without pivoting (symmetric positive definite operator), step k in two kernels
struct GjStep1 // save column k, scale row k
{
    double* A;
    double* colk;
    int n, k;
    DAB_HD void operator()(int j) const
    {
        const double p = A[(size_t)k * n + k];
        colk[j] = A[(size_t)j * n + k];
        if (j != k) A[(size_t)k * n + j] /= p;
    }
};
struct GjStep2 // eliminate: thread per element
{
    double* A;
    const double* colk;
    int n, k;
    DAB_HD void operator()(int t) const
    {
        const int i = t / n, j = t - i * n;
        const double p = colk[k];
        if (i == k)
        {
            if (j == k) A[(size_t)k * n + k] = 1.0 / p;
            return;
        }
        const double f = colk[i];
        if (j == k) A[(size_t)i * n + k] = -f / p;
        else A[(size_t)i * n + j] -= f * A[(size_t)k * n + j];
    }
};
struct CoarseApply // yc = Ainv rc (Ainv symmetric: column access is coalesced)
{
    const double* Ainv;
    const double* rc;
    int n;
    double* yc;
    DAB_HD void operator()(int i) const
    {
        double s = 0.0;
        for (int j = 0; j < n; j++) s += Ainv[(size_t)j * n + i] * rc[j];
        yc[i] = s;
    }
};
struct TransposeSq // At = A^T (n x n): a nonsymmetric inverse read by CoarseApply's coalesced column access
{
    const double* A;
    int n;
    double* At;
    DAB_HD void operator()(int t) const
    {
        const int i = t / n, j = t - i * n;
        At[(size_t)j * n + i] = A[t];
    }
};
struct CoarseProlongAdd // z[c] += yc[agg[c]]
{
    const double* yc;
    const int32_t* aggOf;
    double* z;
    DAB_HD void operator()(int c) const { z[c] += yc[aggOf[c]]; }
};

struct PcgProducts // out0 = r*z (or d*q), out1 = |r|
{
    const double *a, *b, *r;
    double *out0, *out1;
    DAB_HD void operator()(int c) const
    {
        out0[c] = a[c] * b[c];
        if (out1) out1[c] = fabs(r[c]);
    }
};
struct ResidualOf // r = b - q
{
    const double *b, *q;
    double* r;
    DAB_HD void operator()(int c) const { r[c] = b[c] - q[c]; }
};

// ---- BiCGStab (van der Vorst) for the nonsymmetric transonic pressure equation, scalars on the device:
// S[0] rho = (rhat, r), S[1] rho of the previous iteration, S[2] alpha, S[3] omega, S[4] beta, S[5] (rhat, v), S[6] (t, s), S[7] (t, t),
// S[8] sum |r|, S[9] breakdown flag (rho, (rhat, v) or (t, t) vanished): once set, alpha = omega = 0 leave x alone until the host
// restarts from the true residual
constexpr double BICG_VSMALL = 1e-300;
struct BicgBeta
{
    double* S;
    int first;
    DAB_HD void operator()(int) const
    {
        if (!(fabs(S[0]) > BICG_VSMALL)) S[9] = 1.0;
        S[4] = (first || S[9] != 0.0) ? 0.0 : (S[0] / S[1]) * (S[2] / S[3]);
        S[1] = S[0];
    }
};
struct BicgAlpha
{
    double* S;
    DAB_HD void operator()(int) const
    {
        if (!(fabs(S[5]) > BICG_VSMALL)) S[9] = 1.0;
        S[2] = S[9] != 0.0 ? 0.0 : S[0] / S[5];
    }
};
struct BicgOmega
{
    double* S;
    DAB_HD void operator()(int) const
    {
        if (!(S[7] > BICG_VSMALL)) S[9] = 1.0;
        S[3] = S[9] != 0.0 ? 0.0 : S[6] / S[7];
    }
};
struct BicgDir // p = r + beta (p - omega v)
{
    const double* S;
    const double *r, *v;
    double* p;
    DAB_HD void operator()(int c) const
    {
        const double beta = S[4];
        p[c] = beta == 0.0 ? r[c] : r[c] + beta * (p[c] - S[3] * v[c]);
    }
};
struct BicgHalf // x += alpha y; s = r - alpha v (in r)
{
    const double* S;
    const double *y, *v;
    double *x, *r;
    DAB_HD void operator()(int c) const
    {
        const double a = S[2];
        x[c] += a * y[c];
        r[c] -= a * v[c];
    }
};
struct BicgFull // x += omega z; r = s - omega t; absr = |r|
{
    const double* S;
    const double *z, *t;
    double *x, *r, *absr;
    DAB_HD void operator()(int c) const
    {
        const double w = S[3];
        x[c] += w * z[c];
        const double v = r[c] - w * t[c];
        r[c] = v;
        absr[c] = fabs(v);
    }
};
struct SpmvEllDot2 // t = A z, out0 = t*s, out1 = t*t
{
    EqnView e;
    const double *z, *s;
    double *t, *out0, *out1;
    DAB_HD void operator()(int c) const
    {
        const int nC = e.nC;
        double acc = e.diag[c] * z[c];
        for (int k = 0; k < e.maxCF; k++)
        {
            const int n = e.cellNbr[(size_t)k * nC + c];
            if (n >= 0) acc += e.off[(size_t)k * nC + c] * z[n];
        }
        t[c] = acc;
        out0[c] = acc * s[c];
        out1[c] = acc * acc;
    }
};
struct FillConst
{
    double* x;
    double v;
    DAB_HD void operator()(int c) const { x[c] = v; }
};

// result of one solvePrimal call (the numbers the reference prints per equation, DAUtility::primalResidualControl)
struct PrimalStats
{
    int iterations = 0, converged = 0, pIterations = 0;
    double maxRes = 0.0, resU[3] = {0, 0, 0}, resP = 0.0, resN = 0.0, resE = 0.0, sec = 0.0;
};

struct SegControl
{
    double tol = 1e-12, relTol = 0.1;
    int maxIter = 1000;
};

// options and work arrays of the primal solver
struct Primal
{
    // system/fvSolution + DAOption (reference dafoam/pyDAFoam.py: primalMinResTol, primalMinResTolDiff, primalMinIters, primalVarBounds)
    double alphaP = 0.3, alphaN = 0.7, alphaE = 0.7, alphaRho = 0.05;
    double minResTol = 1e-8, minResTolDiff = 1e2;
    int minIters = 1, maxIters = 1000, nNonOrth = 0, printInterval = 100;
    bool consistent = false; // SIMPLEC
    SegControl cU, cP, cN, cE;
    double ntMin = 1e-16, ntMax = 1e16;
    double pMin = 20000.0, pMax = 500000.0, TMin = 100.0, TMax = 1000.0, UMax = 1000.0; // DAOption primalVarBounds (compressible)
    double rhoMin = 0.2, rhoMax = 5.0;
    double alphaPEqn = 0.0; // relaxationFactors.equations.p of the transonic pressure equation; 0: not relaxed
    bool allocated = false;
    DevBuf<double> uOff, uDiag, uB, pOff, pDiag, pB, nOff, nDiag, nB;
    DevBuf<double> Utmp, pOld, ntTmp, red, ones, r, z, d, q, eOff, eDiag, eB, heTmp, rAt, gPOld;
    DevBuf<double> pFace, bRhat, bDir, bV, bT, dAcT; // transonic corrector: assembly record, BiCGStab vectors, transposed coarse inverse
    DevBuf<int32_t> dColourOf, dColourList;
    std::vector<int> colourStart; // [nColours+1] into dColourList
    // pressure coarse space
    int nAgg = -1, coarseRefresh = 10, nChunks = 0; // nAgg < 0: choose from the mesh size; 0: off
    bool coarseValid = false;
    DevBuf<int32_t> dAggOf, dAggCells, dAggStart, dChunkStart, dAggChunkOff;
    DevBuf<double> dAc, dColk, dRc, dYc, dPartial, dS;
    VecOps* ops = nullptr;
};

} // namespace dab
