// DARhoSimpleFoam primal: equation-assembly kernels of the compressible SIMPLE loop (reference
// src/adjoint/DASolver/DARhoSimpleFoam/{UEqnRhoSimple,EEqnRhoSimple,pEqnRhoSimple}.H, DARhoSimpleFoam.C:106-164).
// Same construction as primal_kernels.hpp: each equation is assembled by one cell-parallel gather into a per-cell ELL row
// with the discretisation of the compressible residual kernels (comp_kernels.hpp), so the fixed point is R(W) = 0.
// The density is rho = psi*p evaluated from the current (p, T) whenever the closures are refreshed (the reference keeps a
// relaxed rho field between iterations; both have the same fixed point).
#pragma once
#include "comp_kernels.hpp"
#include "primal_kernels.hpp"

namespace dab
{

template <int NF>
struct cUEqnAssemble
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
        const double muEc = r.muE[c];
        double gUc[9];
        for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
        const double trc = gUc[0] + gUc[4] + gUc[8];
        double D0 = 0.0, sumOff = 0.0, X[3] = {0.0, 0.0, 0.0};
        double icMax = 0.0, icMin = 0.0, icAvg = 0.0, icS[3] = {0.0, 0.0, 0.0};
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
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
                const double muEn = r.muE[n];
                const double wp = schU == DIV_LINEAR ? wc : wup;
                const double a = wp * mf;
                const double gf = (wc * muEc + wn * muEn) * mS;
                const double g = gf * dl;
                const double off = mf - a - g;
                e.off[(size_t)k * nC + c] = off;
                D0 += a + g - mf;
                sumOff += fabs(off);
                double gUn[9];
                for (int i = 0; i < 9; i++) gUn[i] = r.gU[(size_t)i * nT + n];
                if (schU == DIV_LINEAR_UPWIND || schU == DIV_LINEAR_UPWIND_V)
                {
                    const bool ownUp = s.phi[f] > 0.0;
                    const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                    double gu[9]; // per-element selects: a pointer into either array would put both in local memory
                    for (int i = 0; i < 9; i++) gu[i] = cUp ? gUc[i] : gUn[i];
                    const int u = cUp ? c : n;
                    const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                    double corr[3];
                    for (int j = 0; j < 3; j++) corr[j] = d[0] * gu[j * 3 + 0] + d[1] * gu[j * 3 + 1] + d[2] * gu[j * 3 + 2];
                    if (schU == DIV_LINEAR_UPWIND_V)
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
                    const double tc = muEc * (Sv[0] * gUc[0 * 3 + j] + Sv[1] * gUc[1 * 3 + j] + Sv[2] * gUc[2 * 3 + j] - (2.0 / 3.0) * trc * Sv[j]);
                    const double tn = muEn * (Sv[0] * gUn[0 * 3 + j] + Sv[1] * gUn[1 * 3 + j] + Sv[2] * gUn[2 * 3 + j] - (2.0 / 3.0) * trn * Sv[j]);
                    X[j] -= fr.s * (wc * tc + wn * tn);
                }
            }
            else
            {
                e.off[(size_t)k * nC + c] = 0.0;
                BoundaryPoint bp;
                boundaryPoint<true>(m, q, s, r, f, c, bp);
                const double im = frcp(mS);
                const double nh[3] = {Sv[0] * im, Sv[1] * im, Sv[2] * im};
                const double G = bp.muE * mS;
                D0 -= mf;
                double mx = 0.0, mn = 0.0, av = 0.0;
                for (int j = 0; j < 3; j++)
                {
                    const double ic = mf * bp.bu.vic[j] - G * bp.bu.gic[j];
                    const double aic = fabs(ic);
                    if (j == 0) { mx = aic; mn = ic; }
                    else { mx = aic > mx ? aic : mx; mn = ic < mn ? ic : mn; }
                    av += ic;
                    icS[j] += ic;
                    X[j] += mf * bp.bu.val[j] - G * bp.bu.sng[j] - ic * Uc[j];
                }
                icMax += mx; icMin += mn; icAvg += av / 3.0;
                double Gb[9];
                for (int j = 0; j < 3; j++)
                {
                    const double nG = nh[0] * gUc[j * 3 + 0] + nh[1] * gUc[j * 3 + 1] + nh[2] * gUc[j * 3 + 2];
                    for (int i = 0; i < 3; i++) Gb[j * 3 + i] = gUc[j * 3 + i] + nh[i] * (bp.bu.sng[j] - nG);
                }
                const double trb = Gb[0] + Gb[4] + Gb[8];
                for (int j = 0; j < 3; j++)
                {
                    const double x = Sv[0] * Gb[0 * 3 + j] + Sv[1] * Gb[1 * 3 + j] + Sv[2] * Gb[2 * 3 + j] - (2.0 / 3.0) * trb * Sv[j];
                    X[j] -= bp.muE * x;
                }
            }
        }
        const double V = m.V[c];
        const double D1 = D0 + icMax;
        const double aD1 = fabs(D1);
        const double D2 = aD1 > sumOff ? aD1 : sumOff;
        const double Dn = D2 * frcp(q.alphaU) - icMin;
        r.rAU[c] = V * frcp(Dn + icAvg);
        double cor[3] = {0.0, 0.0, 0.0}; // MRF.DDt(rho, U), explicit
        if (m.mrfCell && m.mrfCell[c])
        {
            const double* w = m.mrfOmega;
            const double rc = r.rho[c];
            cor[0] = rc * (w[1] * Uc[2] - w[2] * Uc[1]);
            cor[1] = rc * (w[2] * Uc[0] - w[0] * Uc[2]);
            cor[2] = rc * (w[0] * Uc[1] - w[1] * Uc[0]);
        }
        for (int j = 0; j < 3; j++)
        {
            e.diag[(size_t)j * nC + c] = Dn + icS[j];
            e.b[(size_t)j * nC + c] = -X[j] + (Dn - D0) * Uc[j] + (m.fvS ? V * m.fvS[(size_t)j * nC + c] : 0.0) - V * cor[j];
        }
        (void)NF;
    }
};

// energy equation for he: div(phi,he) + div(phi,Ekp|K) - laplacian(alphaEff,he), relaxed
template <int NF>
struct cEEqnAssemble
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    EqnView e;
    double alphaE;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const int schE = q.divE;
        const double heA = q.heIsE ? (q.Cp - q.Rg) : q.Cp;
        const double hec = r.he[c], aEc = r.aE[c], Ekc = r.Ek[c];
        double gHc[3];
        for (int i = 0; i < 3; i++) gHc[i] = r.gHe[(size_t)i * nT + c];
        double D0 = 0.0, sumOff = 0.0, X = 0.0, ic = 0.0, aic = 0.0;
        double twc[3] = {0.0, 0.0, 0.0}, gUt[9]; // DATurboFoam enthalpy form: explicit - div(Teff & U) + div(p (U - URel))
        if (q.turboH)
        {
            for (int i = 0; i < 9; i++) gUt[i] = r.gU[(size_t)i * nT + c];
            const double uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
            double vr[3];
            const bool inZone = m.mrfCell && m.mrfCell[c];
            if (inZone) mrfVelocityAt(m, m.Cx[c], m.Cy[c], m.Cz[c], vr);
            turboWork(gUt, r.muE[c], uc, s.p[c], inZone ? vr : nullptr, twc);
        }
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
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
                if (q.turboH)
                {
                    double gn[9], twn[3], vr[3];
                    for (int i = 0; i < 9; i++) gn[i] = r.gU[(size_t)i * nT + n];
                    const double un[3] = {s.U[3 * n], s.U[3 * n + 1], s.U[3 * n + 2]};
                    const bool inZone = m.mrfCell && m.mrfCell[n];
                    if (inZone) mrfVelocityAt(m, m.Cx[n], m.Cy[n], m.Cz[n], vr);
                    turboWork(gn, r.muE[n], un, s.p[n], inZone ? vr : nullptr, twn);
                    X -= fr.s * (m.Sx[f] * (wc * twc[0] + wn * twn[0]) + m.Sy[f] * (wc * twc[1] + wn * twn[1]) + m.Sz[f] * (wc * twc[2] + wn * twn[2]));
                }
                const bool pos0 = s.phi[f] >= 0.0;
                const double wup = fr.s > 0 ? (pos0 ? 1.0 : 0.0) : (pos0 ? 0.0 : 1.0);
                const double wp = schE == DIV_LINEAR ? wc : wup;
                const double a = wp * mf;
                const double gf = (wc * aEc + wn * r.aE[n]) * mS;
                const double g = gf * dl;
                const double off = mf - a - g;
                e.off[(size_t)k * nC + c] = off;
                D0 += a + g - mf;
                sumOff += fabs(off);
                if (schE == DIV_LINEAR_UPWIND)
                {
                    const bool ownUp = s.phi[f] > 0.0;
                    const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                    const int u = cUp ? c : n;
                    const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                    double corr = 0.0;
                    for (int i = 0; i < 3; i++) corr += d[i] * r.gHe[(size_t)i * nT + u];
                    X += mf * corr;
                }
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                double cg = 0.0;
                for (int i = 0; i < 3; i++) cg += kv[i] * (wc * gHc[i] + wn * r.gHe[(size_t)i * nT + n]);
                X -= fr.s * gf * cg;
                const double wk = q.divEkp == DIV_LINEAR ? wc : wup;
                X += mf * (wk * Ekc + (1.0 - wk) * r.Ek[n] - Ekc);
            }
            else
            {
                e.off[(size_t)k * nC + c] = 0.0;
                BoundaryPoint bp;
                boundaryPoint<true>(m, q, s, r, f, c, bp);
                const double sngH = heA * bp.sngT;
                const double icf = mf * (1.0 - bp.frT) + bp.aE * mS * bp.frT * dl;
                ic += icf;
                aic += fabs(icf);
                D0 -= mf;
                X += mf * bp.th.he - bp.aE * mS * sngH - icf * hec;
                X += mf * (bp.Ek - Ekc);
                if (q.turboH)
                {
                    const double im = frcp(mS);
                    const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
                    double Gb[9], twb[3], vr[3];
                    for (int j = 0; j < 3; j++)
                    {
                        const double nG = nh[0] * gUt[j * 3 + 0] + nh[1] * gUt[j * 3 + 1] + nh[2] * gUt[j * 3 + 2];
                        for (int i = 0; i < 3; i++) Gb[j * 3 + i] = gUt[j * 3 + i] + nh[i] * (bp.bu.sng[j] - nG);
                    }
                    const bool onZone = m.mrfType && m.mrfType[f - m.nIF] != 0;
                    if (onZone) mrfVelocityAt(m, m.Cfx[f], m.Cfy[f], m.Cfz[f], vr);
                    turboWork(Gb, bp.muE, bp.bu.val, bp.p, onZone ? vr : nullptr, twb);
                    X -= m.Sx[f] * twb[0] + m.Sy[f] * twb[1] + m.Sz[f] * twb[2];
                }
            }
        }
        if (m.fvS) X -= m.V[c] * (m.fvS[c] * s.U[3 * c] + m.fvS[(size_t)nC + c] * s.U[3 * c + 1] + m.fvS[(size_t)2 * nC + c] * s.U[3 * c + 2]);
        const double D1 = D0 + aic;
        const double aD1 = fabs(D1);
        const double D2 = aD1 > sumOff ? aD1 : sumOff;
        const double Dn = D2 * frcp(alphaE) - ic;
        e.diag[c] = Dn + ic;
        e.b[c] = -X + (Dn - D0) * hec;
        (void)NF;
    }
};

struct RhoRelax // rho <- rho + alpha (psi p - rho)   (rho = thermo.rho(); rho.relax())
{
    Params q;
    StateView s;
    double* rho;
    double alpha;
    DAB_HD void operator()(int c) const
    {
        const double rn = s.p[c] * frcp(q.Rg * s.T[c]);
        rho[c] += alpha * (rn - rho[c]);
    }
};

struct TFromHe // T = (he - heB)/heA on the owned cells
{
    Params q;
    const double* he;
    double* T;
    DAB_HD void operator()(int c) const
    {
        const double heA = q.heIsE ? (q.Cp - q.Rg) : q.Cp;
        T[c] = (he[c] + q.Cp * q.TRef) * frcp(heA);
    }
};

// phiHbyA on a boundary face without the density factor (constrainHbyA rule)
DAB_HD double cPhBoundary(const MeshView& m, const Params& q, const RecordView& r, const BoundaryPoint& bp, int f, int c)
{
    const int nT = m.nCtot;
    const int kU = q.bcKind[F_U][m.bPatch[f - m.nIF]];
    const bool assignable = (kU == BC_INLET_OUTLET || kU == BC_OUTLET_INLET || kU == BC_ZERO_GRADIENT);
    if (q.constrainHbyA && !assignable)
        return mrfBoundaryFlux(m, f, m.Sx[f] * bp.bu.val[0] + m.Sy[f] * bp.bu.val[1] + m.Sz[f] * bp.bu.val[2], 1.0);
    return mrfBoundaryFlux(m, f, m.Sx[f] * r.HbyA[c] + m.Sy[f] * r.HbyA[(size_t)nT + c] + m.Sz[f] * r.HbyA[(size_t)2 * nT + c], 1.0);
}

// pressure equation div(phiHbyA) - laplacian(rho rAU, p) = 0, sign-flipped to the SPD form
template <int NF>
struct cPEqnAssemble
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    EqnView e;
    Simplec sc; // DATurboFoam / consistent: AtU = AU - H1 (reference pEqnTurbo.H:13-15, 64-70)
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        double D = 0.0, B = 0.0;
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
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
                const double rhof = w * r.rho[o] + (1.0 - w) * r.rho[n];
                double gam = (w * r.rho[o] * r.rAU[o] + (1.0 - w) * r.rho[n] * r.rAU[n]) * mS;
                double phr = rhof * ph;
                if (sc.rAt)
                {
                    // phiHbyA += interpolate(rho/AtU - rho/AU) snGrad(p) |Sf|, laplacian(rho/AtU, p)
                    const double gamT = (w * r.rho[o] * sc.rAt[o] + (1.0 - w) * r.rho[n] * sc.rAt[n]) * mS;
                    double cgOld = 0.0;
                    for (int j = 0; j < 3; j++) cgOld += kv[j] * (w * sc.gPOld[(size_t)j * nT + o] + (1.0 - w) * sc.gPOld[(size_t)j * nT + n]);
                    phr += (gamT - gam) * (dl * (sc.pOld[n] - sc.pOld[o]) + cgOld);
                    gam = gamT;
                }
                e.off[(size_t)k * nC + c] = -gam * dl;
                D += gam * dl;
                B -= fr.s * (phr - gam * cg);
            }
            else
            {
                e.off[(size_t)k * nC + c] = 0.0;
                BoundaryPoint bp;
                boundaryPoint<false>(m, q, s, r, f, c, bp);
                double gU = bp.th.rho * r.rAU[c] * mS, phr = bp.th.rho * cPhBoundary(m, q, r, bp, f, c);
                if (sc.rAt)
                {
                    const int pa = m.bPatch[f - m.nIF];
                    double pv, snOld, fr_;
                    bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], sc.pOld[c], s.phi[f], dl, pv, snOld, fr_);
                    const double gT = bp.th.rho * sc.rAt[c] * mS;
                    phr += (gT - gU) * snOld;
                    gU = gT;
                }
                const double gb = gU * dl * bp.frP;
                D += gb;
                B += gb * q.bcVal[F_P][m.bPatch[f - m.nIF]][0] - phr;
            }
        }
        e.diag[c] = D;
        e.b[c] = B;
        (void)NF;
    }
};

template <int NF>
struct cPhiUpdate
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
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
            if (fr.f < 0) break;
            if (fr.s < 0) continue;
            const int f = fr.f;
            if (!fr.bnd)
            {
                double F = cFaceF(m, q, s, r, f, c, fr.n);
                if (sc.rAt)
                {
                    const int n = fr.n;
                    const double w = m.w[f], dl = m.delta[f];
                    const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                    double cg = 0.0, cgOld = 0.0;
                    for (int j = 0; j < 3; j++)
                    {
                        cg += kv[j] * (w * r.gP[(size_t)j * nT + c] + (1.0 - w) * r.gP[(size_t)j * nT + n]);
                        cgOld += kv[j] * (w * sc.gPOld[(size_t)j * nT + c] + (1.0 - w) * sc.gPOld[(size_t)j * nT + n]);
                    }
                    const double dg = (w * r.rho[c] * (sc.rAt[c] - r.rAU[c]) + (1.0 - w) * r.rho[n] * (sc.rAt[n] - r.rAU[n])) * m.magSf[f];
                    F += dg * ((dl * (sc.pOld[n] - sc.pOld[c]) + cgOld) - (dl * (s.p[n] - s.p[c]) + cg));
                }
                phi[f] = F;
            }
            else
            {
                BoundaryPoint bp;
                boundaryPoint<false>(m, q, s, r, f, c, bp);
                double gU = bp.th.rho * r.rAU[c] * m.magSf[f], phr = bp.th.rho * cPhBoundary(m, q, r, bp, f, c);
                if (sc.rAt)
                {
                    const int pa = m.bPatch[f - m.nIF];
                    double pv, snOld, fr_;
                    bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], sc.pOld[c], s.phi[f], m.delta[f], pv, snOld, fr_);
                    const double gT = bp.th.rho * sc.rAt[c] * m.magSf[f];
                    phr += (gT - gU) * snOld;
                    gU = gT;
                }
                phi[f] = phr - gU * bp.sngP;
            }
        }
        (void)NF;
    }
};

// rho = thermo.rho() = psi p, bounded (DAUtility::boundVar); the transonic corrector does not relax it (pEqnTurbo.H:1-8)
struct RhoThermo
{
    Params q;
    StateView s;
    double* rho;
    double lo, hi;
    DAB_HD void operator()(int c) const
    {
        const double rn = s.p[c] * frcp(q.Rg * s.T[c]);
        rho[c] = rn < lo ? lo : (rn > hi ? hi : rn);
    }
};

// div(phid,p) face weight of the owner's p: the transonic branch of cFaceF, evaluated on the current p (the limiter is frozen in
// the matrix, as fvm::div does)
DAB_HD double cPhidWeight(const MeshView& m, const Params& q, const StateView& s, const RecordView& r, double phid, int f, int o, int n)
{
    const double w = m.w[f];
    if (q.divPhidP == DIV_LINEAR) return w;
    if (q.divPhidP == DIV_LIMITED_LINEAR)
    {
        double dl, gf, gc;
        bool fb;
        const double lim = limitedLinearLimiter(m, s, r, q.phidK, phid > 0.0, o, n, dl, gf, gc, fb);
        return lim * w + (1.0 - lim) * (phid >= 0.0 ? 1.0 : 0.0);
    }
    return phid >= 0.0 ? 1.0 : 0.0;
}

// phid = psi_f (S_f.HbyA_f - relative-frame flux) and gam = (rho rAU)_f of an internal face: the same arithmetic as cFaceF
DAB_HD void cPhidFace(const MeshView& m, const Params& q, const StateView& s, const RecordView& r, int f, int o, int n, double& phid,
                      double& gam, double& cg)
{
    const int nT = m.nCtot;
    const double w = m.w[f];
    double ph = 0.0;
    cg = 0.0;
    const double Sv[3] = {m.Sx[f], m.Sy[f], m.Sz[f]};
    const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
    for (int j = 0; j < 3; j++)
    {
        ph += Sv[j] * (w * r.HbyA[(size_t)j * nT + o] + (1.0 - w) * r.HbyA[(size_t)j * nT + n]);
        cg += kv[j] * (w * r.gP[(size_t)j * nT + o] + (1.0 - w) * r.gP[(size_t)j * nT + n]);
    }
    gam = w * r.rho[o] * r.rAU[o] + (1.0 - w) * r.rho[n] * r.rAU[n];
    if (m.mrfFlux) ph -= m.mrfFlux[f];
    phid = (w * frcp(q.Rg * s.T[o]) + (1.0 - w) * frcp(q.Rg * s.T[n])) * ph;
}

// transonic pressure equation (pEqnTurbo.H transonic branch): fvm::div(phid, p) - fvm::laplacian(rho rAU, p) with an explicit
// non-orthogonal correction, row c = sum over its faces of s_f F_f, F_f the transonic face flux of cFaceF.  Boundary faces:
// F_b = psi_b p_b ph - rho_b rAU_c |S_f| snGrad(p)_b with p_b, snGrad(p)_b linear in p_c through bcScalar.  Not symmetric.
// pEqn.relax() (relaxationFactors.equations.p) when alphaEqn > 0, with the scalar fvMatrix::relax rule of cEEqnAssemble.
// face[] records what pEqn.flux() needs from the assembly: the owner's div(phid,p) weight of internal faces, rho_b of boundary faces.
template <int NF>
struct cPEqnTransonic
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    EqnView e;
    double alphaEqn;
    double* face; // [nF]
    DAB_HD void operator()(int c) const
    {
        const int nC = e.nC;
        double D0 = 0.0, sumOff = 0.0, B = 0.0, ic = 0.0, aic = 0.0;
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
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
                double phid, gam, cg;
                cPhidFace(m, q, s, r, f, o, n, phid, gam, cg);
                const double wf = cPhidWeight(m, q, s, r, phid, f, o, n);
                if (fr.s > 0) face[f] = wf;
                const double wc = fr.s > 0 ? wf : 1.0 - wf;
                const double mphid = fr.s * phid, g = gam * mS * dl;
                const double off = mphid * (1.0 - wc) - g;
                e.off[(size_t)k * nC + c] = off;
                D0 += mphid * wc + g;
                sumOff += fabs(off);
                B += fr.s * gam * mS * cg;
            }
            else
            {
                e.off[(size_t)k * nC + c] = 0.0;
                BoundaryPoint bp;
                boundaryPoint<false>(m, q, s, r, f, c, bp);
                face[f] = bp.th.rho;
                const double pRef = q.bcVal[F_P][m.bPatch[f - m.nIF]][0];
                const double cv = frcp(q.Rg * bp.T) * cPhBoundary(m, q, r, bp, f, c); // psi_b ph
                const double gb = bp.th.rho * r.rAU[c] * mS * dl * bp.frP;
                const double icf = cv * (1.0 - bp.frP) + gb;
                ic += icf;
                aic += fabs(icf);
                B -= (cv - gb) * bp.frP * pRef;
            }
        }
        if (alphaEqn > 0.0)
        {
            const double D1 = D0 + aic;
            const double aD1 = fabs(D1);
            const double D2 = aD1 > sumOff ? aD1 : sumOff;
            const double Dn = D2 * frcp(alphaEqn) - ic;
            e.diag[c] = Dn + ic;
            e.b[c] = B + (Dn - D0) * s.p[c];
        }
        else
        {
            e.diag[c] = D0 + ic;
            e.b[c] = B;
        }
        (void)NF;
    }
};

// phi == pEqn.flux() of the transonic corrector: F_f of the matrix at the solved p, with the div(phid,p) weights and rho_b frozen at
// assembly and the non-orthogonal correction of the assembly's grad(p).  At the fixed point this is the residual's F (cFaceF, cFwdC).
template <int NF>
struct cPhiTransonic
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    const double* face; // cPEqnTransonic's record
    double* phi;
    DAB_HD void operator()(int c) const
    {
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
            if (fr.f < 0) break;
            if (fr.s < 0) continue;
            const int f = fr.f;
            if (!fr.bnd)
            {
                const int n = fr.n;
                double phid, gam, cg;
                cPhidFace(m, q, s, r, f, c, n, phid, gam, cg);
                const double wf = face[f];
                phi[f] = phid * (wf * s.p[c] + (1.0 - wf) * s.p[n]) - gam * m.magSf[f] * (m.delta[f] * (s.p[n] - s.p[c]) + cg);
            }
            else
            {
                BoundaryPoint bp;
                boundaryPoint<false>(m, q, s, r, f, c, bp);
                const double cv = frcp(q.Rg * bp.T) * cPhBoundary(m, q, r, bp, f, c);
                phi[f] = cv * bp.p - face[f] * r.rAU[c] * m.magSf[f] * bp.sngP;
            }
        }
        (void)NF;
    }
};

// nuTilda equation, compressible form (DASpalartAllmaras.C:452-462 with rho)
template <int NF>
struct cNutEqnAssemble
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
        const double ntc = s.nt[c], rhoc = r.rho[c], nuc = r.nuL[c];
        const double Gc = rhoc * (ntc + nuc) * (1.0 / SA::sigma);
        double gUc[9], gNc[3];
        for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
        for (int i = 0; i < 3; i++) gNc[i] = r.gNt[(size_t)i * nT + c];
        double D0 = 0.0, sumOff = 0.0, X = 0.0, ic = 0.0, aic = 0.0;
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
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
                const double gf = (wc * Gc + wn * r.rho[n] * (ntn + r.nuL[n]) * (1.0 / SA::sigma)) * mS;
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
                BoundaryPoint bp;
                boundaryPoint<true>(m, q, s, r, f, c, bp);
                const double Gs = bp.th.rho * (bp.nt + bp.th.nu) * (1.0 / SA::sigma) * mS;
                const double icf = mf * (1.0 - bp.frN) + Gs * bp.frN * dl;
                ic += icf;
                aic += fabs(icf);
                D0 -= mf;
                X += mf * bp.nt - Gs * bp.sngN - icf * ntc;
            }
        }
        const double V = m.V[c], y = m.yWall[c];
        const double P = saSource(ntc, nuc, y, gUc, gNc, q.saFv3);
        const double St = saStilda(ntc, nuc, y, gUc, q.saFv3);
        const double mg2 = gNc[0] * gNc[0] + gNc[1] * gNc[1] + gNc[2] * gNc[2];
        const double expl = -(SA::Cb2 * (1.0 / SA::sigma)) * mg2 - SA::Cb1 * St * ntc;
        const double sp = ntc != 0.0 ? (P - expl) / ntc : 0.0;
        D0 += V * rhoc * sp;
        X += V * rhoc * expl;
        const double D1 = D0 + aic;
        const double aD1 = fabs(D1);
        const double D2 = aD1 > sumOff ? aD1 : sumOff;
        const double Dn = D2 * frcp(alphaN) - ic;
        e.diag[c] = Dn + ic;
        e.b[c] = -X + (Dn - D0) * ntc;
        (void)NF;
    }
};

} // namespace dab
