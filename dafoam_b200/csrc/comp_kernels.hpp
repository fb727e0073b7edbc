// DARhoSimpleFoam: forward residual kernels (compressible counterpart of fwd_kernels.hpp).
//
// R(W) of DAResidualRhoSimpleFoam::calcResiduals (reference src/adjoint/DAResidual/DAResidualRhoSimpleFoam.C:84-211)
// with DAResidual::updateThermoVars (DAResidual.C:179-293), the compressible branches of DATurbulenceModel
// (DATurbulenceModel.C:195-212, 259-330, 378-398) and DASpalartAllmaras::calcResiduals (DASpalartAllmaras.C:452-462).
// State ordering [U | p | T | nuTilda | phi], phi = mass flux.  Same gather structure as the incompressible kernels;
// everything that depends on the thermodynamic state is a *cell-local closure* (rho, nu, nut, rho*nuEff, alphaEff, he,
// Ekp) written once per cell by cFwdA and read by the face loops, with the boundary-face closures evaluated inline from
// the boundary values of (U, p, T, nuTilda).
//
//   cFwdA  closures + Gauss gradients of U, p, nuTilda, he
//   cFwdB  momentum row (rho*nuEff) -> URes, rAU, HbyA; SA row (rho-weighted) -> nuTildaRes
//   cFwdE  energy row: div(phi,he) + div(phi,Ekp|K) - laplacian(alphaEff,he) -> TRes
//   cFwdC  F_f = rho_f (S_f.HbyA_f) - (rho rAU)_f |S_f| snGrad(p) -> pRes = +div F, phiRes = F - phi
// Status: forward only (getResiduals); the hand-derived reverse sweep of these kernels is the next step.
#pragma once
#include "views.hpp"
#include "fwd_kernels.hpp"
#include <cmath>

namespace dab
{

struct ThermoPoint
{
    double rho, mu, alpha, nu, he;
};

DAB_HD double heOfT(const Params& q, double T) { return (q.heIsE ? (q.Cp - q.Rg) : q.Cp) * T - q.Cp * q.TRef; }

DAB_HD ThermoPoint thermoOf(const Params& q, double p, double T)
{
    ThermoPoint t;
    t.rho = p * frcp(q.Rg * T);
    if (q.sutherland)
    {
        const double Cv = q.Cp - q.Rg;
        t.mu = q.As * sqrt(T) * frcp(1.0 + q.Ts * frcp(T));
        t.alpha = t.mu * Cv * (1.32 + 1.77 * q.Rg * frcp(Cv)) * frcp(q.Cp);
    }
    else
    {
        t.mu = q.muC;
        t.alpha = t.mu * frcp(q.Pr);
    }
    t.nu = t.mu * frcp(t.rho);
    t.he = heOfT(q, T);
    return t;
}

DAB_HD double cpByCpv(const Params& q) { return q.heIsE ? q.Cp * frcp(q.Cp - q.Rg) : 1.0; }

// boundary-face values and closures of one boundary face (from the cell values through the BCs)
struct BoundaryPoint
{
    BCv bu;
    double p, sngP, frP;
    double T, sngT, frT;
    double nt, sngN, frN;
    ThermoPoint th;
    double nut, muE, aE, Ek;
};

template <bool WF>
DAB_HD void boundaryPoint(const MeshView& m, const Params& q, const StateView& s, const RecordView& r, int f, int c, BoundaryPoint& b)
{
    const int pa = m.bPatch[f - m.nIF];
    const double phib = s.phi[f], dl = m.delta[f], im = frcp(m.magSf[f]);
    const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
    const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
    double uw[3];
    mrfWallRef(m, f, q.bcVal[F_U][pa], uw);
    bcVector(q.bcKind[F_U][pa], uw, Uc, phib, dl, nh, b.bu);
    bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], s.p[c], phib, dl, b.p, b.sngP, b.frP);
    bcScalar(q.bcKindT[pa], q.bcValT[pa], s.T[c], phib, dl, b.T, b.sngT, b.frT);
    b.th = thermoOf(q, b.p, b.T);
    if (q.rhoFrozen)
    {
        // SIMPLE iterations: the boundary density follows the stored (relaxed) cell density; equal to psi_b*p_b at the fixed point
        b.th.rho = r.rho[c] * (b.p * s.T[c]) * frcp(s.p[c] * b.T);
        b.th.nu = b.th.mu * frcp(b.th.rho);
    }
    b.nt = 0.0; b.sngN = 0.0; b.frN = 0.0; b.nut = 0.0;
    if (q.turb)
    {
        bcScalar(q.bcKind[F_NUTILDA][pa], q.bcVal[F_NUTILDA][pa][0], s.nt[c], phib, dl, b.nt, b.sngN, b.frN);
        double dP, dNb, dUn[3];
        b.nut = WF ? nutBoundary<true>(q.bcKind[F_NUT][pa], q.bcVal[F_NUT][pa][0], r.nut[c], b.nt, b.th.nu, Uc, b.bu.val, dl, dP, dNb, dUn)
                   : nutBoundaryBasic(q.bcKind[F_NUT][pa], q.bcVal[F_NUT][pa][0], r.nut[c], b.nt, b.th.nu, dP, dNb);
    }
    b.muE = b.th.rho * (b.th.nu + b.nut);
    b.aE = cpByCpv(q) * (b.th.alpha + b.th.rho * b.nut * frcp(q.Prt));
    b.Ek = 0.5 * (b.bu.val[0] * b.bu.val[0] + b.bu.val[1] * b.bu.val[1] + b.bu.val[2] * b.bu.val[2]);
    if (q.heIsE) b.Ek += b.p * frcp(b.th.rho);
}

template <int NF>
struct cFwdA
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot;
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double pc = s.p[c], Tc = s.T[c];
        const double ntc = q.turb ? s.nt[c] : 0.0;
        // cell closures
        ThermoPoint th = thermoOf(q, pc, Tc);
        if (q.rhoFrozen)
        {
            // SIMPLE iterations: rho is the relaxed field of the previous iteration (reference pEqnRhoSimple.H rho.relax())
            th.rho = r.rho[c];
            th.nu = th.mu * frcp(th.rho);
        }
        const double nut = q.turb ? ntc * fv1f(ntc * frcp(th.nu)) : 0.0;
        r.rho[c] = th.rho;
        r.nuL[c] = th.nu;
        r.nut[c] = nut;
        r.muE[c] = th.rho * (th.nu + nut);
        r.aE[c] = cpByCpv(q) * (th.alpha + th.rho * nut * frcp(q.Prt));
        r.he[c] = th.he;
        r.Ek[c] = 0.5 * (Uc[0] * Uc[0] + Uc[1] * Uc[1] + Uc[2] * Uc[2]) + (q.heIsE ? pc * frcp(th.rho) : 0.0);
        if (c >= m.nC) return;
        double gU[9], gP[3], gN[3], gH[3];
        for (int i = 0; i < 9; i++) gU[i] = 0.0;
        for (int i = 0; i < 3; i++) { gP[i] = 0.0; gN[i] = 0.0; gH[i] = 0.0; }
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            const double S[3] = {fr.s * m.Sx[f], fr.s * m.Sy[f], fr.s * m.Sz[f]};
            double Uf[3], pf, nf = 0.0, hf;
            if (!fr.bnd)
            {
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f], wn = 1.0 - wc;
                const int n = fr.n;
                for (int j = 0; j < 3; j++) Uf[j] = wc * Uc[j] + wn * s.U[3 * n + j];
                pf = wc * pc + wn * s.p[n];
                if (q.turb) nf = wc * ntc + wn * s.nt[n];
                hf = wc * th.he + wn * heOfT(q, s.T[n]);
            }
            else
            {
                const int pa = m.bPatch[f - m.nIF];
                const double phib = s.phi[f], dl = m.delta[f], im = frcp(m.magSf[f]);
                const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
                BCv bu;
                double uw[3];
                mrfWallRef(m, f, q.bcVal[F_U][pa], uw);
                bcVector(q.bcKind[F_U][pa], uw, Uc, phib, dl, nh, bu);
                for (int j = 0; j < 3; j++) Uf[j] = bu.val[j];
                double sn, fr_, Tb;
                bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], pc, phib, dl, pf, sn, fr_);
                if (q.turb) bcScalar(q.bcKind[F_NUTILDA][pa], q.bcVal[F_NUTILDA][pa][0], ntc, phib, dl, nf, sn, fr_);
                bcScalar(q.bcKindT[pa], q.bcValT[pa], Tc, phib, dl, Tb, sn, fr_);
                hf = heOfT(q, Tb);
            }
            for (int j = 0; j < 3; j++)
                for (int i = 0; i < 3; i++) gU[j * 3 + i] += S[i] * Uf[j];
            for (int i = 0; i < 3; i++) { gP[i] += S[i] * pf; gN[i] += S[i] * nf; gH[i] += S[i] * hf; }
        }
        const double iV = frcp(m.V[c]);
        for (int i = 0; i < 9; i++) r.gU[(size_t)i * nT + c] = gU[i] * iV;
        for (int i = 0; i < 3; i++)
        {
            r.gP[(size_t)i * nT + c] = gP[i] * iV;
            r.gNt[(size_t)i * nT + c] = gN[i] * iV;
            r.gHe[(size_t)i * nT + c] = gH[i] * iV;
        }
    }
};

// momentum and SA rows; always compiled with every optional feature (linearUpwindV, wall function)
template <int NF>
struct cFwdB
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    int isPC;
    double* R;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const int schU = isPC ? DIV_UPWIND : q.divU;
        const int schN = isPC ? DIV_UPWIND : q.divNut;
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double muEc = r.muE[c], rhoc = r.rho[c], nuc = r.nuL[c];
        double gUc[9], gNc[3];
        for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
        const double ntc = q.turb ? s.nt[c] : 0.0;
        const double Gc = rhoc * (ntc + nuc) * (1.0 / SA::sigma);
        for (int i = 0; i < 3; i++) gNc[i] = q.turb ? r.gNt[(size_t)i * nT + c] : 0.0;
        const double trc = gUc[0] + gUc[4] + gUc[8];
        double D0 = 0.0, sumOff = 0.0, MV[3] = {0.0, 0.0, 0.0};
        double icMax = 0.0, icMin = 0.0, icAvg = 0.0;
        double NV = 0.0;
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
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
                {
                    const double wp = schU == DIV_LINEAR ? wc : wup;
                    const double a = wp * mf;
                    const double gf = (wc * muEc + wn * muEn) * mS;
                    const double g = gf * dl;
                    const double off = mf - a - g;
                    D0 += a + g - mf;
                    sumOff += fabs(off);
                    for (int j = 0; j < 3; j++) MV[j] += (a + g - mf) * Uc[j] + off * Un[j];
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
                        for (int j = 0; j < 3; j++) MV[j] += mf * corr[j];
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
                        MV[j] -= fr.s * gf * cg;
                    }
                    const double trn = gUn[0] + gUn[4] + gUn[8];
                    for (int j = 0; j < 3; j++)
                    {
                        const double tc = muEc * (Sv[0] * gUc[0 * 3 + j] + Sv[1] * gUc[1 * 3 + j] + Sv[2] * gUc[2 * 3 + j] - (2.0 / 3.0) * trc * Sv[j]);
                        const double tn = muEn * (Sv[0] * gUn[0 * 3 + j] + Sv[1] * gUn[1 * 3 + j] + Sv[2] * gUn[2 * 3 + j] - (2.0 / 3.0) * trn * Sv[j]);
                        MV[j] -= fr.s * (wc * tc + wn * tn);
                    }
                }
                if (q.turb)
                {
                    const double ntn = s.nt[n];
                    const double wp = schN == DIV_LINEAR ? wc : wup;
                    const double a = wp * mf;
                    const double Gn = r.rho[n] * (ntn + r.nuL[n]) * (1.0 / SA::sigma);
                    const double gf = (wc * Gc + wn * Gn) * mS;
                    const double g = gf * dl;
                    NV += (a + g - mf) * ntc + (mf - a - g) * ntn;
                    if (schN == DIV_LINEAR_UPWIND)
                    {
                        const bool ownUp = s.phi[f] > 0.0;
                        const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                        const int u = cUp ? c : n;
                        const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                        double corr = 0.0;
                        for (int i = 0; i < 3; i++) corr += d[i] * r.gNt[(size_t)i * nT + u];
                        NV += mf * corr;
                    }
                    const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                    double cg = 0.0;
                    for (int i = 0; i < 3; i++) cg += kv[i] * (wc * gNc[i] + wn * r.gNt[(size_t)i * nT + n]);
                    NV -= fr.s * gf * cg;
                }
            }
            else
            {
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
                    MV[j] += mf * bp.bu.val[j] - G * bp.bu.sng[j] - mf * Uc[j];
                }
                icMax += mx; icMin += mn; icAvg += av * (1.0 / 3.0);
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
                    MV[j] -= bp.muE * x;
                }
                if (q.turb)
                {
                    const double Gs = bp.th.rho * (bp.nt + bp.th.nu) * (1.0 / SA::sigma) * mS;
                    NV += mf * bp.nt - Gs * bp.sngN - mf * ntc;
                }
            }
        }
        const double V = m.V[c], iV = frcp(V);
        const double D1 = D0 + icMax;
        const double aD1 = fabs(D1);
        double D2, flag;
        if (aD1 > sumOff) { D2 = aD1; flag = D1 < 0.0 ? -1.0 : 1.0; }
        else { D2 = sumOff; flag = 0.0; }
        const double Dn = D2 * frcp(q.alphaU) - icMin;
        const double A = (Dn + icAvg) * iV;
        const double rAU = frcp(A);
        r.rAU[c] = rAU;
        r.D0[c] = D0;
        r.flag[c] = flag;
        const double cU = q.nrU ? 1.0 : V;
        double cor[3] = {0.0, 0.0, 0.0}; // MRF.DDt(rho, U) = rho * (Omega x U) in the zone cells
        if (m.mrfCell && m.mrfCell[c])
        {
            const double* w = m.mrfOmega;
            cor[0] = rhoc * (w[1] * Uc[2] - w[2] * Uc[1]);
            cor[1] = rhoc * (w[2] * Uc[0] - w[0] * Uc[2]);
            cor[2] = rhoc * (w[0] * Uc[1] - w[1] * Uc[0]);
        }
        for (int j = 0; j < 3; j++)
        {
            const double M = MV[j] * iV + cor[j] - (m.fvS ? m.fvS[(size_t)j * nC + c] : 0.0); // UEqn ... + MRF.DDt - fvSource
            r.HbyA[(size_t)j * nT + c] = Uc[j] - rAU * M;
            R[3 * c + j] = (M + r.gP[(size_t)j * nT + c]) * cU;
        }
        if (q.turb)
        {
            const double src = rhoc * saSource(ntc, nuc, m.yWall[c], gUc, gNc, q.saFv3);
            R[5 * (size_t)nC + c] = (NV * iV + src) * (q.nrNut ? 1.0 : V);
        }
    }
};

// DATurboFoam, enthalpy form (DAResidualTurboFoam.C:117-121): the vector Teff & U - p (U - URel) whose Gauss-linear divergence
// is subtracted from the energy row; Teff = muEff dev(twoSymm(grad U)), gU[j*3+i] = d_i U_j, vrel = Omega x r or null
DAB_HD void turboWork(const double* gU, double mu, const double* u, double p, const double* vrel, double* out)
{
    const double tr = gU[0] + gU[4] + gU[8];
    for (int j = 0; j < 3; j++)
    {
        double acc = 0.0;
        for (int i = 0; i < 3; i++)
        {
            double te = gU[j * 3 + i] + gU[i * 3 + j];
            if (i == j) te -= (2.0 / 3.0) * tr;
            acc += te * u[i];
        }
        out[j] = mu * acc - (vrel ? p * vrel[j] : 0.0);
    }
}
// adjoint: qb = d(row)/d(out); accumulates d/d(gU), d/d(mu), d/d(u), d/d(p)
DAB_HD void turboWorkAdj(const double* gU, double mu, const double* u, const double* vrel, const double* qb, double* gUb, double& mub, double* ub,
                         double& pb)
{
    const double tr = gU[0] + gU[4] + gU[8];
    double trb = 0.0;
    for (int j = 0; j < 3; j++)
        for (int i = 0; i < 3; i++)
        {
            double te = gU[j * 3 + i] + gU[i * 3 + j];
            if (i == j) te -= (2.0 / 3.0) * tr;
            mub += te * u[i] * qb[j];
            ub[i] += mu * te * qb[j];
            const double teb = mu * u[i] * qb[j];
            gUb[j * 3 + i] += teb;
            gUb[i * 3 + j] += teb;
            if (i == j) trb -= (2.0 / 3.0) * teb;
        }
    gUb[0] += trb; gUb[4] += trb; gUb[8] += trb;
    if (vrel) pb -= vrel[0] * qb[0] + vrel[1] * qb[1] + vrel[2] * qb[2];
}
// Omega x (x - origin)
DAB_HD void mrfVelocityAt(const MeshView& m, double x, double y, double z, double* v)
{
    const double r[3] = {x - m.mrfOrigin[0], y - m.mrfOrigin[1], z - m.mrfOrigin[2]};
    const double* w = m.mrfOmega;
    v[0] = w[1] * r[2] - w[2] * r[1];
    v[1] = w[2] * r[0] - w[0] * r[2];
    v[2] = w[0] * r[1] - w[1] * r[0];
}

// energy row: TRes = (EEqn & he), EEqn = div(phi,he) + div(phi,Ekp|K) - laplacian(alphaEff,he)
template <int NF>
struct cFwdE
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    int isPC;
    double* R;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const int schE = isPC ? DIV_UPWIND : q.divE;
        const double hec = r.he[c], aEc = r.aE[c], Ekc = r.Ek[c];
        double gHc[3];
        for (int i = 0; i < 3; i++) gHc[i] = r.gHe[(size_t)i * nT + c];
        double EV = 0.0;
        double twc[3] = {0.0, 0.0, 0.0}, gUt[9]; // turboH: the work vector of this cell
        if (q.turboH)
        {
            for (int i = 0; i < 9; i++) gUt[i] = r.gU[(size_t)i * nT + c];
            const double uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
            double vr[3];
            const bool inZone = m.mrfCell && m.mrfCell[c];
            if (inZone) mrfVelocityAt(m, m.Cx[c], m.Cy[c], m.Cz[c], vr);
            turboWork(gUt, r.muE[c], uc, s.p[c], inZone ? vr : nullptr, twc);
        }
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            const double mf = fr.s * s.phi[f];
            const double mS = m.magSf[f], dl = m.delta[f];
            if (!fr.bnd)
            {
                const int n = fr.n;
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f], wn = 1.0 - wc;
                const bool pos0 = s.phi[f] >= 0.0;
                const double wup = fr.s > 0 ? (pos0 ? 1.0 : 0.0) : (pos0 ? 0.0 : 1.0);
                const double hen = r.he[n];
                const double wp = schE == DIV_LINEAR ? wc : wup;
                const double a = wp * mf;
                const double gf = (wc * aEc + wn * r.aE[n]) * mS;
                const double g = gf * dl;
                EV += (a + g - mf) * hec + (mf - a - g) * hen;
                if (schE == DIV_LINEAR_UPWIND)
                {
                    const bool ownUp = s.phi[f] > 0.0;
                    const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                    const int u = cUp ? c : n;
                    const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                    double corr = 0.0;
                    for (int i = 0; i < 3; i++) corr += d[i] * r.gHe[(size_t)i * nT + u];
                    EV += mf * corr;
                }
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                double cg = 0.0;
                for (int i = 0; i < 3; i++) cg += kv[i] * (wc * gHc[i] + wn * r.gHe[(size_t)i * nT + n]);
                EV -= fr.s * gf * cg;
                // fvc::div(phi, Ekp): bounded Gauss upwind | linear
                const double wk = q.divEkp == DIV_LINEAR ? wc : wup;
                const double Ekf = wk * Ekc + (1.0 - wk) * r.Ek[n];
                EV += mf * (Ekf - Ekc);
                if (q.turboH)
                {
                    double gn[9], twn[3], vr[3];
                    for (int i = 0; i < 9; i++) gn[i] = r.gU[(size_t)i * nT + n];
                    const double un[3] = {s.U[3 * n], s.U[3 * n + 1], s.U[3 * n + 2]};
                    const bool inZone = m.mrfCell && m.mrfCell[n];
                    if (inZone) mrfVelocityAt(m, m.Cx[n], m.Cy[n], m.Cz[n], vr);
                    turboWork(gn, r.muE[n], un, s.p[n], inZone ? vr : nullptr, twn);
                    EV -= fr.s * (m.Sx[f] * (wc * twc[0] + wn * twn[0]) + m.Sy[f] * (wc * twc[1] + wn * twn[1]) + m.Sz[f] * (wc * twc[2] + wn * twn[2]));
                }
            }
            else
            {
                BoundaryPoint bp;
                boundaryPoint<true>(m, q, s, r, f, c, bp);
                const double heb = bp.th.he;
                const double sngH = (q.heIsE ? (q.Cp - q.Rg) : q.Cp) * bp.sngT;
                EV += mf * heb - bp.aE * mS * sngH - mf * hec;
                EV += mf * (bp.Ek - Ekc);
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
                    EV -= m.Sx[f] * twb[0] + m.Sy[f] * twb[1] + m.Sz[f] * twb[2];
                }
            }
        }
        if (m.fvS) // - fvSourceEnergy = -(fvSource & U)
            EV -= m.V[c] * (m.fvS[c] * s.U[3 * c] + m.fvS[(size_t)nC + c] * s.U[3 * c + 1] + m.fvS[(size_t)2 * nC + c] * s.U[3 * c + 2]);
        R[4 * (size_t)nC + c] = EV * (q.nrT ? frcp(m.V[c]) : 1.0);
    }
};

// limitedLinear(k) limiter of the face value of p convected by phid (OpenFOAM limitedLinear.H, NVDTVD.H::r): returns the limiter
// and (for the adjoint) its slope d(limiter)/d(r) (0 where clipped) with r = 2 gradcf/gradf - 1, gradcf = d . grad(p)_upwind.
// fluxPositive: phid > 0 (strict, as in NVDTVD::r); o/n owner and neighbour of the face
DAB_HD double limitedLinearLimiter(const MeshView& m, const StateView& s, const RecordView& r, double k, bool fluxPositive, int o, int n,
                                   double& dLimDr, double& gradf, double& gradcf, bool& farBranch)
{
    const int nT = m.nCtot;
    const int u = fluxPositive ? o : n;
    const double d[3] = {m.Cx[n] - m.Cx[o], m.Cy[n] - m.Cy[o], m.Cz[n] - m.Cz[o]};
    gradf = s.p[n] - s.p[o];
    gradcf = d[0] * r.gP[u] + d[1] * r.gP[(size_t)nT + u] + d[2] * r.gP[(size_t)2 * nT + u];
    farBranch = fabs(gradcf) >= 1000.0 * fabs(gradf);
    const double rr = farBranch ? 2.0 * 1000.0 * (gradcf >= 0.0 ? 1.0 : -1.0) * (gradf >= 0.0 ? 1.0 : -1.0) - 1.0 : 2.0 * (gradcf / gradf) - 1.0;
    const double twoByk = 2.0 / (k > 1e-15 ? k : 1e-15);
    const double lim = twoByk * rr;
    dLimDr = (lim > 0.0 && lim < 1.0 && !farBranch) ? twoByk : 0.0;
    return lim > 1.0 ? 1.0 : (lim < 0.0 ? 0.0 : lim);
}

// F_f of an internal face from the owner's point of view (compressible).  Transonic (q.transonic, DAResidualTurboFoam.C:148-189,
// DAResidualRhoSimpleCFoam.C:160-183): phid p_f - (rho rAU)_f |S_f| snGrad(p), phid = psi_f (S_f.HbyA_f - relative-frame flux),
// p_f by the div(phid,p) scheme (weights only: the matrix flux and the matrix residual see the same face value)
DAB_HD double cFaceF(const MeshView& m, const Params& q, const StateView& s, const RecordView& r, int f, int o, int n)
{
    const int nT = m.nCtot;
    const double w = m.w[f], mS = m.magSf[f];
    double ph = 0.0, cg = 0.0;
    const double Sv[3] = {m.Sx[f], m.Sy[f], m.Sz[f]};
    const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
    for (int j = 0; j < 3; j++)
    {
        ph += Sv[j] * (w * r.HbyA[(size_t)j * nT + o] + (1.0 - w) * r.HbyA[(size_t)j * nT + n]);
        cg += kv[j] * (w * r.gP[(size_t)j * nT + o] + (1.0 - w) * r.gP[(size_t)j * nT + n]);
    }
    const double gam = w * r.rho[o] * r.rAU[o] + (1.0 - w) * r.rho[n] * r.rAU[n];
    const double sn = m.delta[f] * (s.p[n] - s.p[o]) + cg;
    if (m.mrfFlux) ph -= m.mrfFlux[f]; // MRF.makeRelative(interpolate(rho), phiHbyA)
    if (q.transonic)
    {
        if (q.transonic == 2) return -gam * mS * sn; // preconditioner residual without div(phid,p)
        const double phid = (w * frcp(q.Rg * s.T[o]) + (1.0 - w) * frcp(q.Rg * s.T[n])) * ph;
        double wf;
        if (q.divPhidP == DIV_LINEAR) wf = w;
        else if (q.divPhidP == DIV_LIMITED_LINEAR)
        {
            double dl, gf, gc;
            bool fb;
            const double lim = limitedLinearLimiter(m, s, r, q.phidK, phid > 0.0, o, n, dl, gf, gc, fb);
            wf = lim * w + (1.0 - lim) * (phid >= 0.0 ? 1.0 : 0.0);
        }
        else wf = phid >= 0.0 ? 1.0 : 0.0;
        return phid * (wf * s.p[o] + (1.0 - wf) * s.p[n]) - gam * mS * sn;
    }
    const double rhof = w * r.rho[o] + (1.0 - w) * r.rho[n];
    return rhof * ph - gam * mS * sn;
}

template <int NF>
struct cFwdC
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    double* R;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const size_t offP = (size_t)3 * nC, offPhi = (size_t)(q.turb ? 6 : 5) * nC;
        double div = 0.0;
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            double F;
            if (!fr.bnd)
            {
                const int o = fr.s > 0 ? c : fr.n, n = fr.s > 0 ? fr.n : c;
                F = cFaceF(m, q, s, r, f, o, n);
            }
            else
            {
                BoundaryPoint bp;
                boundaryPoint<false>(m, q, s, r, f, c, bp); // nut_b is not needed here
                const int pa = m.bPatch[f - m.nIF];
                const int kU = q.bcKind[F_U][pa];
                const bool assignable = (kU == BC_INLET_OUTLET || kU == BC_OUTLET_INLET || kU == BC_ZERO_GRADIENT);
                double ph;
                if (q.constrainHbyA && !assignable)
                    ph = m.Sx[f] * bp.bu.val[0] + m.Sy[f] * bp.bu.val[1] + m.Sz[f] * bp.bu.val[2];
                else
                    ph = m.Sx[f] * r.HbyA[c] + m.Sy[f] * r.HbyA[(size_t)nT + c] + m.Sz[f] * r.HbyA[(size_t)2 * nT + c];
                ph = mrfBoundaryFlux(m, f, ph, 1.0);
                if (q.transonic == 2) ph = 0.0; // preconditioner residual without div(phid,p): its boundary part psi_b p_b ph = rho_b ph goes too
                F = bp.th.rho * ph - bp.th.rho * r.rAU[c] * m.magSf[f] * bp.sngP;
            }
            div += fr.s * F;
            if (q.transonic == 3 && fr.s > 0) R[offPhi + f] = s.phi[f] * (q.nrPhi ? frcp(m.magSf[f]) : 1.0); // transonicPCOption 2
            else if (fr.s > 0) R[offPhi + f] = (F - s.phi[f]) * (q.nrPhi ? frcp(m.magSf[f]) : 1.0);
            else if (fr.n >= nC) R[offPhi + f] = 0.0;
        }
        R[offP + c] = div * (q.nrP ? frcp(m.V[c]) : 1.0);
    }
};

} // namespace dab
