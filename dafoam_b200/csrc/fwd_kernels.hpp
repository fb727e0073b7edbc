// Forward residual R(W) of DASimpleFoam (+SA) as three fused cell-parallel gather kernels.
//
//   FwdA  per cell: nut = nuTilda*fv1 (DASpalartAllmaras::correctNut, reference DASpalartAllmaras.C:215-233)
//         and the Gauss-linear gradients grad(U), grad(p), grad(nuTilda) (boundary-face values from the BCs,
//         reference DAResidualSimpleFoam::correctBoundaryConditions DAResidualSimpleFoam.C:253-265)
//   FwdB  per cell: the momentum row (div(phi,U) - laplacian(nuEff,U) - div(nuEff*dev2(T(grad(U)))), relax,
//         A(), H()) -> URes, rAU, HbyA (reference DAResidualSimpleFoam.C:141-179, DATurbulenceModel.C:378-398)
//         and the SA row -> nuTildaRes (reference DASpalartAllmaras.C:452-485)
//   FwdC  per cell: F_f = phiHbyA_f - rAU_f |S_f| snGrad(p)_f on the cell's faces -> pRes = -div(F)
//         and (owner side) phiRes = F - phi (reference DAResidualSimpleFoam.C:181-212)
//
// Every kernel is a gather over the ELL cell->face table: no atomics, deterministic summation order.
// All arithmetic is fp64; the path is HBM-bandwidth bound (no tensor cores).
#pragma once
#include "views.hpp"
#include <cmath>

namespace dab
{

template <int NF>
struct FwdA
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot;
        if (q.turb) r.nut[c] = s.nt[c] * fv1f(s.nt[c] * frcp(q.nu));
        else r.nut[c] = 0.0;
        if (c >= m.nC) return;
        double gU[9], gP[3], gN[3];
        for (int i = 0; i < 9; i++) gU[i] = 0.0;
        for (int i = 0; i < 3; i++) { gP[i] = 0.0; gN[i] = 0.0; }
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double pc = s.p[c];
        const double ntc = q.turb ? s.nt[c] : 0.0;
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            const double S[3] = {fr.s * m.Sx[f], fr.s * m.Sy[f], fr.s * m.Sz[f]}; // outward
            double Uf[3], pf, nf = 0.0;
            if (!fr.bnd)
            {
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f];
                const double wn = 1.0 - wc;
                const int n = fr.n;
                for (int j = 0; j < 3; j++) Uf[j] = wc * Uc[j] + wn * s.U[3 * n + j];
                pf = wc * pc + wn * s.p[n];
                if (q.turb) nf = wc * ntc + wn * s.nt[n];
            }
            else
            {
                const int b = f - m.nIF, pa = m.bPatch[b];
                const double phib = s.phi[f], dl = m.delta[f];
                const double im = frcp(m.magSf[f]);
                const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
                BCv bu;
                double uw[3];
                mrfWallRef(m, f, q.bcVal[F_U][pa], uw);
                bcVector(q.bcKind[F_U][pa], uw, Uc, phib, dl, nh, bu);
                for (int j = 0; j < 3; j++) Uf[j] = bu.val[j];
                double sn, fr_;
                bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], pc, phib, dl, pf, sn, fr_);
                if (q.turb) bcScalar(q.bcKind[F_NUTILDA][pa], q.bcVal[F_NUTILDA][pa][0], ntc, phib, dl, nf, sn, fr_);
            }
            for (int j = 0; j < 3; j++)
                for (int i = 0; i < 3; i++) gU[j * 3 + i] += S[i] * Uf[j];
            for (int i = 0; i < 3; i++) { gP[i] += S[i] * pf; gN[i] += S[i] * nf; }
        }
        const double iV = frcp(m.V[c]);
        for (int i = 0; i < 9; i++) r.gU[(size_t)i * nT + c] = gU[i] * iV;
        for (int i = 0; i < 3; i++)
        {
            r.gP[(size_t)i * nT + c] = gP[i] * iV;
            r.gNt[(size_t)i * nT + c] = gN[i] * iV;
        }
    }
};

// Stilda of the SA model.  Standard (DASpalartAllmaras.C:144-157): max(Omega + fv2 nt/(kappa y)^2, Cs Omega) with
// fv2 = 1 - chi/(1 + chi fv1); fv3 variant (DASpalartAllmarasFv3.C:158-175, 452-456): fv3 Omega + fv2 nt/(kappa y)^2
// with fv2 = (1 + chi/Cv2)^-3, fv3 = (1 + chi fv1)(1/Cv2)(3(1 + chi/Cv2) + (chi/Cv2)^2)/(1 + chi/Cv2)^3, no clip.
DAB_HD double saStilda(double nt, double nu, double y, const double* gU, int fv3)
{
    const double chi = nt * frcp(nu);
    const double fv1 = fv1f(chi);
    const double w01 = 0.5 * (gU[1 * 3 + 0] - gU[0 * 3 + 1]);
    const double w02 = 0.5 * (gU[2 * 3 + 0] - gU[0 * 3 + 2]);
    const double w12 = 0.5 * (gU[2 * 3 + 1] - gU[1 * 3 + 2]);
    const double Omega = sqrt(2.0) * sqrt(2.0 * (w01 * w01 + w02 * w02 + w12 * w12));
    const double ky2 = (SA::kappa * y) * (SA::kappa * y);
    if (fv3)
    {
        const double t = 1.0 + chi * (1.0 / SA::Cv2), t3 = t * t * t;
        const double fv2 = frcp(t3);
        const double f3 = (1.0 + chi * fv1) * ((1.0 / SA::Cv2)) * (3.0 * t + (chi * (1.0 / SA::Cv2)) * (chi * (1.0 / SA::Cv2))) * frcp(t3);
        return f3 * Omega + fv2 * nt * frcp(ky2);
    }
    const double fv2 = 1.0 - chi * frcp(1.0 + chi * fv1);
    const double S1 = Omega + fv2 * nt * frcp(ky2), S2 = SA::Cs * Omega;
    return S1 > S2 ? S1 : S2;
}

// SA cell-local source terms: P = -Cb2/sigma |grad nt|^2 - Cb1 Stilda nt + Cw1 fw nt^2 / y^2
// (returned per unit volume).  gU: d_i U_j at [j*3+i].
DAB_HD double saSource(double nt, double nu, double y, const double* gU, const double* gN, int fv3)
{
    const double St = saStilda(nt, nu, y, gU, fv3);
    const double ky2 = (SA::kappa * y) * (SA::kappa * y);
    const double Sm = St > 1e-15 ? St : 1e-15;
    double rr = nt * frcp(Sm * ky2);
    rr = rr < 10.0 ? rr : 10.0;
    const double r2 = rr * rr;
    const double g = rr + SA::Cw2 * (r2 * r2 * r2 - rr);
    const double g2 = g * g;
    const double fw = g * cbrt(sqrt((1.0 + SA::Cw3p6) * frcp(g2 * g2 * g2 + SA::Cw3p6))); // x^(1/6)
    const double mg2 = gN[0] * gN[0] + gN[1] * gN[1] + gN[2] * gN[2];
    return -(SA::Cb2 * (1.0 / SA::sigma)) * mg2 - SA::Cb1 * St * nt + SA::Cw1 * fw * nt * nt * frcp(y * y);
}

// FEAT: bit 0 = linearUpwindV limiter compiled in, bit 1 = wall-function nut BC compiled in (the common
// configuration without them keeps its register budget)
template <int NF, int FEAT>
struct FwdB
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    int isPC;
    double* R; // residual vector (reference layout); URes and nuTildaRes written here
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const int schU = isPC ? DIV_UPWIND : q.divU;
        const int schN = isPC ? DIV_UPWIND : q.divNut;
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double nuEc = r.nut[c] + q.nu;
        double gUc[9], gNc[3];
        for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
        const double ntc = q.turb ? s.nt[c] : 0.0;
        const double Gc = (ntc + q.nu) * (1.0 / SA::sigma);
        for (int i = 0; i < 3; i++) gNc[i] = q.turb ? r.gNt[(size_t)i * nT + c] : 0.0;
        const double trc = gUc[0] + gUc[4] + gUc[8];

        double D0 = 0.0, sumOff = 0.0, MV[3] = {0.0, 0.0, 0.0}; // MV = V*(UEqn & U)
        double icMax = 0.0, icMin = 0.0, icAvg = 0.0;
        double NV = 0.0; // V*(nuTildaEqn & nuTilda) without the cell-local sources
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
                const double nuEn = r.nut[n] + q.nu;
                // ---- momentum row
                {
                    const double wp = schU == DIV_LINEAR ? wc : wup;
                    const double a = wp * mf;
                    const double gf = (wc * nuEc + wn * nuEn) * mS;
                    const double g = gf * dl;
                    const double off = mf - a - g;
                    D0 += a + g - mf;
                    sumOff += fabs(off);
                    for (int j = 0; j < 3; j++) MV[j] += (a + g - mf) * Uc[j] + off * Un[j];
                    // explicit sources (moved to the left-hand side: MV -= Src)
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
                            // maxCorr = (1-w)(U_nei - U_own) for phi > 0, w (U_own - U_nei) otherwise
                            const double wo_ = m.w[f];
                            const double cf = ownUp ? (1.0 - wo_) : -wo_;
                            double maxCorr[3];
                            for (int j = 0; j < 3; j++) maxCorr[j] = cf * fr.s * (Un[j] - Uc[j]);
                            luvLimit(corr, maxCorr, corr);
                        }
                        for (int j = 0; j < 3; j++) MV[j] += mf * corr[j]; // Src -= s*phi*corr
                    }
                    const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                    const double wo = m.w[f]; // owner weight for face-interpolated gradients
                    const bool own = fr.s > 0; // value selects: a pointer into either gradient array would put both in local memory
                    for (int j = 0; j < 3; j++)
                    {
                        double cg = 0.0;
                        for (int i = 0; i < 3; i++)
                        {
                            const double gO = own ? gUc[j * 3 + i] : gUn[j * 3 + i], gN_ = own ? gUn[j * 3 + i] : gUc[j * 3 + i];
                            cg += kv[i] * (wo * gO + (1.0 - wo) * gN_);
                        }
                        MV[j] -= fr.s * gf * cg; // Src += s*gf*cg
                    }
                    // dev2 term: Src_j += s*(w T_P + (1-w) T_N)_j, T_X,j = nuEff_X (sum_i S_i d_j U_i - 2/3 tr S_j)
                    const double trn = gUn[0] + gUn[4] + gUn[8];
                    for (int j = 0; j < 3; j++)
                    {
                        const double tc = nuEc * (Sv[0] * gUc[0 * 3 + j] + Sv[1] * gUc[1 * 3 + j] + Sv[2] * gUc[2 * 3 + j] - (2.0 / 3.0) * trc * Sv[j]);
                        const double tn = nuEn * (Sv[0] * gUn[0 * 3 + j] + Sv[1] * gUn[1 * 3 + j] + Sv[2] * gUn[2 * 3 + j] - (2.0 / 3.0) * trn * Sv[j]);
                        MV[j] -= fr.s * (wc * tc + wn * tn);
                    }
                }
                // ---- SA row
                if (q.turb)
                {
                    const double ntn = s.nt[n];
                    const double wp = schN == DIV_LINEAR ? wc : wup;
                    const double a = wp * mf;
                    const double gf = (wc * Gc + wn * (ntn + q.nu) * (1.0 / SA::sigma)) * mS;
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
                    for (int i = 0; i < 3; i++)
                    {
                        const double gn = r.gNt[(size_t)i * nT + n];
                        cg += kv[i] * (wc * gNc[i] + wn * gn);
                    }
                    NV -= fr.s * gf * cg;
                }
            }
            else
            {
                const int b = f - m.nIF, pa = m.bPatch[b];
                const double im = frcp(mS);
                const double nh[3] = {Sv[0] * im, Sv[1] * im, Sv[2] * im};
                BCv bu;
                double uw[3];
                mrfWallRef(m, f, q.bcVal[F_U][pa], uw);
                bcVector(q.bcKind[F_U][pa], uw, Uc, mf, dl, nh, bu);
                double ntb = 0.0, sngN = 0.0, frN;
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
                    MV[j] += mf * bu.val[j] - G * bu.sng[j] - mf * Uc[j];
                }
                icMax += mx; icMin += mn; icAvg += av * (1.0 / 3.0);
                // dev2 boundary term: boundary grad(U) = cell value with the normal component replaced by snGrad
                double Gb[9]; // Gb[j*3+i] = d_i U_j at the face
                for (int j = 0; j < 3; j++)
                {
                    const double nG = nh[0] * gUc[j * 3 + 0] + nh[1] * gUc[j * 3 + 1] + nh[2] * gUc[j * 3 + 2];
                    for (int i = 0; i < 3; i++) Gb[j * 3 + i] = gUc[j * 3 + i] + nh[i] * (bu.sng[j] - nG);
                }
                const double trb = Gb[0] + Gb[4] + Gb[8];
                for (int j = 0; j < 3; j++)
                {
                    const double x = Sv[0] * Gb[0 * 3 + j] + Sv[1] * Gb[1 * 3 + j] + Sv[2] * Gb[2 * 3 + j] - (2.0 / 3.0) * trb * Sv[j];
                    MV[j] -= (nutb + q.nu) * x;
                }
                if (q.turb)
                {
                    const double Gs = (ntb + q.nu) * (1.0 / SA::sigma) * mS;
                    NV += mf * ntb - Gs * sngN - mf * ntc;
                }
            }
        }
        const double V = m.V[c], iV = frcp(V);
        // relax (fvMatrix::relax, OpenFOAM-v1812)
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
        double cor[3] = {0.0, 0.0, 0.0}; // MRF.DDt(U): Omega x U in the zone cells
        if (m.mrfCell && m.mrfCell[c])
        {
            const double* w = m.mrfOmega;
            cor[0] = w[1] * Uc[2] - w[2] * Uc[1];
            cor[1] = w[2] * Uc[0] - w[0] * Uc[2];
            cor[2] = w[0] * Uc[1] - w[1] * Uc[0];
        }
        for (int j = 0; j < 3; j++)
        {
            const double M = MV[j] * iV + cor[j] - (m.fvS ? m.fvS[(size_t)j * nC + c] : 0.0); // UEqn ... + MRF.DDt(U) - fvSource
            r.HbyA[(size_t)j * nT + c] = Uc[j] - rAU * M; // HbyA = rAU*H = U - rAU*(UEqn & U)
            R[3 * c + j] = (M + r.gP[(size_t)j * nT + c]) * cU;
        }
        if (q.turb)
        {
            const double src = saSource(ntc, q.nu, m.yWall[c], gUc, gNc, q.saFv3);
            R[4 * (size_t)nC + c] = (NV * iV + src) * (q.nrNut ? 1.0 : V);
        }
    }
};

// F_f = phiHbyA_f - rAU_f |S_f| snGrad(p)_f for an internal face, from the owner's point of view
DAB_HD double faceF(const MeshView& m, const StateView& s, const RecordView& r, int f, int o, int n)
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
    const double gam = w * r.rAU[o] + (1.0 - w) * r.rAU[n];
    const double sn = m.delta[f] * (s.p[n] - s.p[o]) + cg;
    if (m.mrfFlux) ph -= m.mrfFlux[f]; // MRF.makeRelative(phiHbyA)
    return ph - gam * mS * sn;
}

template <int NF>
struct FwdC
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    double* R;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const size_t offP = (size_t)3 * nC, offPhi = (size_t)(q.turb ? 5 : 4) * nC;
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
                F = faceF(m, s, r, f, o, n);
            }
            else
            {
                const int b = f - m.nIF, pa = m.bPatch[b];
                const double mS = m.magSf[f], dl = m.delta[f], phib = s.phi[f];
                const int kU = q.bcKind[F_U][pa];
                const bool assignable = (kU == BC_INLET_OUTLET || kU == BC_OUTLET_INLET || kU == BC_ZERO_GRADIENT);
                double ph = 0.0;
                if (q.constrainHbyA && !assignable)
                {
                    const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
                    const double im = frcp(mS);
                    const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
                    BCv bu;
                    double uw[3];
                    mrfWallRef(m, f, q.bcVal[F_U][pa], uw);
                    bcVector(kU, uw, Uc, phib, dl, nh, bu);
                    ph = m.Sx[f] * bu.val[0] + m.Sy[f] * bu.val[1] + m.Sz[f] * bu.val[2];
                }
                else
                    ph = m.Sx[f] * r.HbyA[c] + m.Sy[f] * r.HbyA[(size_t)nT + c] + m.Sz[f] * r.HbyA[(size_t)2 * nT + c];
                ph = mrfBoundaryFlux(m, f, ph, 1.0);
                double pv, sn, fr_;
                bcScalar(q.bcKind[F_P][pa], q.bcVal[F_P][pa][0], s.p[c], phib, dl, pv, sn, fr_);
                F = ph - r.rAU[c] * mS * sn;
            }
            div += fr.s * F;
            if (fr.s > 0) R[offPhi + f] = (F - s.phi[f]) * (q.nrPhi ? frcp(m.magSf[f]) : 1.0);
            else if (fr.n >= nC) R[offPhi + f] = 0.0; // cut face whose phi belongs to the neighbouring rank
        }
        R[offP + c] = -div * (q.nrP ? frcp(m.V[c]) : 1.0);
    }
};

} // namespace dab
