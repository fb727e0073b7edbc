// DARhoSimpleFoam: hand-derived reverse sweep y = diag(n) (dR/dW)^T x of the kernels in comp_kernels.hpp
// (the compressible counterpart of rev_kernels.hpp; reference DASolver::dRdWTMatVecMultFunction, DASolver.C:1364-1409).
//
// Structure: every dependence on the thermodynamic state goes through the cell closures (rho, nu, nut, rho*nuEff,
// alphaEff, he, Ekp) and their boundary-face counterparts.  The face kernels accumulate the adjoints of the closures;
// `closureAdj` (cell) and `boundaryPointAdj` (boundary face, followed by the BC transposes) turn them into adjoints of
// (U, p, T, nuTilda).  Gathers only, no atomics, as in the incompressible sweep.
//
//   cRevA  adjoint of cFwdC + cell-level adjoint of the momentum row
//   cRevB  face-level adjoint of the momentum and SA rows, phi adjoint (owner side)
//   cRevE  adjoint of the energy row (adds its phi part)
//   cRevC  adjoint of cFwdA: gradient transposes, closure adjoint, final sum and state scaling
#pragma once
#include "comp_kernels.hpp"
#include "rev_kernels.hpp"

namespace dab
{

// adjoints of the boundary values / closures of one boundary face (all start at zero)
struct BoundaryAdj
{
    double val[3], sng[3];
    double p, sngP, T, sngT, nt, sngN;
    double rho, nu, nut, muE, aE, Ek;
    DAB_HD void clear()
    {
        for (int j = 0; j < 3; j++) val[j] = sng[j] = 0.0;
        p = sngP = T = sngT = nt = sngN = rho = nu = nut = muE = aE = Ek = 0.0;
    }
};

DAB_HD double dmuSutherland(const Params& q, double T)
{
    const double sT = sqrt(T), den = 1.0 + q.Ts * frcp(T);
    return q.As * (0.5 * frcp(sT)) * frcp(den) + q.As * sT * (q.Ts * frcp(T * T)) * frcp(den * den);
}

// adjoint of the thermo point rho(p,T), mu(T), alpha(T), nu = mu/rho given adjoints of rho, nu and alpha
DAB_HD void thermoAdj(const Params& q, double p, double T, const ThermoPoint& th, double rhob, double nub, double alphab, double& pb, double& Tb)
{
    double mub = nub * frcp(th.rho);
    rhob -= nub * th.mu * frcp(th.rho * th.rho);
    if (q.sutherland)
    {
        const double Cv = q.Cp - q.Rg;
        mub += alphab * Cv * (1.32 + 1.77 * q.Rg * frcp(Cv)) * frcp(q.Cp);
        Tb += mub * dmuSutherland(q, T);
    }
    pb += rhob * frcp(q.Rg * T);
    Tb -= rhob * th.rho * frcp(T);
    (void)p;
}

// transpose of boundaryPoint: the adjoints in `a` -> adjoints of the cell values U_c, p_c, T_c, nuTilda_c and of nut_c
template <bool WF>
DAB_HD void boundaryPointAdj(const MeshView& m, const Params& q, const StateView& s, const RecordView& r, int f, int c, const BoundaryPoint& b,
                             BoundaryAdj a, double* Ub, double& pb, double& Tb, double& ntb, double& nutPb)
{
    const int pa = m.bPatch[f - m.nIF];
    const double phib = s.phi[f], dl = m.delta[f], im = frcp(m.magSf[f]);
    const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
    // Ek_b = 0.5|U_b|^2 (+ p_b/rho_b)
    for (int j = 0; j < 3; j++) a.val[j] += a.Ek * b.bu.val[j];
    if (q.heIsE)
    {
        a.p += a.Ek * frcp(b.th.rho);
        a.rho -= a.Ek * b.p * frcp(b.th.rho * b.th.rho);
    }
    // aE_b = CpByCpv (alpha_b + rho_b nut_b / Prt), muE_b = rho_b (nu_b + nut_b)
    const double kc = cpByCpv(q);
    double alphab = kc * a.aE;
    a.rho += kc * a.aE * b.nut * frcp(q.Prt) + a.muE * (b.th.nu + b.nut);
    a.nut += kc * a.aE * b.th.rho * frcp(q.Prt) + a.muE * b.th.rho;
    a.nu += a.muE * b.th.rho;
    // nut_b by BC kind
    if (q.turb && a.nut != 0.0)
    {
        const int kind = q.bcKind[F_NUT][pa];
        if (kind == BC_CALCULATED)
        {
            const double chi = b.nt * frcp(b.th.nu), c3 = chi * chi * chi, den = c3 + SA::Cv1c;
            const double fv1 = c3 * frcp(den), dfv1 = 3.0 * chi * chi * SA::Cv1c * frcp(den * den);
            a.nt += a.nut * (fv1 + chi * dfv1);
            a.nu -= a.nut * chi * chi * dfv1;
        }
        else if (kind == BC_NUT_SPALDING)
        {
            if (WF)
            {
                const double d[3] = {s.U[3 * c] - b.bu.val[0], s.U[3 * c + 1] - b.bu.val[1], s.U[3 * c + 2] - b.bu.val[2]};
                const double magUp = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
                double dM, dNu;
                nutSpalding2(magUp, dl, b.th.nu, dM, dNu);
                if (magUp > 0.0)
                    for (int j = 0; j < 3; j++)
                    {
                        Ub[j] += a.nut * dM * d[j] * frcp(magUp);
                        a.val[j] -= a.nut * dM * d[j] * frcp(magUp);
                    }
                a.nu += a.nut * dNu;
            }
        }
        else if (kind != BC_FIXED_VALUE && kind != BC_NUT_LOW_RE)
            nutPb += a.nut; // zeroGradient / symmetry: nut_b = nut_c
    }
    thermoAdj(q, b.p, b.T, b.th, a.rho, a.nu, alphab, a.p, a.T);
    // boundary values -> cell values through the BCs
    bcVectorAdj(q.bcKind[F_U][pa], phib, dl, nh, a.val, a.sng, Ub);
    pb += (1.0 - b.frP) * a.p - b.frP * dl * a.sngP;
    Tb += (1.0 - b.frT) * a.T - b.frT * dl * a.sngT;
    ntb += (1.0 - b.frN) * a.nt - b.frN * dl * a.sngN;
}

template <int NF>
struct cRevA
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    AdjView a;
    PsiView x;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double V = m.V[c];
        const double psiPc = x.p[c] * (q.nrP ? frcp(V) : 1.0);
        const double rhoc = r.rho[c], rAUc = r.rAU[c];
        double HbA[3] = {0, 0, 0}, rAUb = 0.0, pb = 0.0, Tb = 0.0, ntb = 0.0, nutPb = 0.0, gPb[3] = {0, 0, 0}, Ub[3] = {0, 0, 0}, rhob = 0.0;
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            const double mS = m.magSf[f], dl = m.delta[f];
            const double cphi = q.nrPhi ? frcp(mS) : 1.0;
            const double Sv[3] = {m.Sx[f], m.Sy[f], m.Sz[f]};
            if (!fr.bnd)
            {
                const int n = fr.n;
                const double psiPn = x.p[n] * (q.nrP ? frcp(m.V[n]) : 1.0);
                // F_f enters pRes_own with +1, pRes_nei with -1, phiRes_f with +1
                const double Fb = cphi * x.phi[f] + fr.s * (psiPc - psiPn);
                const double w = m.w[f];
                const double wc = fr.s > 0 ? w : 1.0 - w, wn = 1.0 - wc;
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                double cg = 0.0, ph = 0.0;
                for (int j = 0; j < 3; j++)
                {
                    cg += kv[j] * (wc * r.gP[(size_t)j * nT + c] + wn * r.gP[(size_t)j * nT + n]);
                    ph += Sv[j] * (wc * r.HbyA[(size_t)j * nT + c] + wn * r.HbyA[(size_t)j * nT + n]);
                }
                const double sn = fr.s * dl * (s.p[n] - s.p[c]) + cg;
                const double rhon = r.rho[n];
                const double rhof = wc * rhoc + wn * rhon;
                const double gam = wc * rhoc * rAUc + wn * rhon * r.rAU[n];
                if (m.mrfFlux) ph -= m.mrfFlux[f]; // owner-oriented, like ph, sn and Fb
                if (q.transonic)
                {
                    // F = phid p_f - gam |S| sn, phid = psi_f ph, p_f = wf p_own + (1 - wf) p_nei (cFaceF); this cell's share
                    const int o = fr.s > 0 ? c : n, nn = fr.s > 0 ? n : c;
                    const double Tc = s.T[c];
                    const double psif = wc * frcp(q.Rg * Tc) + wn * frcp(q.Rg * s.T[n]);
                    const double phid = psif * ph;
                    const double up = phid >= 0.0 ? 1.0 : 0.0;
                    double wf = up, dLimDr = 0.0, gradf = 1.0, gradcf = 0.0;
                    bool farBranch = false;
                    if (q.divPhidP == DIV_LINEAR) wf = w;
                    else if (q.divPhidP == DIV_LIMITED_LINEAR)
                    {
                        const double lim = limitedLinearLimiter(m, s, r, q.phidK, phid > 0.0, o, nn, dLimDr, gradf, gradcf, farBranch);
                        wf = lim * w + (1.0 - lim) * up;
                    }
                    const double pS = wf * s.p[o] + (1.0 - wf) * s.p[nn];
                    for (int j = 0; j < 3; j++) HbA[j] += wc * Sv[j] * psif * pS * Fb;
                    Tb -= wc * frcp(q.Rg * Tc * Tc) * ph * pS * Fb;
                    pb += (fr.s > 0 ? wf : 1.0 - wf) * phid * Fb;
                    if (dLimDr != 0.0)
                    {
                        const double G = phid * Fb * (s.p[o] - s.p[nn]) * (w - up) * dLimDr;
                        pb += G * (-2.0 * gradcf / (gradf * gradf)) * (-fr.s);
                        if ((phid > 0.0 ? o : nn) == c)
                        {
                            const double d[3] = {m.Cx[nn] - m.Cx[o], m.Cy[nn] - m.Cy[o], m.Cz[nn] - m.Cz[o]};
                            for (int j = 0; j < 3; j++) gPb[j] += G * (2.0 / gradf) * d[j];
                        }
                    }
                    rhob -= wc * rAUc * mS * sn * Fb;
                }
                else
                {
                    for (int j = 0; j < 3; j++) HbA[j] += wc * Sv[j] * rhof * Fb;
                    rhob += wc * (ph - rAUc * mS * sn) * Fb;
                }
                for (int j = 0; j < 3; j++) gPb[j] -= gam * mS * wc * kv[j] * Fb;
                rAUb -= wc * rhoc * mS * sn * Fb;
                pb += fr.s * gam * mS * dl * Fb;
            }
            else
            {
                BoundaryPoint bp;
                boundaryPoint<false>(m, q, s, r, f, c, bp);
                const int pa = m.bPatch[f - m.nIF];
                const double Fb = cphi * x.phi[f] + psiPc;
                const int kU = q.bcKind[F_U][pa];
                const bool assignable = (kU == BC_INLET_OUTLET || kU == BC_OUTLET_INLET || kU == BC_ZERO_GRADIENT);
                BoundaryAdj ba;
                ba.clear();
                double ph;
                const int mty = m.mrfType ? m.mrfType[f - m.nIF] : 0;
                if (mty == 1)
                    ph = 0.0; // rotating wall of the MRF zone: zero relative flux
                else if (q.constrainHbyA && !assignable)
                {
                    ph = Sv[0] * bp.bu.val[0] + Sv[1] * bp.bu.val[1] + Sv[2] * bp.bu.val[2];
                    for (int j = 0; j < 3; j++) ba.val[j] += Sv[j] * bp.th.rho * Fb;
                }
                else
                {
                    ph = Sv[0] * r.HbyA[c] + Sv[1] * r.HbyA[(size_t)nT + c] + Sv[2] * r.HbyA[(size_t)2 * nT + c];
                    for (int j = 0; j < 3; j++) HbA[j] += Sv[j] * bp.th.rho * Fb;
                }
                if (mty == 2) ph -= m.mrfFlux[f];
                ba.rho += (ph - rAUc * mS * bp.sngP) * Fb;
                rAUb -= bp.th.rho * mS * bp.sngP * Fb;
                ba.sngP -= bp.th.rho * rAUc * mS * Fb;
                boundaryPointAdj<false>(m, q, s, r, f, c, bp, ba, Ub, pb, Tb, ntb, nutPb);
            }
        }
        // cell-level adjoint of the momentum row: URes = cU*(M + grad p), HbyA = U - rAU*M, rAU = V/(Dn + icAvg)
        const double cU = q.nrU ? 1.0 : V;
        const double D0 = r.D0[c];
        double rAUtot = rAUb;
        double Mbv[3];
        for (int j = 0; j < 3; j++)
        {
            const double M = (Uc[j] - r.HbyA[(size_t)j * nT + c]) * frcp(rAUc);
            const double psiU = cU * x.U[3 * c + j];
            const double Mb = psiU - rAUc * HbA[j];
            Mbv[j] = Mb;
            rAUtot -= M * HbA[j];
            const double mt = Mb * frcp(V);
            a.mt[(size_t)j * nT + c] = mt;
            a.Udir[(size_t)j * nC + c] = Ub[j] + HbA[j] + D0 * mt;
            a.gPb[(size_t)j * nT + c] = gPb[j] + psiU;
        }
        if (m.mrfCell && m.mrfCell[c])
        {
            // adjoint of M += rho * (Omega x U): Ub += rho * (Mb x Omega), rhob += Mb . (Omega x U)
            const double* w = m.mrfOmega;
            a.Udir[c] += rhoc * (Mbv[1] * w[2] - Mbv[2] * w[1]);
            a.Udir[(size_t)nC + c] += rhoc * (Mbv[2] * w[0] - Mbv[0] * w[2]);
            a.Udir[(size_t)2 * nC + c] += rhoc * (Mbv[0] * w[1] - Mbv[1] * w[0]);
            rhob += Mbv[0] * (w[1] * Uc[2] - w[2] * Uc[1]) + Mbv[1] * (w[2] * Uc[0] - w[0] * Uc[2]) + Mbv[2] * (w[0] * Uc[1] - w[1] * Uc[0]);
        }
        a.Dn[c] = -rAUc * rAUc * rAUtot * frcp(V);
        a.pdir[c] = pb;
        a.Tdir[c] = Tb;
        a.cRho[c] = rhob;
        (void)ntb;
        (void)nutPb; // boundaryPoint<false>: no nut dependence in the pressure/flux rows
    }
};

template <int NF>
struct cRevB
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    AdjView a;
    PsiView x;
    double* y;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const size_t offPhi = (size_t)(q.turb ? 6 : 5) * nC;
        const int schU = q.divU, schN = q.divNut;
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double muEc = r.muE[c], rhoc = r.rho[c], nuc = r.nuL[c];
        double gUc[9], gNc[3];
        for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
        const double ntc = q.turb ? s.nt[c] : 0.0;
        const double Gc = rhoc * (ntc + nuc) * (1.0 / SA::sigma);
        for (int i = 0; i < 3; i++) gNc[i] = q.turb ? r.gNt[(size_t)i * nT + c] : 0.0;
        const double trc = gUc[0] + gUc[4] + gUc[8];
        const double V = m.V[c];
        const double mtc[3] = {a.mt[c], a.mt[(size_t)nT + c], a.mt[(size_t)2 * nT + c]};
        const double Dnc = a.Dn[c], flc = r.flag[c];
        const double D2c = Dnc * frcp(q.alphaU);
        const double D1c = flc != 0.0 ? flc * D2c : 0.0;
        const double soc = flc != 0.0 ? 0.0 : D2c;
        const double D0c = D1c + mtc[0] * Uc[0] + mtc[1] * Uc[1] + mtc[2] * Uc[2];
        const double psiN = q.turb ? x.nt[c] : 0.0;
        const double qc = psiN * (q.nrNut ? frcp(V) : 1.0);
        const double zc = psiN * (q.nrNut ? 1.0 : V);

        double U2[3] = {0, 0, 0}, nt2 = 0.0, muEb = 0.0, gUb[9], gNb[3] = {0, 0, 0};
        double rhob = 0.0, nub = 0.0, pb = 0.0, Tb = 0.0, nutPb = 0.0;
        for (int i = 0; i < 9; i++) gUb[i] = 0.0;

        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            const double phi = s.phi[f];
            const double mf = fr.s * phi;
            const double Sv[3] = {m.Sx[f], m.Sy[f], m.Sz[f]};
            const double mS = m.magSf[f], dl = m.delta[f];
            double phib_acc = 0.0;
            if (!fr.bnd)
            {
                const int n = fr.n;
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f], wn = 1.0 - wc;
                const bool pos0 = phi >= 0.0;
                const double wupc = fr.s > 0 ? (pos0 ? 1.0 : 0.0) : (pos0 ? 0.0 : 1.0);
                const double Un[3] = {s.U[3 * n], s.U[3 * n + 1], s.U[3 * n + 2]};
                const double muEn = r.muE[n];
                const double mtn[3] = {a.mt[n], a.mt[(size_t)nT + n], a.mt[(size_t)2 * nT + n]};
                const double Dnn = a.Dn[n], fln = r.flag[n];
                const double D2n = Dnn * frcp(q.alphaU);
                const double D1n = fln != 0.0 ? fln * D2n : 0.0;
                const double son = fln != 0.0 ? 0.0 : D2n;
                const double D0n = D1n + mtn[0] * Un[0] + mtn[1] * Un[1] + mtn[2] * Un[2];
                const bool ownUp = phi > 0.0;
                const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                const double dC[3] = {m.Cfx[f] - m.Cx[c], m.Cfy[f] - m.Cy[c], m.Cfz[f] - m.Cz[c]};
                {
                    const double wpc = schU == DIV_LINEAR ? wc : wupc;
                    const double wpn = schU == DIV_LINEAR ? wn : 1.0 - wupc;
                    const double gf = (wc * muEc + wn * muEn) * mS;
                    const double g = gf * dl;
                    const double offc = mf - wpc * mf - g;
                    const double offn = -mf + wpn * mf - g;
                    const double offbc = mtc[0] * Un[0] + mtc[1] * Un[1] + mtc[2] * Un[2] + sgn(offc) * soc;
                    const double offbn = mtn[0] * Uc[0] + mtn[1] * Uc[1] + mtn[2] * Uc[2] + sgn(offn) * son;
                    for (int j = 0; j < 3; j++) U2[j] += offn * mtn[j];
                    const double abc = D0c - offbc, abn = D0n - offbn;
                    double gb = abc + abn;
                    double gfb = 0.0;
                    const double lam[3] = {fr.s * (mtc[0] - mtn[0]), fr.s * (mtc[1] - mtn[1]), fr.s * (mtc[2] - mtn[2])};
                    double gUn[9];
                    for (int i = 0; i < 9; i++) gUn[i] = r.gU[(size_t)i * nT + n];
                    if (fr.s > 0)
                    {
                        const double mbc = -D0c + offbc + wpc * abc;
                        const double mbn = -D0n + offbn + wpn * abn;
                        phib_acc += mbc - mbn;
                    }
                    if (schU == DIV_LINEAR_UPWIND || schU == DIV_LINEAR_UPWIND_V)
                    {
                        double gu[9]; // per-element selects: a pointer into either array would put both in local memory
                        for (int i = 0; i < 9; i++) gu[i] = cUp ? gUc[i] : gUn[i];
                        const int u = cUp ? c : n;
                        const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                        double corr[3], corrL[3], outb[3], corrb[3] = {0, 0, 0};
                        for (int j = 0; j < 3; j++)
                        {
                            corr[j] = d[0] * gu[j * 3 + 0] + d[1] * gu[j * 3 + 1] + d[2] * gu[j * 3 + 2];
                            outb[j] = phi * lam[j];
                        }
                        if (schU == DIV_LINEAR_UPWIND_V)
                        {
                            const double wo_ = m.w[f];
                            const double cf = ownUp ? (1.0 - wo_) : -wo_;
                            double maxCorr[3], maxCorrb[3] = {0, 0, 0};
                            for (int j = 0; j < 3; j++) maxCorr[j] = cf * fr.s * (Un[j] - Uc[j]);
                            luvLimit(corr, maxCorr, corrL);
                            luvLimitAdj(corr, maxCorr, outb, corrb, maxCorrb);
                            for (int j = 0; j < 3; j++) U2[j] -= cf * fr.s * maxCorrb[j];
                        }
                        else
                            for (int j = 0; j < 3; j++) { corrL[j] = corr[j]; corrb[j] = outb[j]; }
                        if (cUp)
                            for (int j = 0; j < 3; j++)
                                for (int i = 0; i < 3; i++) gUb[j * 3 + i] += dC[i] * corrb[j];
                        if (fr.s > 0)
                            for (int j = 0; j < 3; j++) phib_acc += corrL[j] * lam[j];
                    }
                    for (int j = 0; j < 3; j++)
                    {
                        double cg = 0.0;
                        for (int i = 0; i < 3; i++) cg += kv[i] * (wc * gUc[j * 3 + i] + wn * gUn[j * 3 + i]);
                        gfb -= cg * lam[j];
                        const double cgb = -gf * lam[j];
                        for (int i = 0; i < 3; i++) gUb[j * 3 + i] += wc * kv[i] * cgb;
                    }
                    double trb = 0.0;
                    for (int j = 0; j < 3; j++)
                    {
                        const double tcb = -wc * lam[j];
                        const double tcj = Sv[0] * gUc[0 * 3 + j] + Sv[1] * gUc[1 * 3 + j] + Sv[2] * gUc[2 * 3 + j] - (2.0 / 3.0) * trc * Sv[j];
                        muEb += tcb * tcj;
                        for (int i = 0; i < 3; i++) gUb[i * 3 + j] += muEc * Sv[i] * tcb;
                        trb -= (2.0 / 3.0) * muEc * Sv[j] * tcb;
                    }
                    gUb[0] += trb; gUb[4] += trb; gUb[8] += trb;
                    muEb += wc * mS * (dl * gb + gfb);
                }
                if (q.turb)
                {
                    const double ntn = s.nt[n];
                    const double qn = x.nt[n] * (q.nrNut ? frcp(m.V[n]) : 1.0);
                    const double wpc = schN == DIV_LINEAR ? wc : wupc;
                    const double wpn = schN == DIV_LINEAR ? wn : 1.0 - wupc;
                    const double Gn = r.rho[n] * (ntn + r.nuL[n]) * (1.0 / SA::sigma);
                    const double gf = (wc * Gc + wn * Gn) * mS;
                    const double g = gf * dl;
                    nt2 += qc * (wpc * mf + g - mf) + qn * (-mf + wpn * mf - g);
                    const double gb = (qc - qn) * (ntc - ntn);
                    double gfb = 0.0;
                    const double lam = fr.s * (qc - qn);
                    if (fr.s > 0) phib_acc += qc * (1.0 - wpc) * (ntn - ntc) - qn * (1.0 - wpn) * (ntc - ntn);
                    if (schN == DIV_LINEAR_UPWIND)
                    {
                        if (cUp)
                            for (int i = 0; i < 3; i++) gNb[i] += dC[i] * phi * lam;
                        if (fr.s > 0)
                        {
                            const int u = cUp ? c : n;
                            const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                            double corr = 0.0;
                            for (int i = 0; i < 3; i++) corr += d[i] * r.gNt[(size_t)i * nT + u];
                            phib_acc += corr * lam;
                        }
                    }
                    double cg = 0.0;
                    for (int i = 0; i < 3; i++) cg += kv[i] * (wc * gNc[i] + wn * r.gNt[(size_t)i * nT + n]);
                    gfb -= cg * lam;
                    const double cgb = -gf * lam;
                    for (int i = 0; i < 3; i++) gNb[i] += wc * kv[i] * cgb;
                    // adjoint of G_c = rho_c (nuTilda_c + nu_c) / sigma
                    const double Gcb = wc * mS * (dl * gb + gfb);
                    nt2 += Gcb * rhoc * (1.0 / SA::sigma);
                    nub += Gcb * rhoc * (1.0 / SA::sigma);
                    rhob += Gcb * (ntc + nuc) * (1.0 / SA::sigma);
                }
            }
            else
            {
                BoundaryPoint bp;
                boundaryPoint<true>(m, q, s, r, f, c, bp);
                const double im = frcp(mS);
                const double nh[3] = {Sv[0] * im, Sv[1] * im, Sv[2] * im};
                const double G = bp.muE * mS;
                BoundaryAdj ba;
                ba.clear();
                double ic[3];
                int kmax = 0, kmin = 0;
                for (int j = 0; j < 3; j++)
                {
                    ic[j] = mf * bp.bu.vic[j] - G * bp.bu.gic[j];
                    if (j > 0)
                    {
                        if (fabs(ic[j]) > fabs(ic[kmax])) kmax = j;
                        if (ic[j] < ic[kmin]) kmin = j;
                    }
                }
                double mb = -D0c, Gb_ = 0.0;
                for (int j = 0; j < 3; j++)
                {
                    double icb = Dnc * (1.0 / 3.0);
                    if (j == kmin) icb -= Dnc;
                    if (j == kmax) icb += D1c * sgn(ic[j]);
                    mb += bp.bu.vic[j] * icb + mtc[j] * bp.bu.val[j];
                    Gb_ += -bp.bu.gic[j] * icb - mtc[j] * bp.bu.sng[j];
                }
                for (int j = 0; j < 3; j++) { ba.val[j] = mf * mtc[j]; ba.sng[j] = -G * mtc[j]; }
                double Gbd[9];
                for (int j = 0; j < 3; j++)
                {
                    const double nG = nh[0] * gUc[j * 3 + 0] + nh[1] * gUc[j * 3 + 1] + nh[2] * gUc[j * 3 + 2];
                    for (int i = 0; i < 3; i++) Gbd[j * 3 + i] = gUc[j * 3 + i] + nh[i] * (bp.bu.sng[j] - nG);
                }
                const double trbv = Gbd[0] + Gbd[4] + Gbd[8];
                double muEBb = mS * Gb_;
                double Gbb[9];
                for (int i = 0; i < 9; i++) Gbb[i] = 0.0;
                double trbb = 0.0;
                for (int j = 0; j < 3; j++)
                {
                    const double X = Sv[0] * Gbd[0 * 3 + j] + Sv[1] * Gbd[1 * 3 + j] + Sv[2] * Gbd[2 * 3 + j] - (2.0 / 3.0) * trbv * Sv[j];
                    muEBb -= X * mtc[j];
                    const double Xb = -bp.muE * mtc[j];
                    for (int i = 0; i < 3; i++) Gbb[i * 3 + j] += Sv[i] * Xb;
                    trbb -= (2.0 / 3.0) * Sv[j] * Xb;
                }
                Gbb[0] += trbb; Gbb[4] += trbb; Gbb[8] += trbb;
                boundaryGradAdj(nh, Gbb, gUb, ba.sng);
                ba.muE += muEBb;
                if (q.turb)
                {
                    // SA boundary part: NV += mf*nt_b - Gs*sngN - mf*nt_c, Gs = rho_b (nt_b + nu_b)/sigma |S|
                    const double Gs = bp.th.rho * (bp.nt + bp.th.nu) * (1.0 / SA::sigma) * mS;
                    mb += qc * (bp.nt - ntc);
                    ba.nt += qc * mf;
                    ba.sngN -= qc * Gs;
                    const double Gsb = -qc * bp.sngN;
                    ba.rho += Gsb * (bp.nt + bp.th.nu) * (1.0 / SA::sigma) * mS;
                    ba.nt += Gsb * bp.th.rho * (1.0 / SA::sigma) * mS;
                    ba.nu += Gsb * bp.th.rho * (1.0 / SA::sigma) * mS;
                    nt2 -= qc * mf;
                }
                boundaryPointAdj<true>(m, q, s, r, f, c, bp, ba, U2, pb, Tb, nt2, nutPb);
                phib_acc += mb;
            }
            if (fr.s > 0)
                y[offPhi + f] = (phib_acc - (q.nrPhi ? frcp(mS) : 1.0) * x.phi[f]) * phiRowScale(q, mS);
            else if (fr.n >= nC)
                y[offPhi + f] = 0.0;
        }
        if (q.turb)
        {
            // cell-local SA sources: rho_c * saSource(nt, nu_c, ...)
            rhob += zc * saSource(ntc, nuc, m.yWall[c], gUc, gNc, q.saFv3);
            saSourceAdj(ntc, nuc, m.yWall[c], gUc, gNc, zc * rhoc, nt2, gUb, gNb, q.saFv3, &nub);
        }
        for (int j = 0; j < 3; j++) a.U2[(size_t)j * nC + c] = U2[j];
        a.nt2[c] = nt2;
        a.nutb[c] = nutPb;
        a.cMuE[c] = muEb;
        a.cNu[c] = nub;
        a.cRho[c] += rhob;
        a.pdir[c] += pb;
        a.Tdir[c] += Tb;
        for (int i = 0; i < 9; i++) a.gUb[(size_t)i * nT + c] = gUb[i];
        for (int i = 0; i < 3; i++) a.gNtb[(size_t)i * nT + c] = gNb[i];
    }
};

template <int NF>
struct cRevE
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    AdjView a;
    PsiView x;
    double* y;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const size_t offPhi = (size_t)(q.turb ? 6 : 5) * nC;
        const int schE = q.divE;
        const double heA = q.heIsE ? (q.Cp - q.Rg) : q.Cp;
        const double hec = r.he[c], aEc = r.aE[c], Ekc = r.Ek[c];
        double gHc[3];
        for (int i = 0; i < 3; i++) gHc[i] = r.gHe[(size_t)i * nT + c];
        const double qc = x.T[c] * (q.nrT ? frcp(m.V[c]) : 1.0);
        double he2 = 0.0, aEb = 0.0, Ekb = 0.0, gHb[3] = {0, 0, 0};
        double Ub[3] = {0, 0, 0}, pb = 0.0, Tb = 0.0, ntb = 0.0, nutPb = 0.0;
        double twb[3] = {0.0, 0.0, 0.0}, gUt[9], gUtb[9]; // turboH: adjoint of this cell's work vector, grad(U) and its adjoint
        if (q.turboH)
            for (int i = 0; i < 9; i++)
            {
                gUt[i] = r.gU[(size_t)i * nT + c];
                gUtb[i] = 0.0;
            }
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            const double phi = s.phi[f];
            const double mf = fr.s * phi;
            const double mS = m.magSf[f], dl = m.delta[f];
            double phib_acc = 0.0;
            if (!fr.bnd)
            {
                const int n = fr.n;
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f], wn = 1.0 - wc;
                const bool pos0 = phi >= 0.0;
                const double wupc = fr.s > 0 ? (pos0 ? 1.0 : 0.0) : (pos0 ? 0.0 : 1.0);
                const bool ownUp = phi > 0.0;
                const bool cUp = fr.s > 0 ? ownUp : !ownUp;
                const double hen = r.he[n];
                const double qn = x.T[n] * (q.nrT ? frcp(m.V[n]) : 1.0);
                const double wpc = schE == DIV_LINEAR ? wc : wupc;
                const double wpn = schE == DIV_LINEAR ? wn : 1.0 - wupc;
                const double gf = (wc * aEc + wn * r.aE[n]) * mS;
                const double g = gf * dl;
                he2 += qc * (wpc * mf + g - mf) + qn * (-mf + wpn * mf - g);
                const double gb = (qc - qn) * (hec - hen);
                double gfb = 0.0;
                const double lam = fr.s * (qc - qn);
                if (fr.s > 0) phib_acc += qc * (1.0 - wpc) * (hen - hec) - qn * (1.0 - wpn) * (hec - hen);
                const double kv[3] = {m.kx[f], m.ky[f], m.kz[f]};
                if (schE == DIV_LINEAR_UPWIND)
                {
                    const double dC[3] = {m.Cfx[f] - m.Cx[c], m.Cfy[f] - m.Cy[c], m.Cfz[f] - m.Cz[c]};
                    if (cUp)
                        for (int i = 0; i < 3; i++) gHb[i] += dC[i] * phi * lam;
                    if (fr.s > 0)
                    {
                        const int u = cUp ? c : n;
                        const double d[3] = {m.Cfx[f] - m.Cx[u], m.Cfy[f] - m.Cy[u], m.Cfz[f] - m.Cz[u]};
                        double corr = 0.0;
                        for (int i = 0; i < 3; i++) corr += d[i] * r.gHe[(size_t)i * nT + u];
                        phib_acc += corr * lam;
                    }
                }
                double cg = 0.0;
                for (int i = 0; i < 3; i++) cg += kv[i] * (wc * gHc[i] + wn * r.gHe[(size_t)i * nT + n]);
                gfb -= cg * lam;
                const double cgb = -gf * lam;
                for (int i = 0; i < 3; i++) gHb[i] += wc * kv[i] * cgb;
                aEb += wc * mS * (dl * gb + gfb);
                // Ekp term: row c  mf (1-wk_c)(Ek_n - Ek_c), row n  mf wk_c (Ek_n - Ek_c)
                const double wk = q.divEkp == DIV_LINEAR ? wc : wupc;
                Ekb -= mf * (qc * (1.0 - wk) + qn * wk);
                if (fr.s > 0) phib_acc += (qc * (1.0 - wk) + qn * wk) * (r.Ek[n] - Ekc);
                if (q.turboH)
                {
                    // the cell's work vector enters row c and row n through this face with weight wc
                    const double cf = -fr.s * wc * (qc - qn);
                    twb[0] += cf * m.Sx[f];
                    twb[1] += cf * m.Sy[f];
                    twb[2] += cf * m.Sz[f];
                }
            }
            else
            {
                BoundaryPoint bp;
                boundaryPoint<true>(m, q, s, r, f, c, bp);
                BoundaryAdj ba;
                ba.clear();
                const double sngH = heA * bp.sngT;
                // EV += mf*he_b - aE_b |S| sngH - mf*he_c + mf (Ek_b - Ek_c)
                ba.T += heA * qc * mf;
                ba.sngT -= heA * qc * bp.aE * mS;
                ba.aE -= qc * mS * sngH;
                ba.Ek += qc * mf;
                he2 -= qc * mf;
                Ekb -= qc * mf;
                phib_acc += qc * (bp.th.he - hec + bp.Ek - Ekc);
                if (q.turboH)
                {
                    const double im = frcp(mS);
                    const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
                    double Gb[9], Gbb[9], vr[3];
                    for (int j = 0; j < 3; j++)
                    {
                        const double nG = nh[0] * gUt[j * 3 + 0] + nh[1] * gUt[j * 3 + 1] + nh[2] * gUt[j * 3 + 2];
                        for (int i = 0; i < 3; i++)
                        {
                            Gb[j * 3 + i] = gUt[j * 3 + i] + nh[i] * (bp.bu.sng[j] - nG);
                            Gbb[j * 3 + i] = 0.0;
                        }
                    }
                    const bool onZone = m.mrfType && m.mrfType[f - m.nIF] != 0;
                    if (onZone) mrfVelocityAt(m, m.Cfx[f], m.Cfy[f], m.Cfz[f], vr);
                    const double qb3[3] = {-qc * m.Sx[f], -qc * m.Sy[f], -qc * m.Sz[f]};
                    turboWorkAdj(Gb, bp.muE, bp.bu.val, onZone ? vr : nullptr, qb3, Gbb, ba.muE, ba.val, ba.p);
                    boundaryGradAdj(nh, Gbb, gUtb, ba.sng);
                }
                boundaryPointAdj<true>(m, q, s, r, f, c, bp, ba, Ub, pb, Tb, ntb, nutPb);
            }
            if (fr.s > 0) y[offPhi + f] += phib_acc * phiRowScale(q, mS);
        }
        if (q.turboH)
        {
            const double uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
            double vr[3], mub = 0.0;
            const bool inZone = m.mrfCell && m.mrfCell[c];
            if (inZone) mrfVelocityAt(m, m.Cx[c], m.Cy[c], m.Cz[c], vr);
            turboWorkAdj(gUt, r.muE[c], uc, inZone ? vr : nullptr, twb, gUtb, mub, Ub, pb);
            a.cMuE[c] += mub;
            for (int i = 0; i < 9; i++) a.gUb[(size_t)i * nT + c] += gUtb[i];
        }
        a.cAE[c] = aEb;
        a.cHe[c] = he2;
        a.cEk[c] = Ekb;
        for (int i = 0; i < 3; i++) a.gHeb[(size_t)i * nT + c] = gHb[i];
        if (m.fvS)
            for (int j = 0; j < 3; j++) Ub[j] -= x.T[c] * (q.nrT ? 1.0 : m.V[c]) * m.fvS[(size_t)j * nC + c]; // EV -= V (fvSource . U)
        for (int j = 0; j < 3; j++) a.Udir[(size_t)j * nC + c] += Ub[j];
        a.pdir[c] += pb;
        a.Tdir[c] += Tb;
        a.nt2[c] += ntb;
        a.nutb[c] += nutPb;
    }
};

template <int NF>
struct cRevC
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    AdjView a;
    double* y;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        const double heA = q.heIsE ? (q.Cp - q.Rg) : q.Cp;
        const double Uc[3] = {s.U[3 * c], s.U[3 * c + 1], s.U[3 * c + 2]};
        const double iVc = frcp(m.V[c]);
        double Ub[3], pb = a.pdir[c], Tb = a.Tdir[c], nb = q.turb ? a.nt2[c] : 0.0, heb = a.cHe[c];
        for (int j = 0; j < 3; j++) Ub[j] = a.Udir[(size_t)j * nC + c] + a.U2[(size_t)j * nC + c];
        double gUbc[9], gPbc[3], gNbc[3], gHbc[3];
        for (int i = 0; i < 9; i++) gUbc[i] = a.gUb[(size_t)i * nT + c] * iVc;
        for (int i = 0; i < 3; i++)
        {
            gPbc[i] = a.gPb[(size_t)i * nT + c] * iVc;
            gNbc[i] = q.turb ? a.gNtb[(size_t)i * nT + c] * iVc : 0.0;
            gHbc[i] = a.gHeb[(size_t)i * nT + c] * iVc;
        }
        DAB_FACE_PREFETCH(NF)
        _Pragma("unroll") for (int k = 0; k < (NF > 0 ? NF : m.maxCF); k++)
        {
            const FaceRef fr = DAB_FACE(NF, k);
            if (fr.f < 0) break;
            const int f = fr.f;
            const double So[3] = {fr.s * m.Sx[f], fr.s * m.Sy[f], fr.s * m.Sz[f]};
            if (!fr.bnd)
            {
                const int n = fr.n;
                const double wc = fr.s > 0 ? m.w[f] : 1.0 - m.w[f];
                const double iVn = frcp(m.V[n]);
                for (int j = 0; j < 3; j++)
                {
                    double t = 0.0;
                    for (int i = 0; i < 3; i++) t += So[i] * (gUbc[j * 3 + i] - a.gUb[(size_t)(j * 3 + i) * nT + n] * iVn);
                    Ub[j] += wc * t;
                }
                double tp = 0.0, tn = 0.0, th = 0.0;
                for (int i = 0; i < 3; i++)
                {
                    tp += So[i] * (gPbc[i] - a.gPb[(size_t)i * nT + n] * iVn);
                    if (q.turb) tn += So[i] * (gNbc[i] - a.gNtb[(size_t)i * nT + n] * iVn);
                    th += So[i] * (gHbc[i] - a.gHeb[(size_t)i * nT + n] * iVn);
                }
                pb += wc * tp;
                nb += wc * tn;
                heb += wc * th;
            }
            else
            {
                const int pa = m.bPatch[f - m.nIF];
                const double phib = s.phi[f], dl = m.delta[f];
                const double im = frcp(m.magSf[f]);
                const double nh[3] = {m.Sx[f] * im, m.Sy[f] * im, m.Sz[f] * im};
                double valb[3];
                const double sngb[3] = {0.0, 0.0, 0.0};
                for (int j = 0; j < 3; j++) valb[j] = So[0] * gUbc[j * 3 + 0] + So[1] * gUbc[j * 3 + 1] + So[2] * gUbc[j * 3 + 2];
                bcVectorAdj(q.bcKind[F_U][pa], phib, dl, nh, valb, sngb, Ub);
                const double frp = bcFrac(q.bcKind[F_P][pa], phib);
                pb += (1.0 - frp) * (So[0] * gPbc[0] + So[1] * gPbc[1] + So[2] * gPbc[2]);
                if (q.turb)
                {
                    const double frn = bcFrac(q.bcKind[F_NUTILDA][pa], phib);
                    nb += (1.0 - frn) * (So[0] * gNbc[0] + So[1] * gNbc[1] + So[2] * gNbc[2]);
                }
                // he_b = he(T_b), T_b = frT*Tref + (1-frT)*T_c
                const double frt = bcFrac(q.bcKindT[pa], phib);
                Tb += heA * (1.0 - frt) * (So[0] * gHbc[0] + So[1] * gHbc[1] + So[2] * gHbc[2]);
            }
        }
        // cell closure adjoint: rho, nu, nut, muE = rho (nu + nut), aE = k (alpha + rho nut/Prt), he = heA T + heB, Ek
        {
            const double pc = s.p[c], Tc = s.T[c];
            const ThermoPoint th = thermoOf(q, pc, Tc);
            const double ntc = q.turb ? s.nt[c] : 0.0;
            const double nut = r.nut[c];
            const double kc = cpByCpv(q);
            double rhob = a.cRho[c], nub = q.turb ? a.cNu[c] : 0.0, nutb = q.turb ? a.nutb[c] : 0.0;
            const double muEb = a.cMuE[c], aEb = a.cAE[c], Ekb = a.cEk[c];
            for (int j = 0; j < 3; j++) Ub[j] += Ekb * Uc[j];
            if (q.heIsE)
            {
                pb += Ekb * frcp(th.rho);
                rhob -= Ekb * pc * frcp(th.rho * th.rho);
            }
            Tb += heA * heb;
            const double alphab = kc * aEb;
            rhob += kc * aEb * nut * frcp(q.Prt) + muEb * (th.nu + nut);
            nutb += kc * aEb * th.rho * frcp(q.Prt) + muEb * th.rho;
            nub += muEb * th.rho;
            if (q.turb)
            {
                const double chi = ntc * frcp(th.nu), c3 = chi * chi * chi, den = c3 + SA::Cv1c;
                const double fv1 = c3 * frcp(den), dfv1 = 3.0 * chi * chi * SA::Cv1c * frcp(den * den);
                nb += nutb * (fv1 + chi * dfv1);
                nub -= nutb * chi * chi * dfv1;
            }
            thermoAdj(q, pc, Tc, th, rhob, nub, alphab, pb, Tb);
        }
        for (int j = 0; j < 3; j++) y[3 * c + j] = Ub[j] * q.sU;
        y[(size_t)3 * nC + c] = pb * q.sP;
        y[(size_t)4 * nC + c] = Tb * q.sT;
        if (q.turb) y[(size_t)5 * nC + c] = nb * q.sNut;
    }
};

// ---- force / moment function (DAFunctionForce.C:79-153 with the compressible devRhoReff = -rho*nuEff*dev(twoSymm(grad U)))
// fv (optional, modes 0, 1): the face's force vector Sf (p_b - pRef) + Sf & devRhoReff_b
DAB_HD double cForceFace(const MeshView& m, const Params& q, const StateView& s, const RecordView& r, const ForceSpec& fs, int f, int c,
                         double seed, double* Ub, double* pb, double* Tb, double* ntb, double* nutPb, double* gUb, double* fv = nullptr)
{
    const int nT = m.nCtot;
    const double mS = m.magSf[f];
    const double Sv[3] = {m.Sx[f], m.Sy[f], m.Sz[f]};
    const double im = frcp(mS);
    const double nh[3] = {Sv[0] * im, Sv[1] * im, Sv[2] * im};
    double gUc[9];
    for (int i = 0; i < 9; i++) gUc[i] = r.gU[(size_t)i * nT + c];
    BoundaryPoint bp;
    boundaryPoint<true>(m, q, s, r, f, c, bp);
    if (fs.mode >= 2)
    {
        const double U2 = bp.bu.val[0] * bp.bu.val[0] + bp.bu.val[1] * bp.bu.val[1] + bp.bu.val[2] * bp.bu.val[2];
        const double wA = mS * frcp(fs.areaSum);
        const double SU = Sv[0] * bp.bu.val[0] + Sv[1] * bp.bu.val[1] + Sv[2] * bp.bu.val[2];
        double F, pTp = 0.0, pTT = 0.0, pTU = 0.0; // mode 4: d(pT)/dp, /dT, /d(|U|^2)
        if (fs.mode == 4)
        {
            // p (1 + (gamma-1)/2 Ma^2)^(gamma/(gamma-1)), Ma^2 = |U|^2/(gamma R T), R = Cp - Cp/gamma (DAFunctionTotalPressureRatio.C:96-125)
            const double gam = fs.gamma, Rg = q.Cp - q.Cp * frcp(gam), ex = gam * frcp(gam - 1.0);
            const double Ma2 = U2 * frcp(gam * Rg * bp.T);
            const double base = 1.0 + 0.5 * (gam - 1.0) * Ma2;
            const double pw = pow(base, ex);
            const double dMa = bp.p * ex * pw * frcp(base) * 0.5 * (gam - 1.0); // d(pT)/d(Ma2)
            F = fs.scale * (bp.p * pw - fs.shift) * wA;
            pTp = pw;
            pTU = dMa * frcp(gam * Rg * bp.T);
            pTT = -dMa * Ma2 * frcp(bp.T);
        }
        else
            F = fs.scale * (fs.mode == 2 ? (bp.p + 0.5 * bp.th.rho * U2 - fs.shift) * wA : bp.th.rho * SU);
        if (gUb)
        {
            const double fb = seed * fs.scale;
            BoundaryAdj ba;
            ba.clear();
            if (fs.mode == 4)
            {
                ba.p += fb * wA * pTp;
                ba.T += fb * wA * pTT;
                for (int j = 0; j < 3; j++) ba.val[j] += fb * wA * pTU * 2.0 * bp.bu.val[j];
            }
            else if (fs.mode == 2)
            {
                ba.p += fb * wA;
                ba.rho += fb * wA * 0.5 * U2;
                for (int j = 0; j < 3; j++) ba.val[j] += fb * wA * bp.th.rho * bp.bu.val[j];
            }
            else
            {
                ba.rho += fb * SU;
                for (int j = 0; j < 3; j++) ba.val[j] += fb * bp.th.rho * Sv[j];
            }
            boundaryPointAdj<true>(m, q, s, r, f, c, bp, ba, Ub, *pb, *Tb, *ntb, *nutPb);
        }
        return F;
    }
    double Gbd[9];
    for (int j = 0; j < 3; j++)
    {
        const double nG = nh[0] * gUc[j * 3 + 0] + nh[1] * gUc[j * 3 + 1] + nh[2] * gUc[j * 3 + 2];
        for (int i = 0; i < 3; i++) Gbd[j * 3 + i] = gUc[j * 3 + i] + nh[i] * (bp.bu.sng[j] - nG);
    }
    const double trb = Gbd[0] + Gbd[4] + Gbd[8];
    double ed[3] = {fs.dir[0], fs.dir[1], fs.dir[2]};
    if (fs.faceDir)
        for (int j = 0; j < 3; j++) ed[j] = fs.faceDir[3 * (f - m.nIF) + j];
    else if (fs.mode == 1)
    {
        const double rv[3] = {m.Cfx[f] - fs.center[0], m.Cfy[f] - fs.center[1], m.Cfz[f] - fs.center[2]};
        ed[0] = fs.dir[1] * rv[2] - fs.dir[2] * rv[1];
        ed[1] = fs.dir[2] * rv[0] - fs.dir[0] * rv[2];
        ed[2] = fs.dir[0] * rv[1] - fs.dir[1] * rv[0];
    }
    double F = 0.0, sj[3];
    for (int j = 0; j < 3; j++)
    {
        double t = 0.0;
        for (int i = 0; i < 3; i++) t += Sv[i] * (Gbd[j * 3 + i] + Gbd[i * 3 + j]);
        sj[j] = t - (2.0 / 3.0) * trb * Sv[j];
        const double fj = Sv[j] * (bp.p - fs.pRef) - bp.muE * sj[j];
        if (fv) fv[j] = fj;
        F += fj * ed[j];
    }
    F *= fs.scale;
    if (gUb)
    {
        BoundaryAdj ba;
        ba.clear();
        double Gbb[9];
        for (int i = 0; i < 9; i++) Gbb[i] = 0.0;
        double trbb = 0.0;
        for (int j = 0; j < 3; j++)
        {
            const double fb = seed * fs.scale * ed[j];
            ba.p += Sv[j] * fb;
            ba.muE -= sj[j] * fb;
            const double sb = -bp.muE * fb;
            for (int i = 0; i < 3; i++)
            {
                Gbb[j * 3 + i] += Sv[i] * sb;
                Gbb[i * 3 + j] += Sv[i] * sb;
            }
            trbb -= (2.0 / 3.0) * Sv[j] * sb;
        }
        Gbb[0] += trbb; Gbb[4] += trbb; Gbb[8] += trbb;
        boundaryGradAdj(nh, Gbb, gUb, ba.sng);
        boundaryPointAdj<true>(m, q, s, r, f, c, bp, ba, Ub, *pb, *Tb, *ntb, *nutPb);
    }
    return F;
}

struct cForceFwd
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    ForceSpec fs;
    double* out; // [nBF]
    DAB_HD void operator()(int b) const
    {
        const int f = m.nIF + b;
        if (!((fs.mask >> m.bPatch[b]) & 1u))
        {
            if (!fs.accumulate) out[b] = 0.0;
            return;
        }
        out[b] = cForceFace(m, q, s, r, fs, f, m.own[f], 0.0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    }
};

// seeds every reverse work array of the cell with dF/d(cell variables); cRevC then finishes the sweep
template <int NF>
struct cForceRevA
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    AdjView a;
    ForceSpec fs;
    double seed;
    DAB_HD void operator()(int c) const
    {
        const int nT = m.nCtot, nC = m.nC;
        double Ub[3] = {0, 0, 0}, pb = 0.0, Tb = 0.0, ntb = 0.0, nutPb = 0.0, gUb[9];
        for (int i = 0; i < 9; i++) gUb[i] = 0.0;
        for (int k = 0; k < m.maxCF; k++)
        {
            const FaceRef fr = faceOf(m, c, k);
            if (fr.f < 0) break;
            if (!fr.bnd) continue;
            if (!((fs.mask >> m.bPatch[fr.f - m.nIF]) & 1u)) continue;
            cForceFace(m, q, s, r, fs, fr.f, c, seed, Ub, &pb, &Tb, &ntb, &nutPb, gUb);
        }
        for (int j = 0; j < 3; j++)
        {
            a.Udir[(size_t)j * nC + c] = 0.0;
            a.U2[(size_t)j * nC + c] = Ub[j];
        }
        a.pdir[c] = pb;
        a.Tdir[c] = Tb;
        a.nt2[c] = ntb;
        a.nutb[c] = nutPb;
        a.cRho[c] = a.cNu[c] = a.cMuE[c] = a.cAE[c] = a.cHe[c] = a.cEk[c] = 0.0;
        for (int i = 0; i < 9; i++) a.gUb[(size_t)i * nT + c] = gUb[i];
        (void)NF;
    }
};

} // namespace dab
