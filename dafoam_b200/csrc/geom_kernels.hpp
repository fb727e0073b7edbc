// Mesh geometry on the device (the same formulas as HostMesh::computeGeometry, which restates OpenFOAM's
// primitiveMesh face/cell centres and areas, surfaceInterpolation weights, nonOrthDeltaCoeffs and
// nonOrthCorrectionVectors) and the kernels of the `volCoord` input: [dR/dx_v]^T psi and dF/dx_v
// (reference src/adjoint/DAInput/DAInputVolCoord.C:35-70 through DASolver::calcJacTVecProduct, DASolver.C:1690-1839).
//
// The reference differentiates the geometry + residual with CoDiPack.  Here the product is evaluated by coloured
// central differences over the mesh points (the approach of the reference's own pre-AD DAPartDeriv machinery):
// points whose residual footprints are disjoint are moved together, the geometry and R(W) are re-evaluated on the
// device with the hot-path kernels, and psi . (R+ - R-)/(2 eps) is attributed to the point whose footprint the row
// lies in.  Exact to O(eps^2) ~ 1e-9 relative; a hand-derived reverse of the geometry dependence is the planned
// replacement (DESIGN.md).
#pragma once
#include "views.hpp"
#include <cmath>

namespace dab
{

struct GeomView
{
    int nC, nF, nIF, maxCF;
    const int32_t *fOff, *fLab, *own, *nei, *cellFaces;
    const double* pts; // [3*nP]
    double *Sx, *Sy, *Sz, *magSf, *w, *delta, *kx, *ky, *kz, *Cfx, *Cfy, *Cfz, *Cx, *Cy, *Cz, *V;
    // partitioned local mesh with cyclic pairs: faceXf[f] = k > 0 puts face f into the neighbour's frame (inverse of transform k,
    // rotations Rtab / translations Ttab as in comm.hpp); nullptr: no such face
    const int32_t* faceXf;
    const double *Rtab, *Ttab;
};

// face area vector and centroid (primitiveMesh::makeFaceCentresAndAreas)
struct GeomFaceK
{
    GeomView g;
    DAB_HD void operator()(int f) const
    {
        const int n = g.fOff[f + 1] - g.fOff[f];
        const int32_t* l = g.fLab + g.fOff[f];
        const double* P = g.pts;
        double cf[3], sf[3];
        if (n == 3)
        {
            double a[3], b[3];
            for (int k = 0; k < 3; k++)
            {
                cf[k] = (P[3 * l[0] + k] + P[3 * l[1] + k] + P[3 * l[2] + k]) / 3.0;
                a[k] = P[3 * l[1] + k] - P[3 * l[0] + k];
                b[k] = P[3 * l[2] + k] - P[3 * l[0] + k];
            }
            sf[0] = 0.5 * (a[1] * b[2] - a[2] * b[1]);
            sf[1] = 0.5 * (a[2] * b[0] - a[0] * b[2]);
            sf[2] = 0.5 * (a[0] * b[1] - a[1] * b[0]);
        }
        else
        {
            double est[3] = {0, 0, 0};
            for (int i = 0; i < n; i++)
                for (int k = 0; k < 3; k++) est[k] += P[3 * l[i] + k];
            for (int k = 0; k < 3; k++) est[k] /= n;
            double sumN[3] = {0, 0, 0}, sumAc[3] = {0, 0, 0}, sumA = 0.0;
            for (int i = 0; i < n; i++)
            {
                const double* p0 = P + 3 * l[i];
                const double* p1 = P + 3 * l[(i + 1) % n];
                double a[3], b[3], nn[3], c[3];
                for (int k = 0; k < 3; k++)
                {
                    a[k] = p1[k] - p0[k];
                    b[k] = est[k] - p0[k];
                    c[k] = p0[k] + p1[k] + est[k];
                }
                nn[0] = a[1] * b[2] - a[2] * b[1];
                nn[1] = a[2] * b[0] - a[0] * b[2];
                nn[2] = a[0] * b[1] - a[1] * b[0];
                const double an = sqrt(nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2]);
                for (int k = 0; k < 3; k++)
                {
                    sumN[k] += nn[k];
                    sumAc[k] += an * c[k];
                }
                sumA += an;
            }
            for (int k = 0; k < 3; k++)
            {
                cf[k] = (1.0 / 3.0) / sumA * sumAc[k];
                sf[k] = 0.5 * sumN[k];
            }
        }
        g.magSf[f] = sqrt(sf[0] * sf[0] + sf[1] * sf[1] + sf[2] * sf[2]);
        const int x = g.faceXf ? g.faceXf[f] : 0;
        if (x > 0)
        {
            // the neighbour-side copy of a coupled face (HostMesh::xfPoint / xfVector, inverse, the same operation order)
            const double* M = g.Rtab + 9 * (x - 1);
            const double* t = g.Ttab + 3 * (x - 1);
            const double d[3] = {cf[0] - t[0], cf[1] - t[1], cf[2] - t[2]}, s0[3] = {sf[0], sf[1], sf[2]};
            for (int a = 0; a < 3; a++)
            {
                cf[a] = M[a] * d[0] + M[3 + a] * d[1] + M[6 + a] * d[2];
                sf[a] = M[a] * s0[0] + M[3 + a] * s0[1] + M[6 + a] * s0[2];
            }
        }
        g.Cfx[f] = cf[0]; g.Cfy[f] = cf[1]; g.Cfz[f] = cf[2];
        g.Sx[f] = sf[0]; g.Sy[f] = sf[1]; g.Sz[f] = sf[2];
    }
};

// cell centroid and volume from the face pyramids (primitiveMesh::makeCellCentresAndVols); owned cells only -- on a partitioned
// mesh the ghost cells' centres and volumes come from their owners through the halo (centres as positions)
struct GeomCellK
{
    GeomView g;
    DAB_HD void operator()(int c) const
    {
        double est[3] = {0, 0, 0};
        int cnt = 0;
        for (int k = 0; k < g.maxCF; k++)
        {
            const int e = g.cellFaces[(size_t)k * g.nC + c];
            if (e < 0) break;
            const int f = e >> 1;
            est[0] += g.Cfx[f]; est[1] += g.Cfy[f]; est[2] += g.Cfz[f];
            cnt++;
        }
        for (int j = 0; j < 3; j++) est[j] /= cnt;
        double C[3] = {0, 0, 0}, V = 0.0;
        for (int k = 0; k < g.maxCF; k++)
        {
            const int e = g.cellFaces[(size_t)k * g.nC + c];
            if (e < 0) break;
            const int f = e >> 1;
            const double s = (e & 1) ? -1.0 : 1.0;
            const double cf[3] = {g.Cfx[f], g.Cfy[f], g.Cfz[f]};
            const double pyr3 = s * (g.Sx[f] * (cf[0] - est[0]) + g.Sy[f] * (cf[1] - est[1]) + g.Sz[f] * (cf[2] - est[2]));
            for (int j = 0; j < 3; j++) C[j] += pyr3 * (0.75 * cf[j] + 0.25 * est[j]);
            V += pyr3;
        }
        g.Cx[c] = C[0] / V; g.Cy[c] = C[1] / V; g.Cz[c] = C[2] / V;
        g.V[c] = V / 3.0;
    }
};

// interpolation weights, nonOrthDeltaCoeffs and nonOrthCorrectionVectors (surfaceInterpolation::makeWeights etc.)
struct GeomDerivedK
{
    GeomView g;
    DAB_HD void operator()(int f) const
    {
        const double S[3] = {g.Sx[f], g.Sy[f], g.Sz[f]}, mS = g.magSf[f];
        const double nh[3] = {S[0] / mS, S[1] / mS, S[2] / mS};
        const double cf[3] = {g.Cfx[f], g.Cfy[f], g.Cfz[f]};
        const int o = g.own[f];
        const double Co[3] = {g.Cx[o], g.Cy[o], g.Cz[o]};
        if (f < g.nIF)
        {
            const int n = g.nei[f];
            const double Cn[3] = {g.Cx[n], g.Cy[n], g.Cz[n]};
            double dO = 0.0, dN = 0.0, d[3], nd = 0.0, md = 0.0;
            for (int k = 0; k < 3; k++)
            {
                dO += S[k] * (cf[k] - Co[k]);
                dN += S[k] * (Cn[k] - cf[k]);
                d[k] = Cn[k] - Co[k];
                nd += nh[k] * d[k];
                md += d[k] * d[k];
            }
            dO = fabs(dO);
            dN = fabs(dN);
            g.w[f] = dN / (dO + dN);
            md = sqrt(md);
            const double lim = 0.05 * md;
            const double dl = 1.0 / (nd > lim ? nd : lim);
            g.delta[f] = dl;
            g.kx[f] = nh[0] - dl * d[0];
            g.ky[f] = nh[1] - dl * d[1];
            g.kz[f] = nh[2] - dl * d[2];
        }
        else
        {
            double dn = 0.0;
            for (int k = 0; k < 3; k++) dn += nh[k] * (cf[k] - Co[k]);
            double nd = 0.0, md = 0.0;
            for (int k = 0; k < 3; k++)
            {
                const double dk = dn * nh[k];
                nd += nh[k] * dk;
                md += dk * dk;
            }
            const double lim = 0.05 * sqrt(md);
            g.w[f] = 1.0;
            g.delta[f] = 1.0 / (nd > lim ? nd : lim);
            g.kx[f] = 0.0; g.ky[f] = 0.0; g.kz[f] = 0.0;
        }
    }
};

// pts[3p+k] = pts0[3p+k] + sign*eps[p] for the points of the list (sign 0 restores)
struct PointMove
{
    double* pts;
    const double* pts0;
    const double* eps;
    const int32_t* list;
    int k;
    double sign;
    DAB_HD void operator()(int t) const
    {
        const int p = list[t];
        pts[3 * p + k] = pts0[3 * p + k] + sign * eps[p];
    }
};

// footprint labels: label[c] = global id of the home cell whose ball c lies in (-1: none), over owned and ghost cells; doubles,
// so that a partitioned mesh refreshes the ghost labels through the halo after every sweep (the ids are exact integers)
struct LabelInit
{
    double* label;
    DAB_HD void operator()(int c) const { label[c] = -1.0; }
};
struct LabelSeed
{
    double* label;
    const int32_t* cells; // local cells (owned or ghost) that are homes of the colour
    const int32_t* ids;   // their global ids
    DAB_HD void operator()(int t) const { label[cells[t]] = (double)ids[t]; }
};
// one propagation sweep over the owned cells
struct LabelSweep
{
    const double* in;
    double* out;
    const int32_t* cellNbr;
    int nC, maxCF;
    DAB_HD void operator()(int c) const
    {
        double l = in[c];
        if (l < 0.0)
            for (int k = 0; k < maxCF; k++)
            {
                const int n = cellNbr[(size_t)k * nC + c];
                if (n >= 0 && in[n] > l) l = in[n];
            }
        out[c] = l;
    }
};

DAB_HD void atomicAddD(double* a, double v)
{
#if defined(__CUDA_ARCH__)
    atomicAdd(a, v);
#else
    *a += v;
#endif
}

// out[3p+k] += psi . (R+ - R-) / (2 eps_p) over the rows of cell c, p = the point of slot `slot` of c's footprint home
struct VolCoordAccumR
{
    MeshView m;
    int ns, offPhi; // cell-state rows: U (3 per cell, AoS) then ns-3 scalar blocks; face rows from offPhi
    const double *Rp, *Rm, *psi;
    const double* label;
    const int32_t* slotPoint; // [global cells * maxSlots]
    int maxSlots, slot, k;
    const double* eps;
    double* out;
    DAB_HD void operator()(int c) const
    {
        const int h = (int)label[c];
        if (h < 0) return;
        const int p = slotPoint[(size_t)h * maxSlots + slot];
        if (p < 0) return;
        const int nC = m.nC;
        double s = 0.0;
        for (int j = 0; j < 3; j++) s += psi[3 * c + j] * (Rp[3 * c + j] - Rm[3 * c + j]);
        for (int b = 3; b < ns; b++) s += psi[(size_t)b * nC + c] * (Rp[(size_t)b * nC + c] - Rm[(size_t)b * nC + c]);
        for (int q = 0; q < m.maxCF; q++)
        {
            const int e = m.cellFaces[(size_t)q * nC + c];
            if (e < 0) break;
            if (e & 1) continue; // the owner side carries the face row
            const int f = e >> 1;
            s += psi[offPhi + f] * (Rp[offPhi + f] - Rm[offPhi + f]);
        }
        if (s != 0.0) atomicAddD(out + 3 * p + k, s / (2.0 * eps[p]));
    }
};

// the same for a function assembled from boundary-face parts (force / moment)
struct VolCoordAccumF
{
    MeshView m;
    const double *Fp, *Fm; // [nBF]
    const double* label;
    const int32_t* slotPoint;
    int maxSlots, slot, k;
    const double* eps;
    double seed;
    double* out;
    DAB_HD void operator()(int b) const
    {
        const int c = m.own[m.nIF + b];
        const int h = (int)label[c];
        if (h < 0) return;
        const int p = slotPoint[(size_t)h * maxSlots + slot];
        if (p < 0) return;
        const double s = Fp[b] - Fm[b];
        if (s != 0.0) atomicAddD(out + 3 * p + k, seed * s / (2.0 * eps[p]));
    }
};

} // namespace dab
