// Host mesh: OpenFOAM polyMesh topology + finite-volume geometry, laid out as the SoA arrays the
// device kernels read.  Replaces, for the adjoint hot path, OpenFOAM's fvMesh / surfaceInterpolation
// geometry (primitiveMeshFaceCentresAndAreas, primitiveMeshCellCentresAndVols, makeWeights,
// makeNonOrthDeltaCoeffs, makeNonOrthCorrectionVectors) that the reference reaches through
// `meshPtr_` (reference src/adjoint/DASolver/DASolver.C:58-64) and the boundary-face maps of DAIndex
// (reference src/adjoint/DAIndex/DAIndex.C:66-112).
#pragma once
#include "foam_io.hpp"
#include <algorithm>
#include <cmath>

namespace dab
{

enum PatchGeom { PG_PATCH = 0, PG_WALL = 1, PG_SYMMETRY = 2, PG_PROCESSOR = 3 };

struct HostMesh
{
    // topology
    int nP = 0, nF = 0, nIF = 0, nBF = 0, nC = 0;
    int nCtot = 0;        // owned + ghost cells (ghosts appended; nCtot == nC on one rank)
    int nInterior = -1;   // owned cells [0, nInterior) have no neighbour on another rank (-1: all of them)
    std::vector<double> points;          // 3*nP
    std::vector<int32_t> fOff, fLab;     // faces -> points
    std::vector<int32_t> own, nei;       // nei sized nIF
    std::vector<PatchDef> patches;
    std::vector<int32_t> patchGeom;      // PatchGeom per patch
    std::vector<int32_t> bPatch;         // patch of boundary face b
    int maxCF = 0;
    std::vector<int32_t> cellFaces;      // ELL: [k*nC + c] = (f<<1)|isNeighbour, -1 padding
    std::vector<int32_t> cellNbr;        // ELL: the cell across that face, -1 on boundary faces / padding
    // cyclic (periodic) patch pairs are merged into internal faces when the mesh is read (mergeCyclics): the owner is the cell on the
    // first patch of the pair, the neighbour the cell on the second one, and cyc[f] = k > 0 names the transform that maps the
    // neighbour's side into the owner's frame (positions x' = R x + t, vectors v' = R v).  The local mesh of a rank holds such a
    // neighbour as a ghost cell whose copies are transformed on the way (partition.hpp, comm.hpp), so no kernel knows about it.
    struct CycXf { double R[9]; double t[3]; };
    std::vector<int32_t> cyc;            // per internal face (global mesh only); empty = no cyclic faces
    std::vector<CycXf> xforms;           // transform k is xforms[k - 1]
    // the coupled face pairs as read, for the check of moved points (checkCyclicPairs): pair i has the points of the first-patch face
    // cycA[cycAOff[i]..] and of the second-patch face cycB[cycBOff[i]..] and the transform cycXf[i]; kept by every local mesh
    std::vector<int32_t> cycAOff, cycA, cycBOff, cycB, cycXf;
    bool hasCyclic() const { return !xforms.empty(); }
    static void xfPoint(const CycXf& X, bool inverse, const double* x, double* y)
    {
        if (!inverse)
            for (int a = 0; a < 3; a++) y[a] = X.R[3 * a] * x[0] + X.R[3 * a + 1] * x[1] + X.R[3 * a + 2] * x[2] + X.t[a];
        else
        {
            const double d[3] = {x[0] - X.t[0], x[1] - X.t[1], x[2] - X.t[2]};
            for (int a = 0; a < 3; a++) y[a] = X.R[a] * d[0] + X.R[3 + a] * d[1] + X.R[6 + a] * d[2];
        }
    }
    static void xfVector(const CycXf& X, bool inverse, const double* v, double* y)
    {
        for (int a = 0; a < 3; a++)
            y[a] = inverse ? X.R[a] * v[0] + X.R[3 + a] * v[1] + X.R[6 + a] * v[2] : X.R[3 * a] * v[0] + X.R[3 * a + 1] * v[1] + X.R[3 * a + 2] * v[2];
    }
    // geometry (SoA)
    std::vector<double> Sf[3], Cf[3], corr[3]; // per face
    std::vector<double> magSf, w, delta;       // per face (w = 1 on boundary faces)
    std::vector<double> C[3], V, yWall;        // per cell

    void read(const std::string& caseDir)
    {
        const std::string pm = caseDir + "/constant/polyMesh/";
        readVectorField(pm + "points", points);
        readFaceList(pm + "faces", fOff, fLab);
        readLabelList(pm + "owner", own);
        readLabelList(pm + "neighbour", nei);
        patches = readBoundary(pm + "boundary");
        mergeCyclics();
        finalizeTopology();
    }

    // centre and area vector of face f from its points (OpenFOAM primitiveMeshFaceCentresAndAreas)
    void faceGeom(int f, double* cf, double* sf) const { polyGeom(&fLab[fOff[f]], fOff[f + 1] - fOff[f], cf, sf); }
    void polyGeom(const int32_t* l, int n, double* cf, double* sf) const
    {
        const double* P = points.data();
        if (n == 3)
        {
            for (int k = 0; k < 3; k++) cf[k] = (P[3 * l[0] + k] + P[3 * l[1] + k] + P[3 * l[2] + k]) / 3.0;
            double a[3], b[3];
            for (int k = 0; k < 3; k++) { a[k] = P[3 * l[1] + k] - P[3 * l[0] + k]; b[k] = P[3 * l[2] + k] - P[3 * l[0] + k]; }
            sf[0] = 0.5 * (a[1] * b[2] - a[2] * b[1]); sf[1] = 0.5 * (a[2] * b[0] - a[0] * b[2]); sf[2] = 0.5 * (a[0] * b[1] - a[1] * b[0]);
            return;
        }
        double est[3] = {0, 0, 0};
        for (int i = 0; i < n; i++)
            for (int k = 0; k < 3; k++) est[k] += P[3 * l[i] + k];
        for (int k = 0; k < 3; k++) est[k] /= n;
        double sumN[3] = {0, 0, 0}, sumAc[3] = {0, 0, 0}, sumA = 0.0;
        for (int i = 0; i < n; i++)
        {
            const double* p0 = &P[3 * l[i]];
            const double* p1 = &P[3 * l[(i + 1) % n]];
            double a[3], b[3], nn[3], c[3];
            for (int k = 0; k < 3; k++) { a[k] = p1[k] - p0[k]; b[k] = est[k] - p0[k]; c[k] = p0[k] + p1[k] + est[k]; }
            nn[0] = a[1] * b[2] - a[2] * b[1]; nn[1] = a[2] * b[0] - a[0] * b[2]; nn[2] = a[0] * b[1] - a[1] * b[0];
            double an = std::sqrt(nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2]);
            for (int k = 0; k < 3; k++) { sumN[k] += nn[k]; sumAc[k] += an * c[k]; }
            sumA += an;
        }
        for (int k = 0; k < 3; k++) { cf[k] = (1.0 / 3.0) / sumA * sumAc[k]; sf[k] = 0.5 * sumN[k]; }
    }

    // the read-time rule of a coupled pair: the transform maps the second face onto the first (centres coincide, area vectors opposite)
    static bool pairMatches(const CycXf& X, const double* cA, const double* sA, const double* cB, const double* sB, double scale)
    {
        double y[3], v[3], mA = 0.0;
        xfPoint(X, false, cB, y);
        xfVector(X, false, sB, v);
        for (int a = 0; a < 3; a++) mA = std::max(mA, std::fabs(sA[a]));
        for (int a = 0; a < 3; a++)
            if (std::fabs(y[a] - cA[a]) > 1e-6 * scale || std::fabs(v[a] + sA[a]) > 1e-6 * mA) return false;
        return true;
    }
    double pointScale() const
    {
        double scale = 0.0;
        for (size_t i = 0; i < points.size(); i++) scale = std::max(scale, std::fabs(points[i]));
        return scale;
    }
    // moved points (updateOFMesh): every coupled pair must still match under its (fixed) transform, i.e. the displacement is periodic
    void checkCyclicPairs() const
    {
        const double scale = pointScale();
        for (size_t i = 0; i + 1 < cycAOff.size(); i++)
        {
            double cA[3], sA[3], cB[3], sB[3];
            polyGeom(&cycA[cycAOff[i]], cycAOff[i + 1] - cycAOff[i], cA, sA);
            polyGeom(&cycB[cycBOff[i]], cycBOff[i + 1] - cycBOff[i], cB, sB);
            if (!pairMatches(xforms[cycXf[i] - 1], cA, sA, cB, sB, scale))
                throw Error("updateOFMesh: coupled face pair " + std::to_string(i) + " of cyclic transform " + std::to_string(cycXf[i])
                            + " no longer matches under the patch transform (the displacement must be periodic)");
        }
    }

    // Cyclic patch pairs -> internal faces (OpenFOAM cyclicPolyPatch: face i of a patch is coupled to face i of its neighbourPatch;
    // DAFoam counts both sides as coupled boundary faces with a phi state each, reference src/adjoint/DAIndex/DAIndex.C:151-167 --
    // here a pair shares ONE face and one phi state, like the cut faces between ranks).  The transform is taken from the geometry of
    // the two patches (translation: mean offset of the face centres; rotation: angle about rotationAxis / rotationCentre that maps
    // the second patch onto the first) and checked on every face pair.
    void mergeCyclics()
    {
        std::vector<int> isCyc(patches.size(), 0);
        bool any = false;
        for (size_t p = 0; p < patches.size(); p++)
            if (patches[p].type == "cyclic") { isCyc[p] = 1; any = true; }
        if (!any) return;
        const int nF0 = (int)own.size(), nIF0 = (int)nei.size();
        auto patchIndex = [&](const std::string& n) {
            for (size_t p = 0; p < patches.size(); p++)
                if (patches[p].name == n) return (int)p;
            throw Error("polyMesh: cyclic neighbourPatch " + n + " not found");
        };
        std::vector<int32_t> newOwn(own.begin(), own.begin() + nIF0), newNei(nei), newCyc(nIF0, 0);
        std::vector<int> faceOrder(nIF0);
        for (int f = 0; f < nIF0; f++) faceOrder[f] = f;
        const double scale = pointScale();
        for (size_t p = 0; p < patches.size(); p++)
        {
            if (!isCyc[p]) continue;
            const int q = patchIndex(patches[p].neighbourPatch);
            if (!isCyc[q] || patches[q].neighbourPatch != patches[p].name) throw Error("polyMesh: cyclic patches " + patches[p].name + " / " + patches[q].name + " do not name each other");
            if ((int)p > q) continue; // handled with its partner
            if ((int)p == q) throw Error("polyMesh: cyclic patch " + patches[p].name + " is its own neighbour");
            const PatchDef &A = patches[p], &B = patches[q];
            if (A.size != B.size) throw Error("polyMesh: cyclic patches " + A.name + " / " + B.name + " differ in size");
            const int n = A.size;
            std::vector<double> cA((size_t)3 * n), sA((size_t)3 * n), cB((size_t)3 * n), sB((size_t)3 * n);
            for (int i = 0; i < n; i++)
            {
                faceGeom(A.start + i, &cA[3 * (size_t)i], &sA[3 * (size_t)i]);
                faceGeom(B.start + i, &cB[3 * (size_t)i], &sB[3 * (size_t)i]);
            }
            CycXf X;
            for (int a = 0; a < 9; a++) X.R[a] = (a % 4 == 0) ? 1.0 : 0.0;
            for (int a = 0; a < 3; a++) X.t[a] = 0.0;
            bool rotational = A.transform == "rotational";
            if (A.transform != "rotational" && A.transform != "translational" && A.hasAxis && n > 0)
            {
                // unknown / noOrdering: coupled faces of a translation have opposite area vectors
                double dev = 0.0, mag = 0.0;
                for (int i = 0; i < 3 * n; i++) { dev = std::max(dev, std::fabs(sA[i] + sB[i])); mag = std::max(mag, std::fabs(sA[i])); }
                rotational = dev > 1e-6 * mag;
            }
            if (rotational)
            {
                if (!A.hasAxis) throw Error("polyMesh: rotational cyclic patch " + A.name + " without rotationAxis");
                double ax[3] = {A.rotationAxis[0], A.rotationAxis[1], A.rotationAxis[2]};
                const double an = std::sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
                if (!(an > 0.0)) throw Error("polyMesh: zero rotationAxis on " + A.name);
                for (int a = 0; a < 3; a++) ax[a] /= an;
                const double* c0 = A.rotationCentre;
                // angle that takes the second patch onto the first: area-weighted mean over the face pairs
                double sumW = 0.0, sumTh = 0.0;
                for (int i = 0; i < n; i++)
                {
                    double rA[3], rB[3], dA = 0.0, dB = 0.0;
                    for (int a = 0; a < 3; a++) { rA[a] = cA[3 * (size_t)i + a] - c0[a]; rB[a] = cB[3 * (size_t)i + a] - c0[a]; dA += rA[a] * ax[a]; dB += rB[a] * ax[a]; }
                    for (int a = 0; a < 3; a++) { rA[a] -= dA * ax[a]; rB[a] -= dB * ax[a]; }
                    const double cr[3] = {rB[1] * rA[2] - rB[2] * rA[1], rB[2] * rA[0] - rB[0] * rA[2], rB[0] * rA[1] - rB[1] * rA[0]};
                    const double sn = cr[0] * ax[0] + cr[1] * ax[1] + cr[2] * ax[2], cs = rA[0] * rB[0] + rA[1] * rB[1] + rA[2] * rB[2];
                    const double wgt = std::sqrt(rA[0] * rA[0] + rA[1] * rA[1] + rA[2] * rA[2]) * std::sqrt(rB[0] * rB[0] + rB[1] * rB[1] + rB[2] * rB[2]);
                    if (!(wgt > 0.0)) continue;
                    sumW += wgt;
                    sumTh += wgt * std::atan2(sn, cs);
                }
                if (!(sumW > 0.0)) throw Error("polyMesh: cannot determine the rotation angle of cyclic patch " + A.name);
                const double th = sumTh / sumW, c = std::cos(th), s1 = std::sin(th), C1 = 1.0 - c;
                const double x = ax[0], y = ax[1], z = ax[2];
                const double R[9] = {c + x * x * C1, x * y * C1 - z * s1, x * z * C1 + y * s1,
                                     y * x * C1 + z * s1, c + y * y * C1, y * z * C1 - x * s1,
                                     z * x * C1 - y * s1, z * y * C1 + x * s1, c + z * z * C1};
                for (int a = 0; a < 9; a++) X.R[a] = R[a];
                for (int a = 0; a < 3; a++) X.t[a] = c0[a] - (R[3 * a] * c0[0] + R[3 * a + 1] * c0[1] + R[3 * a + 2] * c0[2]);
            }
            else
            {
                double t[3] = {0, 0, 0};
                for (int i = 0; i < n; i++)
                    for (int a = 0; a < 3; a++) t[a] += cA[3 * (size_t)i + a] - cB[3 * (size_t)i + a];
                for (int a = 0; a < 3; a++) X.t[a] = n ? t[a] / n : 0.0;
            }
            // every coupled pair must map onto each other: centres coincide, area vectors are opposite
            for (int i = 0; i < n; i++)
                if (!pairMatches(X, &cA[3 * (size_t)i], &sA[3 * (size_t)i], &cB[3 * (size_t)i], &sB[3 * (size_t)i], scale))
                    throw Error("polyMesh: faces " + std::to_string(i) + " of cyclic patches " + A.name + " / " + B.name
                                + " do not match under the patch transform (ordering or transform entry)");
            xforms.push_back(X);
            const int k = (int)xforms.size();
            if (cycAOff.empty()) { cycAOff.push_back(0); cycBOff.push_back(0); }
            for (int i = 0; i < n; i++)
            {
                for (int q = fOff[A.start + i]; q < fOff[A.start + i + 1]; q++) cycA.push_back(fLab[q]);
                for (int q = fOff[B.start + i]; q < fOff[B.start + i + 1]; q++) cycB.push_back(fLab[q]);
                cycAOff.push_back((int32_t)cycA.size());
                cycBOff.push_back((int32_t)cycB.size());
                cycXf.push_back(k);
            }
            for (int i = 0; i < n; i++)
            {
                newOwn.push_back(own[A.start + i]);
                newNei.push_back(own[B.start + i]);
                newCyc.push_back(k);
                faceOrder.push_back(A.start + i);
            }
        }
        const int nIF1 = (int)newNei.size();
        std::vector<PatchDef> newPatches;
        for (size_t p = 0; p < patches.size(); p++)
        {
            if (isCyc[p]) continue;
            PatchDef pd = patches[p];
            pd.start = (int)faceOrder.size();
            for (int i = 0; i < patches[p].size; i++)
            {
                faceOrder.push_back(patches[p].start + i);
                newOwn.push_back(own[patches[p].start + i]);
            }
            newPatches.push_back(pd);
        }
        (void)nF0;
        std::vector<int32_t> nOff(1, 0), nLab;
        nLab.reserve(fLab.size());
        for (int f : faceOrder)
        {
            for (int i = fOff[f]; i < fOff[f + 1]; i++) nLab.push_back(fLab[i]);
            nOff.push_back((int32_t)nLab.size());
        }
        fOff.swap(nOff);
        fLab.swap(nLab);
        own.swap(newOwn);
        nei.swap(newNei);
        cyc.swap(newCyc);
        patches.swap(newPatches);
        (void)nIF1;
    }

    void finalizeTopology()
    {
        nP = (int)(points.size() / 3);
        nF = (int)own.size();
        nIF = (int)nei.size();
        nBF = nF - nIF;
        if ((int)fOff.size() != nF + 1) throw Error("polyMesh: faces/owner size mismatch");
        nC = 0;
        for (int f = 0; f < nF; f++) nC = std::max(nC, own[f] + 1);
        for (int f = 0; f < nIF; f++) nC = std::max(nC, nei[f] + 1);
        nCtot = nC;
        patchGeom.resize(patches.size());
        bPatch.assign(nBF, -1);
        for (size_t p = 0; p < patches.size(); p++)
        {
            const std::string& ty = patches[p].type;
            patchGeom[p] = ty == "wall" ? PG_WALL : ((ty == "symmetry" || ty == "symmetryPlane") ? PG_SYMMETRY : PG_PATCH);
            if (patches[p].start < nIF || patches[p].start + patches[p].size > nF) throw Error("polyMesh: bad patch range " + patches[p].name);
            for (int i = 0; i < patches[p].size; i++) bPatch[patches[p].start - nIF + i] = (int32_t)p;
        }
        for (int b = 0; b < nBF; b++)
            if (bPatch[b] < 0) throw Error("polyMesh: boundary face without patch");
        // ELL cell -> faces
        std::vector<int> cnt(nC, 0);
        for (int f = 0; f < nF; f++)
        {
            cnt[own[f]]++;
            if (f < nIF) cnt[nei[f]]++;
        }
        maxCF = *std::max_element(cnt.begin(), cnt.end());
        cellFaces.assign((size_t)maxCF * nC, -1);
        std::fill(cnt.begin(), cnt.end(), 0);
        // rows filled in ascending face id, and boundary ids are >= nIF: every row is [internal..., boundary..., -1 padding]
        // (checkEllOrder).  RevB walks a row in two passes on this invariant (rev_kernels.hpp)
        for (int f = 0; f < nF; f++)
        {
            int c = own[f];
            cellFaces[(size_t)cnt[c]++ * nC + c] = (f << 1);
            if (f < nIF)
            {
                c = nei[f];
                cellFaces[(size_t)cnt[c]++ * nC + c] = (f << 1) | 1;
            }
        }
        checkEllOrder();
    }

    // every ELL row lists its internal faces, then its boundary faces, then padding
    void checkEllOrder() const
    {
        for (int c = 0; c < nC; c++)
        {
            int stage = 0; // 0 internal, 1 boundary, 2 padding
            for (int k = 0; k < maxCF; k++)
            {
                const int e = cellFaces[(size_t)k * nC + c];
                const int s = e < 0 ? 2 : ((e >> 1) >= nIF ? 1 : 0);
                if (s < stage) throw Error("mesh: ELL row of cell " + std::to_string(c) + " is not ordered internal, boundary, padding");
                stage = s;
            }
        }
    }

    void buildCellNbr()
    {
        cellNbr.assign(cellFaces.size(), -1);
        for (size_t i = 0; i < cellFaces.size(); i++)
        {
            const int e = cellFaces[i];
            if (e < 0) continue;
            const int f = e >> 1;
            if (f < nIF) cellNbr[i] = (e & 1) ? own[f] : nei[f];
        }
    }

    // OpenFOAM-v1812 geometry definitions (see file header)
    void computeGeometry()
    {
        for (int k = 0; k < 3; k++)
        {
            Sf[k].assign(nF, 0.0); Cf[k].assign(nF, 0.0); corr[k].assign(nF, 0.0); C[k].assign(nC, 0.0);
        }
        magSf.assign(nF, 0.0); w.assign(nF, 1.0); delta.assign(nF, 0.0); V.assign(nC, 0.0);
        for (int f = 0; f < nF; f++)
        {
            double cf[3], sf[3];
            faceGeom(f, cf, sf);
            for (int k = 0; k < 3; k++) { Cf[k][f] = cf[k]; Sf[k][f] = sf[k]; }
            magSf[f] = std::sqrt(sf[0] * sf[0] + sf[1] * sf[1] + sf[2] * sf[2]);
        }
        // face centre / area vector as the cell on `side` sees them: the neighbour of a cyclic face lives in its own frame
        auto sideGeom = [&](int f, int side, double* cf, double* sf) {
            for (int k = 0; k < 3; k++) { cf[k] = Cf[k][f]; sf[k] = Sf[k][f]; }
            if (side == 1 && f < (int)cyc.size() && cyc[f] > 0)
            {
                const CycXf& X = xforms[cyc[f] - 1];
                double c0[3] = {cf[0], cf[1], cf[2]}, s0[3] = {sf[0], sf[1], sf[2]};
                xfPoint(X, true, c0, cf);
                xfVector(X, true, s0, sf);
            }
        };
        std::vector<double> est((size_t)3 * nC, 0.0);
        std::vector<int> cnt(nC, 0);
        for (int f = 0; f < nF; f++)
            for (int side = 0; side < (f < nIF ? 2 : 1); side++)
            {
                const int c = side == 0 ? own[f] : nei[f];
                double cf[3], sf[3];
                sideGeom(f, side, cf, sf);
                for (int k = 0; k < 3; k++) est[3 * (size_t)c + k] += cf[k];
                cnt[c]++;
            }
        for (int c = 0; c < nC; c++)
            for (int k = 0; k < 3; k++) est[3 * (size_t)c + k] /= cnt[c];
        for (int f = 0; f < nF; f++)
        {
            for (int side = 0; side < (f < nIF ? 2 : 1); side++)
            {
                const int c = side == 0 ? own[f] : nei[f];
                double cf[3], sf[3];
                sideGeom(f, side, cf, sf);
                double pyr3 = 0.0;
                for (int k = 0; k < 3; k++)
                    pyr3 += sf[k] * (side == 0 ? (cf[k] - est[3 * (size_t)c + k]) : (est[3 * (size_t)c + k] - cf[k]));
                for (int k = 0; k < 3; k++) C[k][c] += pyr3 * (0.75 * cf[k] + 0.25 * est[3 * (size_t)c + k]);
                V[c] += pyr3;
            }
        }
        for (int c = 0; c < nC; c++)
        {
            for (int k = 0; k < 3; k++) C[k][c] /= V[c];
            V[c] /= 3.0;
            if (!(V[c] > 0.0)) throw Error("polyMesh: non-positive cell volume");
        }
        for (int f = 0; f < nF; f++)
        {
            double nh[3] = {Sf[0][f] / magSf[f], Sf[1][f] / magSf[f], Sf[2][f] / magSf[f]};
            if (f < nIF)
            {
                const int o = own[f], n = nei[f];
                double Cn[3] = {C[0][n], C[1][n], C[2][n]};
                if (f < (int)cyc.size() && cyc[f] > 0)
                {
                    const double c0[3] = {Cn[0], Cn[1], Cn[2]};
                    xfPoint(xforms[cyc[f] - 1], false, c0, Cn); // the neighbour's centre in the owner's frame
                }
                double dO = 0.0, dN = 0.0, d[3], nd = 0.0, md = 0.0;
                for (int k = 0; k < 3; k++)
                {
                    dO += Sf[k][f] * (Cf[k][f] - C[k][o]);
                    dN += Sf[k][f] * (Cn[k] - Cf[k][f]);
                    d[k] = Cn[k] - C[k][o];
                    nd += nh[k] * d[k];
                    md += d[k] * d[k];
                }
                dO = std::fabs(dO); dN = std::fabs(dN);
                w[f] = dN / (dO + dN);
                md = std::sqrt(md);
                delta[f] = 1.0 / std::max(nd, 0.05 * md);
                for (int k = 0; k < 3; k++) corr[k][f] = nh[k] - delta[f] * d[k];
            }
            else
            {
                const int o = own[f];
                double dn = 0.0;
                for (int k = 0; k < 3; k++) dn += nh[k] * (Cf[k][f] - C[k][o]);
                double d[3], nd = 0.0, md = 0.0;
                for (int k = 0; k < 3; k++) { d[k] = dn * nh[k]; nd += nh[k] * d[k]; md += d[k] * d[k]; }
                delta[f] = 1.0 / std::max(nd, 0.05 * std::sqrt(md));
            }
        }
    }

    // ---- exact distance to the wall faces for the cells next to a wall (OpenFOAM wallDist `correctWalls true`: patchWave ->
    // cellDistFuncs::correctBoundaryFaceCells / correctBoundaryPointCells; face::nearestPointClassify decomposes a face into the
    // triangles (p_i, p_i+1, face centre) and takes the closest point over them).  Opt-in (option wallDistCorrectWalls): the
    // default keeps the centre distance everywhere, which is what the oracle and the committed golden vectors use.
    static double distToTriangle(const double* a, const double* b, const double* c, const double* p)
    {
        // closest point on a triangle to p (Ericson, Real-Time Collision Detection 5.1.5), returned as a distance
        double ab[3], ac[3], ap[3];
        for (int k = 0; k < 3; k++) { ab[k] = b[k] - a[k]; ac[k] = c[k] - a[k]; ap[k] = p[k] - a[k]; }
        auto dot = [](const double* x, const double* y) { return x[0] * y[0] + x[1] * y[1] + x[2] * y[2]; };
        auto dist = [&](const double* q) { return std::sqrt((p[0] - q[0]) * (p[0] - q[0]) + (p[1] - q[1]) * (p[1] - q[1]) + (p[2] - q[2]) * (p[2] - q[2])); };
        const double d1 = dot(ab, ap), d2 = dot(ac, ap);
        if (d1 <= 0.0 && d2 <= 0.0) return dist(a);
        double bp[3];
        for (int k = 0; k < 3; k++) bp[k] = p[k] - b[k];
        const double d3 = dot(ab, bp), d4 = dot(ac, bp);
        if (d3 >= 0.0 && d4 <= d3) return dist(b);
        const double vc = d1 * d4 - d3 * d2;
        double q[3];
        if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0)
        {
            const double v = d1 / (d1 - d3);
            for (int k = 0; k < 3; k++) q[k] = a[k] + v * ab[k];
            return dist(q);
        }
        double cp[3];
        for (int k = 0; k < 3; k++) cp[k] = p[k] - c[k];
        const double d5 = dot(ab, cp), d6 = dot(ac, cp);
        if (d6 >= 0.0 && d5 <= d6) return dist(c);
        const double vb = d5 * d2 - d1 * d6;
        if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0)
        {
            const double w = d2 / (d2 - d6);
            for (int k = 0; k < 3; k++) q[k] = a[k] + w * ac[k];
            return dist(q);
        }
        const double va = d3 * d6 - d5 * d4;
        if (va <= 0.0 && (d4 - d3) >= 0.0 && (d5 - d6) >= 0.0)
        {
            const double w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
            for (int k = 0; k < 3; k++) q[k] = b[k] + w * (c[k] - b[k]);
            return dist(q);
        }
        const double den = 1.0 / (va + vb + vc), v = vb * den, w = vc * den;
        for (int k = 0; k < 3; k++) q[k] = a[k] + ab[k] * v + ac[k] * w;
        return dist(q);
    }
    double distToFace(int f, const double* p) const
    {
        const int n = fOff[f + 1] - fOff[f];
        const int32_t* l = &fLab[fOff[f]];
        const double* P = points.data();
        if (n == 3) return distToTriangle(&P[3 * l[0]], &P[3 * l[1]], &P[3 * l[2]], p);
        const double ctr[3] = {Cf[0][f], Cf[1][f], Cf[2][f]};
        double best = 1e300;
        for (int i = 0; i < n; i++) best = std::min(best, distToTriangle(&P[3 * l[i]], &P[3 * l[(i + 1) % n]], ctr, p));
        return best;
    }
    void correctWallDistance(const std::vector<uint8_t>* only = nullptr)
    {
        // wall faces around every wall point
        std::vector<std::vector<int>> pointWallFaces(nP);
        std::vector<uint8_t> wallPoint(nP, 0);
        for (int b = 0; b < nBF; b++)
        {
            if (patchGeom[bPatch[b]] != PG_WALL) continue;
            const int f = nIF + b;
            for (int q = fOff[f]; q < fOff[f + 1]; q++)
            {
                pointWallFaces[fLab[q]].push_back(f);
                wallPoint[fLab[q]] = 1;
            }
        }
        std::vector<double> corrected(nC, -1.0);
        auto consider = [&](int c, int f) {
            if (only && !(*only)[c]) return;
            const double p[3] = {C[0][c], C[1][c], C[2][c]};
            const double d = distToFace(f, p);
            corrected[c] = corrected[c] < 0.0 ? d : std::min(corrected[c], d);
        };
        // cells that own a wall face: that face and the wall faces sharing a point with it
        for (int b = 0; b < nBF; b++)
        {
            if (patchGeom[bPatch[b]] != PG_WALL) continue;
            const int f = nIF + b, c = own[f];
            for (int q = fOff[f]; q < fOff[f + 1]; q++)
                for (int g : pointWallFaces[fLab[q]]) consider(c, g);
        }
        // cells that only touch the wall with a point (or an edge): the wall faces around that point
        std::vector<uint8_t> faceCell(nC, 0);
        for (int c = 0; c < nC; c++) faceCell[c] = corrected[c] >= 0.0;
        for (int f = 0; f < nF; f++)
            for (int side = 0; side < (f < nIF ? 2 : 1); side++)
            {
                if (side == 1 && f < (int)cyc.size() && cyc[f] > 0) continue; // the points of a coupled face are the owner side's
                const int c = side == 0 ? own[f] : nei[f];
                if (faceCell[c]) continue;
                for (int q = fOff[f]; q < fOff[f + 1]; q++)
                    if (wallPoint[fLab[q]])
                        for (int g : pointWallFaces[fLab[q]]) consider(c, g);
            }
        for (int c = 0; c < nC; c++)
            if (corrected[c] >= 0.0) yWall[c] = corrected[c];
    }

    // frozen wall distance (meshWaveFrozen role, reference src/adjoint/DAMisc/meshWaveFrozen): distance
    // from the cell centre to the nearest wall-face centre, evaluated once
    // only != nullptr: wall distance of the flagged cells only (a rank of a decomposed run needs its own cells, not all of the global
    // mesh: at 8 ranks on a 16-core host the global query was 18 s of the set-up)
    void computeWallDistance(const std::vector<uint8_t>* only = nullptr)
    {
        yWall.assign(nC, 1e30);
        std::vector<int> wf;
        for (int b = 0; b < nBF; b++)
            if (patchGeom[bPatch[b]] == PG_WALL) wf.push_back(nIF + b);
        if (wf.empty()) return;
        // k-d tree over the wall-face centres (median splits, implicit layout), exact nearest-neighbour query
        // cyclic patches: the nearest wall face may be the periodic image of one (one layer of images on either side of every pair)
        const int nImg = 1 + 2 * (int)xforms.size();
        const int nw = (int)wf.size() * nImg;
        std::vector<double> pts((size_t)3 * nw);
        for (size_t i = 0; i < wf.size(); i++)
        {
            const double c0[3] = {Cf[0][wf[i]], Cf[1][wf[i]], Cf[2][wf[i]]};
            for (int k = 0; k < 3; k++) pts[3 * (nImg * i) + k] = c0[k];
            for (size_t x = 0; x < xforms.size(); x++)
            {
                xfPoint(xforms[x], false, c0, &pts[3 * (nImg * i + 1 + 2 * x)]);
                xfPoint(xforms[x], true, c0, &pts[3 * (nImg * i + 2 + 2 * x)]);
            }
        }
        std::vector<int> idx(nw), axisOf(nw, 0);
        for (int i = 0; i < nw; i++) idx[i] = i;
        struct Range { int lo, hi, depth; };
        {
            std::vector<Range> st{{0, nw, 0}};
            while (!st.empty())
            {
                Range r = st.back();
                st.pop_back();
                if (r.hi - r.lo <= 1) continue;
                // split along the widest axis of the range
                double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
                for (int i = r.lo; i < r.hi; i++)
                    for (int k = 0; k < 3; k++)
                    {
                        mn[k] = std::min(mn[k], pts[3 * (size_t)idx[i] + k]);
                        mx[k] = std::max(mx[k], pts[3 * (size_t)idx[i] + k]);
                    }
                int ax = 0;
                for (int k = 1; k < 3; k++)
                    if (mx[k] - mn[k] > mx[ax] - mn[ax]) ax = k;
                const int mid = (r.lo + r.hi) / 2;
                std::nth_element(idx.begin() + r.lo, idx.begin() + mid, idx.begin() + r.hi,
                                 [&](int a, int b) { return pts[3 * (size_t)a + ax] < pts[3 * (size_t)b + ax]; });
                axisOf[mid] = ax;
                st.push_back({r.lo, mid, r.depth + 1});
                st.push_back({mid + 1, r.hi, r.depth + 1});
            }
        }
        // the queries are independent: host threads (the set-up of a 10M-cell mesh is otherwise minutes of one core)
        detail::parallelFor(nC, detail::hostThreads(), [&](int, int cb, int ce) {
        std::vector<Range> stack;
        for (int c = cb; c < ce; c++)
        {
            if (only && !(*only)[c]) continue;
            const double q[3] = {C[0][c], C[1][c], C[2][c]};
            double best = 1e300;
            stack.assign(1, Range{0, nw, 0});
            while (!stack.empty())
            {
                Range r = stack.back();
                stack.pop_back();
                if (r.hi <= r.lo) continue;
                const int mid = (r.lo + r.hi) / 2;
                const double* pm = &pts[3 * (size_t)idx[mid]];
                const double d2 = (pm[0] - q[0]) * (pm[0] - q[0]) + (pm[1] - q[1]) * (pm[1] - q[1]) + (pm[2] - q[2]) * (pm[2] - q[2]);
                best = std::min(best, d2);
                if (r.hi - r.lo == 1) continue;
                const int ax = axisOf[mid];
                const double diff = q[ax] - pm[ax];
                const Range nearR = diff < 0 ? Range{r.lo, mid, 0} : Range{mid + 1, r.hi, 0};
                const Range farR = diff < 0 ? Range{mid + 1, r.hi, 0} : Range{r.lo, mid, 0};
                if (diff * diff < best) stack.push_back(farR); // visited after the near side (stack order)
                stack.push_back(nearR);
            }
            yWall[c] = std::sqrt(best);
        }
        });
    }
    // Mesh quality report of DACheckMesh::run (reference src/adjoint/DACheckMesh/DACheckMesh.C:45-79, DACheckGeometry.C:256-478;
    // OpenFOAM primitiveMeshCheck semantics): the checks that count as failures there - open boundary, open cells /
    // aspect ratio above the threshold, zero face areas, non-positive cell volumes, faces more than 90 degrees non-orthogonal,
    // more than maxIncorrectlyOrientedFaces negative face pyramids, skewness above the threshold.  Severe non-orthogonality
    // (> maxNonOrth) is reported but, as in OpenFOAM, is not a failure.
    struct Quality
    {
        double maxNonOrth = 0, avgNonOrth = 0, maxSkewness = 0, maxAspectRatio = 0, minVolume = 0, minFaceArea = 0, maxOpenness = 0;
        int nSevereNonOrth = 0, nErrorNonOrth = 0, nNegativePyramids = 0, nFailedChecks = 0;
    };
    Quality checkMesh(double maxNonOrthDeg, double maxSkew, double maxAspect, int maxBadPyramids) const
    {
        const double SMALL = 1e-15, VSMALL = 1e-300, ROOTVSMALL = 1e-150, PI = 3.14159265358979323846;
        Quality q;
        q.minVolume = 1e300;
        q.minFaceArea = 1e300;
        // closed boundary
        double sb[3] = {0, 0, 0}, smb = 0;
        for (int f = nIF; f < nF; f++)
        {
            if (patchGeomOfFace(f) == PG_PROCESSOR) continue;
            for (int k = 0; k < 3; k++) sb[k] += Sf[k][f];
            smb += magSf[f];
        }
        const bool openBoundary = std::sqrt(sb[0] * sb[0] + sb[1] * sb[1] + sb[2] * sb[2]) > 1e-6 * smb;
        // closed cells + aspect ratio
        std::vector<double> sumC((size_t)3 * nC, 0.0), sumM((size_t)3 * nC, 0.0);
        for (int f = 0; f < nF; f++)
        {
            q.minFaceArea = std::min(q.minFaceArea, magSf[f]);
            const int o = own[f];
            if (o < nC)
                for (int k = 0; k < 3; k++) { sumC[(size_t)3 * o + k] += Sf[k][f]; sumM[(size_t)3 * o + k] += std::fabs(Sf[k][f]); }
            if (f < nIF && nei[f] < nC)
                for (int k = 0; k < 3; k++) { sumC[(size_t)3 * nei[f] + k] -= Sf[k][f]; sumM[(size_t)3 * nei[f] + k] += std::fabs(Sf[k][f]); }
        }
        int nOpen = 0, nAspect = 0;
        for (int c = 0; c < nC; c++)
        {
            double open = 0, mn = 1e300, mx = 0, sm = 0;
            for (int k = 0; k < 3; k++)
            {
                open = std::max(open, std::fabs(sumC[(size_t)3 * c + k]) / (sumM[(size_t)3 * c + k] + ROOTVSMALL));
                mn = std::min(mn, sumM[(size_t)3 * c + k]);
                mx = std::max(mx, sumM[(size_t)3 * c + k]);
                sm += sumM[(size_t)3 * c + k];
            }
            double ar = mx / (mn + ROOTVSMALL);
            ar = std::max(ar, sm / 6.0 / std::pow(std::max(ROOTVSMALL, V[c]), 2.0 / 3.0));
            q.maxOpenness = std::max(q.maxOpenness, open);
            q.maxAspectRatio = std::max(q.maxAspectRatio, ar);
            q.minVolume = std::min(q.minVolume, V[c]);
            if (open > 1e-6) nOpen++;
            if (ar > maxAspect) nAspect++;
        }
        // orthogonality of internal faces
        const double severe = std::cos(maxNonOrthDeg * PI / 180.0);
        double sumOrtho = 0;
        double minOrtho = 1.0;
        for (int f = 0; f < nIF; f++)
        {
            const int o = own[f], n = nei[f];
            double d[3], dd = 0, ds = 0;
            for (int k = 0; k < 3; k++) { d[k] = C[k][n] - C[k][o]; dd += d[k] * d[k]; ds += d[k] * Sf[k][f]; }
            const double ortho = ds / (std::sqrt(dd) * magSf[f] + VSMALL);
            if (ortho < severe) { if (ortho > SMALL) q.nSevereNonOrth++; else q.nErrorNonOrth++; }
            minOrtho = std::min(minOrtho, ortho);
            sumOrtho += ortho;
        }
        if (nIF > 0)
        {
            q.maxNonOrth = std::acos(std::max(-1.0, std::min(1.0, minOrtho))) * 180.0 / PI;
            q.avgNonOrth = std::acos(std::max(-1.0, std::min(1.0, sumOrtho / nIF))) * 180.0 / PI;
        }
        // face pyramids and skewness
        for (int f = 0; f < nF; f++)
        {
            const int o = own[f];
            double cpf[3], pyr = 0;
            for (int k = 0; k < 3; k++) { cpf[k] = Cf[k][f] - C[k][o]; pyr += Sf[k][f] * cpf[k]; }
            bool bad = pyr / 3.0 < -SMALL;
            double d[3], sd = 0, sc = 0, dm = 0;
            if (f < nIF)
            {
                const int n = nei[f];
                double pn = 0;
                for (int k = 0; k < 3; k++) pn += Sf[k][f] * (C[k][n] - Cf[k][f]);
                bad = bad || pn / 3.0 < -SMALL;
                for (int k = 0; k < 3; k++) d[k] = C[k][n] - C[k][o];
            }
            else
            {
                double nc = 0;
                for (int k = 0; k < 3; k++) nc += Sf[k][f] / magSf[f] * cpf[k];
                for (int k = 0; k < 3; k++) d[k] = Sf[k][f] / magSf[f] * nc;
            }
            if (bad) q.nNegativePyramids++;
            for (int k = 0; k < 3; k++) { sd += Sf[k][f] * d[k]; sc += Sf[k][f] * cpf[k]; dm += d[k] * d[k]; }
            double sv[3], svm = 0;
            for (int k = 0; k < 3; k++) { sv[k] = cpf[k] - sc / (sd + ROOTVSMALL) * d[k]; svm += sv[k] * sv[k]; }
            svm = std::sqrt(svm);
            double fd = (f < nIF ? 0.2 : 0.4) * std::sqrt(dm) + ROOTVSMALL;
            for (int i = fOff[f]; i < fOff[f + 1]; i++)
            {
                double t = 0;
                for (int k = 0; k < 3; k++) t += sv[k] / (svm + ROOTVSMALL) * (points[(size_t)3 * fLab[i] + k] - Cf[k][f]);
                fd = std::max(fd, std::fabs(t));
            }
            q.maxSkewness = std::max(q.maxSkewness, svm / fd);
        }
        q.nFailedChecks = (openBoundary ? 1 : 0) + (nOpen > 0 ? 1 : 0) + (nAspect > 0 ? 1 : 0) + (q.minFaceArea < VSMALL ? 1 : 0)
            + (q.minVolume < VSMALL ? 1 : 0) + (q.nErrorNonOrth > 0 ? 1 : 0) + (q.nNegativePyramids > maxBadPyramids ? 1 : 0)
            + (q.maxSkewness > maxSkew ? 1 : 0);
        return q;
    }
    int patchGeomOfFace(int f) const { return patchGeom[bPatch[f - nIF]]; }
};

} // namespace dab
