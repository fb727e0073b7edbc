// forceCouplingOutput (reference DAOutputForceCoupling.C:19-215): the wall force of every listed face split equally over the
// face's points, one 3-vector per (patch, point).  Every kernel gathers over topology tables built once on the host
// (Solver::couplingTables); no atomics, sums in increasing face order.
#pragma once
#include "rev_kernels.hpp"
#include "comp_rev_kernels.hpp"

namespace dab
{

// topology of one output: the listed faces (boundary face indices, patches sorted by name, faces in increasing order), the output
// slot of each of their points (CSR parallel to fOff / fLab), and the listed faces around each slot (CSR, increasing face order)
struct CouplingView
{
    int nFaces, nNodes;
    const int32_t *face, *fsOff, *fsLab, *nfOff, *nfLab;
};

// F_f = Sf (p_b - pRef) + Sf & devRhoReff_b of every listed face -> faceF[3 * i + j]
template <bool COMP>
struct CouplingFaceFwd
{
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    ForceSpec fs;
    CouplingView cv;
    double* faceF;
    DAB_HD void operator()(int i) const
    {
        const int f = m.nIF + cv.face[i];
        double fv[3];
        if constexpr (COMP) cForceFace(m, q, s, r, fs, f, m.own[f], 0.0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, fv);
        else forceFace(m, q, s, r, fs, f, m.own[f], 0.0, nullptr, nullptr, nullptr, nullptr, nullptr, fv);
        for (int j = 0; j < 3; j++) faceF[3 * i + j] = fv[j];
    }
};

// out[3 * n + j] = sum over the faces of slot n, in increasing face order, of F_f,j / nPoints_f
struct CouplingNodeSum
{
    CouplingView cv;
    const double* faceF;
    double* out;
    DAB_HD void operator()(int n) const
    {
        double a[3] = {0.0, 0.0, 0.0};
        for (int q = cv.nfOff[n]; q < cv.nfOff[n + 1]; q++)
        {
            const int i = cv.nfLab[q];
            const double np = (double)(cv.fsOff[i + 1] - cv.fsOff[i]);
            for (int j = 0; j < 3; j++) a[j] += faceF[3 * i + j] / np;
        }
        for (int j = 0; j < 3; j++) out[3 * n + j] = a[j];
    }
};

// the reverse of the point split: d_f = sum over the points of f of seed[slot] / nPoints_f -> faceDir[3 * b + j] (by boundary face)
struct CouplingFaceSeed
{
    CouplingView cv;
    const double* seed;
    double* faceDir;
    DAB_HD void operator()(int i) const
    {
        double d[3] = {0.0, 0.0, 0.0};
        for (int q = cv.fsOff[i]; q < cv.fsOff[i + 1]; q++)
            for (int j = 0; j < 3; j++) d[j] += seed[3 * cv.fsLab[q] + j];
        const double np = (double)(cv.fsOff[i + 1] - cv.fsOff[i]);
        for (int j = 0; j < 3; j++) faceDir[3 * cv.face[i] + j] = d[j] / np;
    }
};

} // namespace dab
