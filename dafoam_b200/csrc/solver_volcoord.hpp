// Solver::volCoordProduct -- [dR/dx_v]^T psi and dF/dx_v for the `volCoord` input (mesh point coordinates), and
// updateMesh (reference DASolvers::updateOFMesh).  See geom_kernels.hpp for the method (coloured central differences
// over the points, geometry and R(W) re-evaluated on the device).
#pragma once

namespace dab
{

// geometry arrays of the (possibly moved) host mesh -> the existing device buffers
inline void Solver::uploadGeometry()
{
    auto put = [&](double* d, const std::vector<double>& h) { be.h2d(d, h.data(), h.size() * sizeof(double)); };
    for (int k = 0; k < 3; k++)
    {
        put(dS[k].p, hm.Sf[k]);
        put(dK[k].p, hm.corr[k]);
        put(dCf[k].p, hm.Cf[k]);
        put(dC.p + (size_t)k * hm.nCtot, hm.C[k]);
    }
    put(dMagSf.p, hm.magSf);
    put(dW.p, hm.w);
    put(dDelta.p, hm.delta);
    put(dV.p, hm.V);
    updateFaceOffsets();
    updateMrfFlux();
    recorded = false;
    kry.pcValid = false;
}

// the device geometry buffers -> the host mesh (a partitioned mesh has no global host mesh to recompute them from)
inline void Solver::downloadGeometry()
{
    auto get = [&](std::vector<double>& h, const double* d) { be.d2h(h.data(), d, h.size() * sizeof(double)); };
    for (int k = 0; k < 3; k++)
    {
        get(hm.Sf[k], dS[k].p);
        get(hm.corr[k], dK[k].p);
        get(hm.Cf[k], dCf[k].p);
        get(hm.C[k], dC.p + (size_t)k * hm.nCtot);
    }
    get(hm.magSf, dMagSf.p);
    get(hm.w, dW.p);
    get(hm.delta, dDelta.p);
    get(hm.V, dV.p);
}

// geometry of the local mesh from the points in volc.dPts, on the device: faces (the neighbour-side copies of coupled faces in the
// neighbour's frame), owned cells, then -- on a partitioned mesh -- the ghost cells' centres (positions) and volumes from their
// owners, then the face quantities that need both cells (weights, deltas, non-orthogonal corrections)
inline void Solver::deviceGeometry()
{
    VolCoord& Vc = volc;
    if (!Vc.topoReady)
    {
        Vc.dFOff.upload(be, hm.fOff);
        Vc.dFLab.upload(be, hm.fLab);
        if (hm.hasCyclic()) Vc.dFaceXf.upload(be, part.faceXf);
        Vc.topoReady = true;
    }
    const size_t nT = hm.nCtot;
    GeomView gv;
    gv.nC = hm.nC; gv.nF = hm.nF; gv.nIF = hm.nIF; gv.maxCF = hm.maxCF;
    gv.fOff = Vc.dFOff.p; gv.fLab = Vc.dFLab.p; gv.own = dOwn.p; gv.nei = dNei.p; gv.cellFaces = dCellFaces.p;
    gv.pts = Vc.dPts.p;
    gv.Sx = dS[0].p; gv.Sy = dS[1].p; gv.Sz = dS[2].p; gv.magSf = dMagSf.p; gv.w = dW.p; gv.delta = dDelta.p;
    gv.kx = dK[0].p; gv.ky = dK[1].p; gv.kz = dK[2].p; gv.Cfx = dCf[0].p; gv.Cfy = dCf[1].p; gv.Cfz = dCf[2].p;
    gv.Cx = dC.p; gv.Cy = dC.p + nT; gv.Cz = dC.p + 2 * nT; gv.V = dV.p;
    gv.faceXf = Vc.dFaceXf.n ? Vc.dFaceXf.p : nullptr;
    gv.Rtab = halo.dRtab.p;
    gv.Ttab = halo.dTtab.p;
    be.launch(hm.nF, GeomFaceK{gv});
    be.launch(hm.nC, GeomCellK{gv});
    if (ghosted())
    {
        HaloItem centres{dC.p, 3, 1, (int)nT};
        centres.position = true;
        halo.exchangeCells({centres, {dV.p, 1, 1, (int)nT}});
    }
    be.launch(hm.nF, GeomDerivedK{gv});
    updateFaceOffsets();
}

// new point coordinates (the wall distance stays frozen: meshWaveFrozen).  Every rank passes the same full point list.
inline void Solver::updateMesh(const double* pts)
{
    const std::vector<double> old(hm.points);
    std::copy(pts, pts + hm.points.size(), hm.points.begin());
    if (!ghosted())
        hm.computeGeometry();
    else
    {
        try
        {
            hm.checkCyclicPairs();
        }
        catch (...)
        {
            hm.points = old;
            throw;
        }
        if (volc.dPts.n != hm.points.size()) volc.dPts.alloc(be, hm.points.size(), false);
        be.h2d(volc.dPts.p, hm.points.data(), hm.points.size() * sizeof(double));
        deviceGeometry();
        downloadGeometry();
    }
    uploadGeometry();
    fvSourceDirty = fvSpec.nDisk > 0;
    if (volc.ready) be.h2d(volc.dPts0.p, hm.points.data(), hm.points.size() * sizeof(double));
}

inline void Solver::volCoordSetup()
{
    VolCoord& Vc = volc;
    if (Vc.ready) return;
    // the colouring, the point steps and the home -> point slots come from the global mesh (periodic adjacency across coupled
    // pairs); a partitioned solver re-reads its topology for that and drops it again
    HostMesh gm;
    const HostMesh* G = &hm;
    if (ghosted())
    {
        gm.read(caseDirectory);
        bool same = gm.points.size() == hm.points.size() && gm.nC == part.nGlobalCells;
        for (int f = 0; f < hm.nF && same; f++)
        {
            const int q = part.faceGlobal[f];
            same = q < gm.nF && gm.fOff[q + 1] - gm.fOff[q] == hm.fOff[f + 1] - hm.fOff[f]
                   && std::equal(hm.fLab.begin() + hm.fOff[f], hm.fLab.begin() + hm.fOff[f + 1], gm.fLab.begin() + gm.fOff[q]);
        }
        if (!same) throw Error("volCoord: the polyMesh in " + caseDirectory + " no longer matches the solver's mesh");
        gm.points = hm.points;
        G = &gm;
    }
    const HostMesh& g = *G;
    const int nC = g.nC, nF = g.nF, nP = g.nP;
    // cells around each point
    std::vector<int> pcOff(nP + 1, 0), pcList;
    {
        std::vector<std::pair<int, int>> pr;
        pr.reserve((size_t)g.fLab.size() * 2);
        for (int f = 0; f < nF; f++)
            for (int q = g.fOff[f]; q < g.fOff[f + 1]; q++)
            {
                pr.emplace_back(g.fLab[q], g.own[f]);
                if (f < g.nIF) pr.emplace_back(g.fLab[q], g.nei[f]);
            }
        std::sort(pr.begin(), pr.end());
        pr.erase(std::unique(pr.begin(), pr.end()), pr.end());
        for (auto& x : pr) pcOff[x.first + 1]++;
        for (int p = 0; p < nP; p++) pcOff[p + 1] += pcOff[p];
        pcList.resize(pr.size());
        for (size_t i = 0; i < pr.size(); i++) pcList[i] = pr[i].second;
    }
    // home cell of every point: the surrounding cell that carries the fewest points so far
    std::vector<int> homed(nC, 0), homeOf(nP, -1), slotOf(nP, 0);
    for (int p = 0; p < nP; p++)
    {
        int best = -1;
        for (int i = pcOff[p]; i < pcOff[p + 1]; i++)
            if (best < 0 || homed[pcList[i]] < homed[best]) best = pcList[i];
        if (best < 0) continue; // unused point
        homeOf[p] = best;
        slotOf[p] = homed[best]++;
    }
    Vc.maxSlots = 1;
    for (int c = 0; c < nC; c++) Vc.maxSlots = std::max(Vc.maxSlots, homed[c]);
    std::vector<int32_t> slotPoint((size_t)nC * Vc.maxSlots, -1);
    for (int p = 0; p < nP; p++)
        if (homeOf[p] >= 0) slotPoint[(size_t)homeOf[p] * Vc.maxSlots + slotOf[p]] = p;
    // colour the home cells: two homes of one colour are more than 2*radius cells apart (disjoint footprints); the merged coupled
    // faces of the global mesh are internal faces, so the distance is the periodic one
    detail::CellGraph CG;
    CG.build(g);
    std::vector<int> colour(nC, -1);
    int nCol = 0;
    {
        std::vector<int> mark, ball;
        for (int c = 0; c < nC; c++)
        {
            if (homed[c] == 0) continue;
            CG.ball(&c, 1, 2 * Vc.radius, ball);
            if ((int)mark.size() < nCol + 1) mark.resize(nCol + 1, -1);
            for (int x : ball)
                if (colour[x] >= 0) mark[colour[x]] = c;
            int k = 0;
            while (k < nCol && mark[k] == c) k++;
            if (k == nCol)
            {
                nCol++;
                mark.push_back(-1);
            }
            colour[c] = k;
        }
    }
    Vc.nColours = nCol;
    // this rank's seeds per colour: local cells (owned and ghost) whose global cell is a home, with that global id
    const int nT = hm.nCtot;
    auto globalOf = [&](int c) { return ghosted() ? (int)part.cellGlobal[c] : c; };
    Vc.homeStart.assign(nCol + 1, 0);
    for (int c = 0; c < nT; c++)
        if (colour[globalOf(c)] >= 0) Vc.homeStart[colour[globalOf(c)] + 1]++;
    for (int k = 0; k < nCol; k++) Vc.homeStart[k + 1] += Vc.homeStart[k];
    std::vector<int32_t> homes(Vc.homeStart[nCol]), homeIds(Vc.homeStart[nCol]);
    {
        std::vector<int> pos(Vc.homeStart.begin(), Vc.homeStart.end() - 1);
        for (int c = 0; c < nT; c++)
            if (colour[globalOf(c)] >= 0)
            {
                const int i = pos[colour[globalOf(c)]]++;
                homes[i] = c;
                homeIds[i] = globalOf(c);
            }
    }
    // point lists per (colour, slot), over the global homes: the same on every rank
    std::vector<std::vector<int>> homesOfColour(nCol);
    for (int c = 0; c < nC; c++)
        if (colour[c] >= 0) homesOfColour[colour[c]].push_back(c);
    Vc.listStart.assign((size_t)nCol * Vc.maxSlots + 1, 0);
    std::vector<int32_t> lists;
    for (int k = 0; k < nCol; k++)
        for (int s = 0; s < Vc.maxSlots; s++)
        {
            for (int h : homesOfColour[k])
            {
                const int p = slotPoint[(size_t)h * Vc.maxSlots + s];
                if (p >= 0) lists.push_back(p);
            }
            Vc.listStart[(size_t)k * Vc.maxSlots + s + 1] = (int)lists.size();
        }
    // step per point: relStep * shortest edge at the point
    std::vector<double> eps(nP, 0.0), minEdge(nP, 1e300);
    for (int f = 0; f < nF; f++)
    {
        const int n = g.fOff[f + 1] - g.fOff[f];
        for (int i = 0; i < n; i++)
        {
            const int a = g.fLab[g.fOff[f] + i], b = g.fLab[g.fOff[f] + (i + 1) % n];
            double d2 = 0.0;
            for (int k = 0; k < 3; k++) d2 += (g.points[3 * a + k] - g.points[3 * b + k]) * (g.points[3 * a + k] - g.points[3 * b + k]);
            const double d = std::sqrt(d2);
            minEdge[a] = std::min(minEdge[a], d);
            minEdge[b] = std::min(minEdge[b], d);
        }
    }
    for (int p = 0; p < nP; p++) eps[p] = minEdge[p] < 1e299 ? Vc.relStep * minEdge[p] : 0.0;
    Vc.dSlotPoint.upload(be, slotPoint);
    Vc.dHomes.upload(be, homes);
    Vc.dHomeIds.upload(be, homeIds);
    Vc.dLists.upload(be, lists);
    Vc.dEps.upload(be, eps);
    Vc.dPts.upload(be, hm.points);
    Vc.dPts0.upload(be, hm.points);
    Vc.dLabelA.alloc(be, nT);
    Vc.dLabelB.alloc(be, nT);
    Vc.dR2.alloc(be, nDof());
    Vc.dOut.alloc(be, (size_t)3 * nP);
    Vc.dF1.alloc(be, hm.nBF + 1);
    Vc.dF2.alloc(be, hm.nBF + 1);
    Vc.ready = true;
    Vc.nEval = 0;
    for (size_t i = 0; i + 1 < Vc.listStart.size(); i++)
        if (Vc.listStart[i + 1] > Vc.listStart[i]) Vc.nEval += 6;
    if (printInfo)
        fprintf(stderr, "[dab200] volCoord: %d colours x %d slots, %d residual evaluations per product\n", Vc.nColours, Vc.maxSlots, Vc.nEval);
}

// out[3*nP] = [dR/dx_v]^T psi (fsv empty) or seed * dF/dx_v of the face groups fsv
inline void Solver::volCoordProduct(const double* psi, const std::vector<ForceSpec>& fsv, double seed, double* out)
{
    volCoordSetup();
    VolCoord& Vc = volc;
    const int nC = hm.nC, nT = hm.nCtot, nP = hm.nP;
    auto geometry = [&]() {
        deviceGeometry();
        if (fvSpec.nDisk > 0) be.launch(nC, FvSourceK{fvSpec, mv.Cx, mv.Cy, mv.Cz, nC, dFvS.p}); // the source follows the cell centres
        updateMrfFlux();                                                                           // and the relative fluxes the faces
    };
    if (psi) be.h2d(dX.p, psi, (size_t)nDof() * sizeof(double));
    be.d2d(Vc.dPts.p, Vc.dPts0.p, (size_t)3 * nP * sizeof(double));
    be.zero(Vc.dOut.p, (size_t)3 * nP * sizeof(double));
    const int ns = nCellStates(), offPhi = ns * nC;
    const bool function = !fsv.empty();
    auto evaluate = [&](double* Rdev, double* Fdev) {
        geometry();
        if (function)
        {
            if (par.comp)
            {
                launchNF<cFwdA>(hm.nCtot, mv, par, sv, rv);
                for (const ForceSpec& fs : fsv) be.launch(hm.nBF, cForceFwd{mv, par, sv, rv, fs, Fdev});
            }
            else
            {
                launchNF<FwdA>(hm.nCtot, mv, par, sv, rv);
                for (const ForceSpec& fs : fsv) be.launch(hm.nBF, ForceFwd{mv, par, sv, rv, fs, Fdev});
            }
        }
        else
            forward(0, Rdev, ghosted());
    };
    for (int col = 0; col < Vc.nColours; col++)
    {
        // footprint labels of this colour's homes (across ranks and coupled pairs: the ghost labels are refreshed after every sweep)
        be.launch(nT, LabelInit{Vc.dLabelA.p});
        be.launch(Vc.homeStart[col + 1] - Vc.homeStart[col], LabelSeed{Vc.dLabelA.p, Vc.dHomes.p + Vc.homeStart[col], Vc.dHomeIds.p + Vc.homeStart[col]});
        double *la = Vc.dLabelA.p, *lb = Vc.dLabelB.p;
        for (int r = 0; r < Vc.radius; r++)
        {
            be.launch(nC, LabelSweep{la, lb, mv.cellNbr, nC, hm.maxCF});
            if (ghosted()) halo.exchangeCells({{lb, 1, 1, nT}});
            std::swap(la, lb);
        }
        for (int slot = 0; slot < Vc.maxSlots; slot++)
        {
            const int l0 = Vc.listStart[(size_t)col * Vc.maxSlots + slot], l1 = Vc.listStart[(size_t)col * Vc.maxSlots + slot + 1];
            if (l1 == l0) continue;
            const int32_t* list = Vc.dLists.p + l0;
            for (int k = 0; k < 3; k++)
            {
                be.launch(l1 - l0, PointMove{Vc.dPts.p, Vc.dPts0.p, Vc.dEps.p, list, k, 1.0});
                evaluate(dR.p, Vc.dF1.p);
                be.launch(l1 - l0, PointMove{Vc.dPts.p, Vc.dPts0.p, Vc.dEps.p, list, k, -1.0});
                evaluate(Vc.dR2.p, Vc.dF2.p);
                be.launch(l1 - l0, PointMove{Vc.dPts.p, Vc.dPts0.p, Vc.dEps.p, list, k, 0.0});
                if (function)
                    be.launch(hm.nBF, VolCoordAccumF{mv, Vc.dF1.p, Vc.dF2.p, la, Vc.dSlotPoint.p, Vc.maxSlots, slot, k, Vc.dEps.p, seed, Vc.dOut.p});
                else
                    be.launch(nC, VolCoordAccumR{mv, ns, offPhi, dR.p, Vc.dR2.p, dX.p, la, Vc.dSlotPoint.p, Vc.maxSlots, slot, k,
                                                 Vc.dEps.p, Vc.dOut.p});
            }
        }
    }
    be.d2h(out, Vc.dOut.p, (size_t)3 * nP * sizeof(double));
    uploadGeometry(); // the unperturbed geometry exactly as the host computed it
    if (fvSpec.nDisk > 0) updateFvSource();
}

} // namespace dab
