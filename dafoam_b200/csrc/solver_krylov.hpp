// Solver::calcPC / applyPC / solveLinearEqn: preconditioner assembly (coloured finite differences of the
// first-order residual, reference DAPartDeriv.C:350-474 + DASolver.C:948-1089), ILU(0), and the
// right-preconditioned restarted GMRES that replaces KSPSolve (reference DALinearEqn.C:341-437).
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdio>

#include <memory>
#include <thread>

namespace dab
{

namespace detail
{
// breadth-first ball over the cell graph with a stamp array (no clearing between calls)
struct CellGraph
{
    int nC;
    std::vector<int> off, adj, stamp, queue;
    int tick = 0;
    // alias != nullptr: ghost cell g (>= nC) stands for the owned cell (*alias)[g - nC] (-1: a cell of another rank) -- the periodic
    // images of a rank's own cells; the graph then holds the true (periodic) adjacency instead of stopping at the coupled patches
    void build(const HostMesh& m, const std::vector<int>* alias = nullptr)
    {
        nC = m.nC;
        auto cellOf = [&](int c) { return c < nC ? c : (alias ? (*alias)[c - nC] : -1); };
        off.assign(nC + 1, 0);
        for (int f = 0; f < m.nIF; f++)
        {
            const int a = cellOf(m.own[f]), b = cellOf(m.nei[f]);
            if (a < 0 || b < 0) continue; // cut face: the other cell is a ghost (block-Jacobi over ranks)
            if (alias && m.own[f] >= nC) continue; // the second local copy of a coupled face
            off[a + 1]++;
            off[b + 1]++;
        }
        for (int c = 0; c < nC; c++) off[c + 1] += off[c];
        adj.resize(off[nC]);
        std::vector<int> pos(off.begin(), off.end() - 1);
        for (int f = 0; f < m.nIF; f++)
        {
            const int a = cellOf(m.own[f]), b = cellOf(m.nei[f]);
            if (a < 0 || b < 0) continue;
            if (alias && m.own[f] >= nC) continue;
            adj[pos[a]++] = b;
            adj[pos[b]++] = a;
        }
        stamp.assign(nC, 0);
    }
    // scratch of one traversal stream (one per host thread in the parallel pattern build)
    struct Scratch
    {
        std::vector<int> stamp;
        int tick = 0;
    };
    void ball(const int* seeds, int nSeeds, int radius, std::vector<int>& out) { ballWith(seeds, nSeeds, radius, out, stamp, tick); }
    void ball(const int* seeds, int nSeeds, int radius, std::vector<int>& out, Scratch& sc) const
    {
        if ((int)sc.stamp.size() != nC) sc.stamp.assign(nC, 0);
        ballWith(seeds, nSeeds, radius, out, sc.stamp, sc.tick);
    }
    // cells within `radius` hops of the seeds (seeds included), appended to out (cleared first)
    // levelEnd != nullptr: (*levelEnd)[k] = number of cells within k hops (the list is in breadth-first order), k = 0..radius
    void ball(const int* seeds, int nSeeds, int radius, std::vector<int>& out, Scratch& sc, std::vector<int>* levelEnd) const
    {
        if ((int)sc.stamp.size() != nC) sc.stamp.assign(nC, 0);
        ballWith(seeds, nSeeds, radius, out, sc.stamp, sc.tick, levelEnd);
    }
    void ballWith(const int* seeds, int nSeeds, int radius, std::vector<int>& out, std::vector<int>& stamp, int& tick,
                  std::vector<int>* levelEnd = nullptr) const
    {
        if (levelEnd) levelEnd->clear();
        out.clear();
        tick++;
        for (int i = 0; i < nSeeds; i++)
            if (stamp[seeds[i]] != tick)
            {
                stamp[seeds[i]] = tick;
                out.push_back(seeds[i]);
            }
        size_t lo = 0;
        if (levelEnd) levelEnd->push_back((int)out.size());
        for (int r = 0; r < radius; r++)
        {
            const size_t hi = out.size();
            for (size_t q = lo; q < hi; q++)
            {
                const int c = out[q];
                for (int e = off[c]; e < off[c + 1]; e++)
                {
                    const int x = adj[e];
                    if (stamp[x] != tick)
                    {
                        stamp[x] = tick;
                        out.push_back(x);
                    }
                }
            }
            lo = hi;
            if (levelEnd) levelEnd->push_back((int)out.size());
        }
    }
};

// greedy colouring: item i conflicts with the items listed by neighbours(i, out)
template <class NbrFn>
int greedyColour(int n, NbrFn nbr, std::vector<int>& colour)
{
    colour.assign(n, -1);
    std::vector<int> mark, tmp;
    int nCol = 0;
    for (int i = 0; i < n; i++)
    {
        nbr(i, tmp);
        if ((int)mark.size() < nCol + 1) mark.resize(nCol + 1, -1);
        for (int x : tmp)
            if (colour[x] >= 0) mark[colour[x]] = i;
        int k = 0;
        while (k < nCol && mark[k] == i) k++;
        if (k == nCol)
        {
            nCol++;
            mark.resize(nCol + 1, -1);
        }
        colour[i] = k;
    }
    return nCol;
}
} // namespace detail

inline void Solver::pcSymbolic()
{
    using detail::CellGraph;
    Krylov& K = kry;
    const int nC = hm.nC, nF = hm.nF, nIF = hm.nIF;
    const int ns = nCellStates();
    const int offPhi = ns * nC;
    K.n = nDof();
    auto tPrev = std::chrono::steady_clock::now();
    auto lap = [&](const char* what) {
        const auto now = std::chrono::steady_clock::now();
        if (printInfo) fprintf(stderr, "[dab200] pcSymbolic %-28s %.3f s\n", what, std::chrono::duration<double>(now - tPrev).count());
        tPrev = now;
    };
    CellGraph G;
    G.build(hm);
    lap("cell graph");
    // connectivity levels of the pattern.  Row = a state, columns = the residuals that see it.
    //   lvCell[s][r]  cell residual r (0 URes, 1 pRes, 2 nuTildaRes) of the cells within that many levels of the state's cell, s = 0 U, 1 p, 2 nuTilda
    //   lvPhiRes[s]   phiRes of the faces of the cells within that many levels of the state's cell
    //   lvOfPhi[r]    cell residual r of the cells within that many levels of the two cells of a phi state's face
    //   phiPhi        a phi state is seen by phiRes of the faces of its two cells (0: of its own face only)
    const bool stateInfo = pcPattern == "stateInfo" && !par.comp;
    int lvCell[3][3], lvPhiRes[3], lvOfPhi[3], phiPhi = 0;
    if (stateInfo)
    {
        // URes {U,p,nut,phi | U,p,nut | U}; pRes {U,p,nut,phi | U,p,nut,phi | U,p,nut | U} capped at 2; phiRes {U,p,nut,phi | U,p,nut | U} capped
        // at 1; nuTildaRes {U,nuTilda,phi | U,nuTilda | nuTilda}  (nut -> nuTilda: DASpalartAllmaras::correctStateResidualModelCon)
        const int cell[3][3] = {{2, 2, 1}, {1, 2, -1}, {1, 2, 2}}; // [state U,p,nt][residual U,p,nt]
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) lvCell[a][b] = std::min(cell[a][b], pcConLevel);
        for (int a = 0; a < 3; a++) lvPhiRes[a] = 1;
        lvOfPhi[0] = 0; lvOfPhi[1] = 1; lvOfPhi[2] = 0;
        phiPhi = 1;
    }
    else
    {
        for (int a = 0; a < 3; a++)
        {
            for (int b = 0; b < 3; b++) lvCell[a][b] = pcConLevel;
            lvPhiRes[a] = 0;
            lvOfPhi[a] = 0;
        }
        // (measured on the host build, 18k cells: adding the flux couplings of the reference's table to the uniform pattern -- phiRes one
        // level away, pRes-phi one level away, phiRes-phi of the two cells' faces -- costs 21 % more entries for 3.6 % fewer applications)
    }
    int Lcc = 0, Lfc = 0, Lcf = 0; // the largest levels: cell-cell, cell state -> phiRes, phi state -> cell residual
    for (int a = 0; a < 3; a++)
    {
        for (int b = 0; b < 3; b++) Lcc = std::max(Lcc, lvCell[a][b]);
        Lfc = std::max(Lfc, lvPhiRes[a]);
        Lcf = std::max(Lcf, lvOfPhi[a]);
    }
    if (phiPhi) Lcf = std::max(Lcf, 1);
    // owned faces per cell (a face belongs to the block of its owner cell)
    // (a cut face whose owner is a ghost sits in the block of its local cell; its row is a trivial identity row)
    auto blockCell = [&](int f) { return hm.own[f] < nC ? hm.own[f] : hm.nei[f]; };
    std::vector<int> ofOff(nC + 1, 0), ofList(nF);
    for (int f = 0; f < nF; f++) ofOff[blockCell(f) + 1]++;
    for (int c = 0; c < nC; c++) ofOff[c + 1] += ofOff[c];
    {
        std::vector<int> pos(ofOff.begin(), ofOff.end() - 1);
        for (int f = 0; f < nF; f++) ofList[pos[blockCell(f)]++] = f;
    }
    // all faces of a cell from the ELL table
    auto facesOf = [&](int c, std::vector<int>& out) {
        for (int k = 0; k < hm.maxCF; k++)
        {
            const int e = hm.cellFaces[(size_t)k * nC + c];
            if (e < 0) break;
            out.push_back(e >> 1);
        }
    };
    // ---- 1. multicolour ordering of the cells: same-colour cells share no matrix entry
    // same-colour cells must be further than `rho` apart; a larger radius gives more colours = an ordering closer to the
    // natural one (better ILU) at the price of more, smaller launches per application (adjEqnOption.pcColourRadius, extension)
    const int rho = std::max(std::max(Lcc, Lfc + 1), Lcf + 1) + pcExtraColourRadius;
    std::vector<int> colour;
    int nCol;
    const int blk = pcBlockCells;
    if (blk > 0)
    {
        // block-Jacobi ILU(0) with the natural (given) cell order inside blocks of `blk` consecutive cells -- the reference's
        // PCASM (overlap 0) + PCILU with natural ordering per block (DALinearEqn.C:212-216, 283-291), scheduled by dependency level:
        // level(c) = 1 + max level of the earlier cells of the same block coupled to c.  Cells of one level (over all blocks) are
        // mutually independent and form one "colour" of the kernels; couplings across blocks are dropped from the pattern below.
        colour.assign(nC, 0);
        std::vector<int> ballCells;
        nCol = 0;
        for (int c = 0; c < nC; c++)
        {
            G.ball(&c, 1, rho, ballCells);
            int lvl = 0;
            for (int x : ballCells)
                if (x < c && x / blk == c / blk) lvl = std::max(lvl, colour[x] + 1);
            colour[c] = lvl;
            nCol = std::max(nCol, lvl + 1);
        }
    }
    else
        nCol = detail::greedyColour(nC, [&](int c, std::vector<int>& out) { G.ball(&c, 1, rho, out); }, colour);
    std::vector<std::vector<int>> cellsOf(nCol);
    for (int c = 0; c < nC; c++) cellsOf[colour[c]].push_back(c);
    K.perm.assign(K.n, -1);
    K.iperm.assign(K.n, -1);
    K.colours.clear();
    std::vector<int> groupOfRow(K.n), groupRows, groupStart;
    int next = 0;
    for (int k = 0; k < nCol; k++)
    {
        auto& cl = cellsOf[k];
        std::stable_sort(cl.begin(), cl.end(), [&](int a, int b) { return (ofOff[a + 1] - ofOff[a]) > (ofOff[b + 1] - ofOff[b]); });
        int maxOwned = 0;
        for (int c : cl) maxOwned = std::max(maxOwned, ofOff[c + 1] - ofOff[c]);
        if (ns + maxOwned > MAXSLOT) throw Error("calcdRdWT: too many faces per cell for the block ordering");
        ColourView cv;
        cv.nCells = (int)cl.size();
        cv.nSlots = ns + maxOwned;
        for (int s = 0; s < MAXSLOT; s++) cv.slotStart[s] = cv.slotCount[s] = 0;
        for (int s = 0; s < cv.nSlots; s++)
        {
            cv.slotStart[s] = next;
            int cnt = 0;
            for (int c : cl)
            {
                int ext;
                if (s < 3) ext = 3 * c + s;
                else if (s < ns) ext = (s)*nC + c; // p at 3nC + c, nuTilda at 4nC + c
                else
                {
                    const int q = s - ns;
                    if (q >= ofOff[c + 1] - ofOff[c]) break; // cells sorted by owned-face count
                    ext = offPhi + ofList[ofOff[c] + q];
                }
                K.perm[next] = ext;
                K.iperm[ext] = next;
                groupOfRow[next] = (int)groupRows.size();
                next++;
                cnt++;
            }
            cv.slotCount[s] = cnt;
            groupStart.push_back(cv.slotStart[s]);
            groupRows.push_back(cnt);
        }
        K.colours.push_back(cv);
    }
    if (next != K.n) throw Error("calcdRdWT: ordering does not cover all states");
    lap("ordering colours + permutation");
    // ---- 2. sparsity pattern (new numbering), two passes: lengths, then ELL fill
    const int nG = (int)groupRows.size();
    std::vector<int> width(nG, 0);
    K.rowLen.assign(K.n, 0);
    auto faceSeeds = [&](int f, int* seeds) {
        int ns_ = 0;
        if (hm.own[f] < nC) seeds[ns_++] = hm.own[f];
        if (f < nIF && hm.nei[f] < nC) seeds[ns_++] = hm.nei[f];
        return ns_;
    };
    // per-thread scratch: the rows of different cells / faces are independent
    struct Work
    {
        CellGraph::Scratch sc;
        std::vector<int> cellsBall, cols, faces, width, levelEnd;
        int64_t nnz = 0;
    };
    const int nThreads = std::max(1, detail::hostThreads() / std::max(1, nRanks)); // the ranks of a node share its cores
    std::vector<Work> work(nThreads);
    for (Work& w : work) w.width.assign(nG, 0);
    // state kind of cell state s (0 U, 1 p, 2 nuTilda; the compressible T follows p) and residual kind of cell-residual slot s
    auto kindOf = [&](int s) { return s < 3 ? 0 : (s == ns - 1 && par.turb ? 2 : 1); };
    // the ball of the cell is gathered once (cellBall) and shared by the rows of its states
    auto cellBall = [&](Work& w, int c) { G.ball(&c, 1, std::max(Lcc, Lfc), w.cellsBall, w.sc, &w.levelEnd); };
    auto cellRowCols = [&](Work& w, int c, int s) {
        std::vector<int>& cols = w.cols;
        cols.clear();
        const int ks = kindOf(s);
        auto within = [&](int lv) { return lv < 0 ? 0 : w.levelEnd[std::min(lv, (int)w.levelEnd.size() - 1)]; };
        for (int r = 0; r < ns; r++)
        {
            const int nIn = within(lvCell[ks][kindOf(r)]);
            for (int q = 0; q < nIn; q++)
            {
                const int x = w.cellsBall[q];
                if (blk > 0 && x / blk != c / blk) continue; // block-Jacobi: couplings across blocks are dropped
                cols.push_back(K.iperm[r < 3 ? 3 * x + r : r * nC + x]);
            }
        }
        w.faces.clear();
        const int nIn = within(lvPhiRes[ks]);
        for (int q = 0; q < nIn; q++) facesOf(w.cellsBall[q], w.faces);
        std::sort(w.faces.begin(), w.faces.end());
        w.faces.erase(std::unique(w.faces.begin(), w.faces.end()), w.faces.end());
        for (int f : w.faces)
            if (!(blk > 0 && blockCell(f) / blk != c / blk)) cols.push_back(K.iperm[offPhi + f]);
        std::sort(cols.begin(), cols.end());
    };
    auto faceRowCols = [&](Work& w, int f) {
        std::vector<int>& cols = w.cols;
        cols.clear();
        if (hm.own[f] >= nC)
        {
            cols.push_back(K.iperm[offPhi + f]); // phi of this cut face belongs to the neighbouring rank
            return;
        }
        int seeds[2];
        const int nSeeds = faceSeeds(f, seeds);
        G.ball(seeds, nSeeds, Lcf, w.cellsBall, w.sc, &w.levelEnd);
        for (int r = 0; r < ns; r++)
        {
            const int lv = lvOfPhi[kindOf(r)];
            const int nIn = lv < 0 ? 0 : w.levelEnd[std::min(lv, (int)w.levelEnd.size() - 1)];
            for (int q = 0; q < nIn; q++)
            {
                const int x = w.cellsBall[q];
                if (blk > 0 && x / blk != blockCell(f) / blk) continue;
                cols.push_back(K.iperm[r < 3 ? 3 * x + r : r * nC + x]);
            }
        }
        if (phiPhi)
        {
            w.faces.clear();
            for (int q = 0; q < nSeeds; q++) facesOf(seeds[q], w.faces);
            w.faces.push_back(f);
            std::sort(w.faces.begin(), w.faces.end());
            w.faces.erase(std::unique(w.faces.begin(), w.faces.end()), w.faces.end());
            for (int g : w.faces)
                if (g == f || !(blk > 0 && blockCell(g) / blk != blockCell(f) / blk)) cols.push_back(K.iperm[offPhi + g]);
        }
        else
            cols.push_back(K.iperm[offPhi + f]);
        std::sort(cols.begin(), cols.end());
    };
    detail::parallelFor(nC, nThreads, [&](int t, int b, int e) {
        Work& w = work[t];
        for (int c = b; c < e; c++)
        {
            cellBall(w, c);
            for (int s = 0; s < ns; s++)
            {
                if (s == 0 || s >= 3) cellRowCols(w, c, s); // the three components of U share their columns
                const int i = K.iperm[s < 3 ? 3 * c + s : s * nC + c];
                K.rowLen[i] = (int)w.cols.size();
                w.width[groupOfRow[i]] = std::max(w.width[groupOfRow[i]], (int)w.cols.size());
            }
        }
    });
    detail::parallelFor(nF, nThreads, [&](int t, int b, int e) {
        Work& w = work[t];
        for (int f = b; f < e; f++)
        {
            faceRowCols(w, f);
            const int i = K.iperm[offPhi + f];
            K.rowLen[i] = (int)w.cols.size();
            w.width[groupOfRow[i]] = std::max(w.width[groupOfRow[i]], (int)w.cols.size());
        }
    });
    lap("pattern: row lengths");
    for (const Work& w : work)
        for (int g = 0; g < nG; g++) width[g] = std::max(width[g], w.width[g]);
    std::vector<int64_t> gOff(nG + 1, 0);
    for (int g = 0; g < nG; g++) gOff[g + 1] = gOff[g] + (int64_t)width[g] * groupRows[g];
    K.ellSize = gOff[nG];
    {
        int g = 0; // groups were pushed colour by colour, slot by slot
        for (ColourView& cv : K.colours)
            for (int sl = 0; sl < cv.nSlots; sl++) cv.slotBase[sl] = gOff[g++];
    }
    K.rowBase.resize(K.n);
    K.rowStride.resize(K.n);
    K.diag.assign(K.n, -1);
    for (int i = 0; i < K.n; i++)
    {
        const int g = groupOfRow[i];
        K.rowBase[i] = gOff[g] + (i - groupStart[g]);
        K.rowStride[i] = groupRows[g];
    }
    // uninitialised on purpose: every row writes its own entries *and* its padding below, so the 4*ellSize bytes (2.7 GB at 1M
    // cells) are first touched by the worker threads instead of one serial fill
    // (a page-locked staging buffer was measured: cudaMallocHost of 2.9 GB costs 1.2 s and the upload phase does not get shorter)
    std::unique_ptr<int32_t[]> hColOwned(new int32_t[(size_t)K.ellSize]);
    int32_t* hCol = hColOwned.get();
    K.nnz = 0;
    lap("pattern: ELL allocation");
    auto putRow = [&](Work& w, int i) {
        const std::vector<int>& cols = w.cols;
        for (size_t e = 0; e < cols.size(); e++)
        {
            hCol[(size_t)(K.rowBase[i] + (int64_t)e * K.rowStride[i])] = cols[e];
            if (cols[e] == i) K.diag[i] = (int)e;
        }
        for (int e = (int)cols.size(); e < width[groupOfRow[i]]; e++) hCol[(size_t)(K.rowBase[i] + (int64_t)e * K.rowStride[i])] = -1;
        w.nnz += (int64_t)cols.size();
        if (K.diag[i] < 0) throw Error("calcdRdWT: missing diagonal in the pattern");
    };
    detail::parallelFor(nC, nThreads, [&](int t, int b, int e) {
        Work& w = work[t];
        for (int c = b; c < e; c++)
        {
            cellBall(w, c);
            for (int s = 0; s < ns; s++)
            {
                if (s == 0 || s >= 3) cellRowCols(w, c, s);
                putRow(w, K.iperm[s < 3 ? 3 * c + s : s * nC + c]);
            }
        }
    });
    detail::parallelFor(nF, nThreads, [&](int t, int b, int e) {
        Work& w = work[t];
        for (int f = b; f < e; f++)
        {
            faceRowCols(w, f);
            putRow(w, K.iperm[offPhi + f]);
        }
    });
    for (const Work& w : work) K.nnz += w.nnz;
    lap("pattern: ELL fill");
    // ---- 3. colouring of the perturbations (DAColoring role).  Two states may share a colour when no
    // residual row in the pattern of one is touched by the other: cells at distance > Lcc + 3 (the
    // first-order pRes reaches 3 levels), faces whose cells are more than Lcf + 1 hops apart.
    std::vector<int> fdCell;
    const int nFdCell = detail::greedyColour(nC, [&](int c, std::vector<int>& out) { G.ball(&c, 1, Lcc + 3, out); }, fdCell);
    std::vector<int> fdFace;
    std::vector<int> tmpCells;
    const int nFdFace = detail::greedyColour(nF, [&](int f, std::vector<int>& out) {
        int seeds[2];
        const int nSeeds = faceSeeds(f, seeds);
        G.ball(seeds, nSeeds, Lcf + 1, tmpCells);
        out.clear();
        for (int x : tmpCells) facesOf(x, out);
    }, fdFace);
    const int nFd = ns * nFdCell + nFdFace;
    std::vector<int> cnt(nFd + 1, 0);
    auto fdColourOf = [&](int ext) {
        if (ext < 3 * nC) return (ext % 3) * nFdCell + fdCell[ext / 3];
        if (ext < offPhi) return (ext / nC) * nFdCell + fdCell[ext % nC];
        return ns * nFdCell + fdFace[ext - offPhi];
    };
    for (int j = 0; j < K.n; j++) cnt[fdColourOf(j) + 1]++;
    for (int k = 0; k < nFd; k++) cnt[k + 1] += cnt[k];
    K.fdStart.assign(cnt.begin(), cnt.end());
    K.fdList.resize(K.n);
    {
        std::vector<int> pos(cnt.begin(), cnt.end() - 1);
        for (int j = 0; j < K.n; j++) K.fdList[pos[fdColourOf(j)]++] = j;
    }
    lap("perturbation colours");
    // ---- upload
    K.dPerm.upload(be, K.perm);
    K.dIPerm.upload(be, K.iperm);
    K.dRowBase.upload(be, K.rowBase);
    K.dRowStride.upload(be, K.rowStride);
    K.dRowLen.upload(be, K.rowLen);
    K.dDiag.upload(be, K.diag);
    K.dCol.alloc(be, (size_t)K.ellSize, false);
    be.h2d(K.dCol.p, hCol, (size_t)K.ellSize * sizeof(int32_t));
    hColOwned.reset();
    K.dVal.alloc(be, (size_t)K.ellSize);
    K.dFdList.upload(be, K.fdList);
    K.R0.alloc(be, K.n);
    K.R1.alloc(be, K.n);
    K.t1.alloc(be, K.n);
    K.t2.alloc(be, K.n);
    K.symbolic = true;
    lap("upload");
    if (printInfo)
        fprintf(stderr, "[dab200] dRdWTPC: %d states, %lld nonzeros (%.1f/row), ELL %lld, %d ordering colours, %d FD colours (%d cell x %d + %d face)\n",
                K.n, (long long)K.nnz, (double)K.nnz / K.n, (long long)K.ellSize, nCol, nFd, nFdCell, ns, nFdFace);
}

inline void Solver::calcPC()
{
    const auto t0 = std::chrono::steady_clock::now();
    Krylov& K = kry;
    if (!K.symbolic) pcSymbolic();
    if (pcSymbolicOnly) return; // profiling hook (adjEqnOption.pcSymbolicOnly): host set-up only, nothing assembled
    auto tPrev = std::chrono::steady_clock::now();
    auto lap = [&](const char* what) {
        if (!printInfo) return;
        be.sync();
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[dab200] calcPC %-34s %.3f s\n", what, std::chrono::duration<double>(now - tPrev).count());
        tPrev = now;
    };
    be.zero(K.dVal.p, (size_t)K.ellSize * sizeof(double));
    StatePtrs sp{dU.p, dP.p, dNt.p, dPhi.p, hm.nC, par.turb, dMagSf.p, par.sU, par.sP, par.sNut, par.sPhi, par.phiNorm};
    if (par.comp)
    {
        sp.T = dT.p;
        sp.sT = par.sT;
    }
    // R0 at the unperturbed state with the div(pc) schemes (DASolver::calcdRdWT isPC=1)
    forward(1, K.R0.p, true);
    const int nFd = (int)K.fdStart.size() - 1;
    EllView A = K.view();
    for (int k = 0; k < nFd; k++)
    {
        const int n = K.fdStart[k + 1] - K.fdStart[k];
        if (n == 0) continue;
        const int32_t* list = K.dFdList.p + K.fdStart[k];
        be.launch(n, FdPerturb{sp, list, fdStep});
        forward(1, K.R1.p, false); // ghosts frozen: block-Jacobi over ranks, no collective inside the loop
        be.launch(n, FdFill{A, list, K.dIPerm.p, K.dPerm.p, K.R0.p, K.R1.p, 1.0 / fdStep});
        be.launch(n, FdPerturb{sp, list, -fdStep});
    }
    // restore the exact states and invalidate the record (it now holds first-order intermediates)
    {
        const size_t nC = hm.nC;
        be.d2d(dU.p, dWext.p, 3 * nC * sizeof(double));
        be.d2d(dP.p, dWext.p + 3 * nC, nC * sizeof(double));
        size_t off = 4 * nC;
        if (par.comp)
        {
            be.d2d(dT.p, dWext.p + off, nC * sizeof(double));
            off += nC;
        }
        if (par.turb)
        {
            be.d2d(dNt.p, dWext.p + off, nC * sizeof(double));
            off += nC;
        }
        be.d2d(dPhi.p, dWext.p + off, (size_t)hm.nF * sizeof(double));
        recorded = false;
    }
    lap("coloured finite differences");
    if (keepPCMatrix)
    {
        K.hValAssembled.resize((size_t)K.ellSize);
        be.d2h(K.hValAssembled.data(), K.dVal.p, (size_t)K.ellSize * sizeof(double));
    }
    // ILU(0), one kernel per colour
    for (const ColourView& cv : K.colours) be.launch(cv.nCells, IluFactorColour{A, cv, 1e-10});
    // adjEqnOption.pcStorage "fp32" (extension): the triangular solves read an fp32 copy of the factors -- the preconditioner is an
    // approximation anyway, the Krylov operator and all vectors stay fp64; 12 -> 8 bytes per nonzero per application
    K.useF32 = pcStorage == "fp32";
    if (K.useF32)
    {
        if (K.dValF.n < (size_t)K.ellSize) K.dValF.alloc(be, (size_t)K.ellSize, false);
        for (int64_t o = 0; o < K.ellSize; o += (int64_t)1 << 30)
            be.launch((int)std::min<int64_t>((int64_t)1 << 30, K.ellSize - o), CvtToFloat{K.dVal.p + o, K.dValF.p + o});
    }
    be.sync();
    lap("ILU(0) factorisation (+ fp32 copy)");
    K.pcValid = true;
    K.pcFactored = true;
    K.pcAssemblies++;
    K.coarse.enabled = coarseAggregates > 0;
    K.coarse.valid = false;
    if (K.coarse.enabled) coarseSetup();
    be.sync();
    lap("coarse space");
    K.pcSec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// aggregated pressure coarse space: greedy breadth-first aggregates of ~nC/coarseAggregates cells; the Galerkin
// coarse operator P^T A P is probed with the matrix-free product (one product per aggregate) and factorised
// densely on the host.  Two-level role: the multicolour ILU(0) damps the short wavelengths, the coarse solve the
// domain-wide pressure modes it cannot see.
inline void Solver::coarseSetup()
{
    Krylov& K = kry;
    Coarse& Cs = K.coarse;
    const int nC = hm.nC, n = nDof(), offP = 3 * nC;
    detail::CellGraph Gagg;
    Gagg.build(hm);
    detail::CellGraph& G = Gagg;
    const int target = std::max(1, nC / std::max(1, coarseAggregates / std::max(1, nRanks)));
    std::vector<int32_t> aggOf(nC, -1);
    int nAgg = 0;
    std::vector<int> queue;
    for (int seed = 0; seed < nC; seed++)
    {
        if (aggOf[seed] >= 0) continue;
        queue.assign(1, seed);
        aggOf[seed] = nAgg;
        int cnt = 1;
        for (size_t q = 0; q < queue.size() && cnt < target; q++)
            for (int e = G.off[queue[q]]; e < G.off[queue[q] + 1] && cnt < target; e++)
            {
                const int x = G.adj[e];
                if (aggOf[x] < 0)
                {
                    aggOf[x] = nAgg;
                    queue.push_back(x);
                    cnt++;
                }
            }
        nAgg++;
    }
    // cells sorted by aggregate, chunks of 32
    std::vector<int32_t> cnt(nAgg + 1, 0), cells(nC);
    for (int c = 0; c < nC; c++) cnt[aggOf[c] + 1]++;
    for (int a = 0; a < nAgg; a++) cnt[a + 1] += cnt[a];
    {
        std::vector<int32_t> pos(cnt.begin(), cnt.end() - 1);
        for (int c = 0; c < nC; c++) cells[pos[aggOf[c]]++] = c;
    }
    std::vector<int32_t> chunkStart, aggChunkOff(1, 0);
    for (int a = 0; a < nAgg; a++)
    {
        for (int i = cnt[a]; i < cnt[a + 1]; i += 32) chunkStart.push_back(i);
        aggChunkOff.push_back((int32_t)chunkStart.size());
    }
    chunkStart.push_back(nC);
    // chunks must not cross aggregates: the end of a chunk is min(next chunk start, end of its aggregate)
    // (consecutive aggregates are contiguous in `cells`, so chunkStart[t+1] is already that end)
    Cs.nChunks = (int)chunkStart.size() - 1;
    Cs.nAggLocal = nAgg;
    // global numbering of the aggregates (rank-major)
    std::vector<double> counts(nRanks, 0.0);
    counts[rank] = nAgg;
    DevBuf<double> tmp;
    tmp.upload(be, counts);
    comm.allreduceSum(be, tmp.p, nRanks);
    be.d2h(counts.data(), tmp.p, nRanks * sizeof(double));
    Cs.aggBase = 0;
    Cs.nAggGlobal = 0;
    for (int r = 0; r < nRanks; r++)
    {
        if (r < rank) Cs.aggBase += (int)counts[r];
        Cs.nAggGlobal += (int)counts[r];
    }
    Cs.dAggOf.upload(be, aggOf);
    Cs.dCells.upload(be, cells);
    Cs.dChunkStart.upload(be, chunkStart);
    Cs.dAggChunkOff.upload(be, aggChunkOff);
    Cs.dPartial.alloc(be, Cs.nChunks + 1);
    Cs.dRc.alloc(be, Cs.nAggGlobal + 1);
    Cs.dYc.alloc(be, Cs.nAggGlobal + 1);
    Cs.hRc.assign(Cs.nAggGlobal, 0.0);
    K.t3.alloc(be, n);
    // sparse A*P collected while probing (adjEqnOption.coarseSparseAP, default 1; 0: one extra matrix-free product per application)
    Cs.apValid = false;
    const bool wantAp = coarseSparseAP != 0;
    if (wantAp)
    {
        Cs.apCap = (long long)3 * n;
        Cs.dApRow.alloc(be, (size_t)Cs.apCap, false);
        Cs.dApAgg.alloc(be, (size_t)Cs.apCap, false);
        Cs.dApVal.alloc(be, (size_t)Cs.apCap, false);
        Cs.dApCount.alloc(be, 1);
    }
    const int offPhiAp = nCellStates() * nC;
    auto extractAp = [&](const int32_t* dSrcOfAgg, int constSrc) {
        if (!wantAp) return;
        be.launch(n, ApExtract{K.t3.p, nC, nCellStates(), offPhiAp, Cs.dAggOf.p, mv.own, mv.nei, dSrcOfAgg, constSrc, Cs.dApCount.p, Cs.apCap,
                               Cs.dApRow.p, Cs.dApAgg.p, Cs.dApVal.p});
    };
    // Galerkin operator, column by column
    const int Kg = Cs.nAggGlobal;
    Cs.lu.assign((size_t)Kg * Kg, 0.0);
    ensureRecorded();
    int nProbes = 0;
    if (nRanks == 1 && coarseProbeReach > 0 && nAgg > 64)
    {
        // cyclic patches: the reach sets follow the periodic adjacency (an image stands for its source cell)
        detail::CellGraph Gp;
        if (partitioned)
        {
            std::vector<int> alias(hm.nCtot - nC, -1);
            for (int i = 0; i < part.halo.selfRecvCount; i++) alias[part.halo.selfRecvStart - nC + i] = part.halo.selfSendCells[i];
            Gp.build(hm, &alias);
        }
        detail::CellGraph& G = partitioned ? Gp : Gagg;
        // Coloured probing (one GPU): the transposed Jacobian couples a pressure DOF to residual rows at most `coarseProbeReach` cell
        // levels away, far less than an aggregate's diameter, so aggregates whose reach sets N(a) (the aggregates within that many
        // levels of a's cells) are disjoint share one probing vector; entry (i, a) is read from the restricted response at the only
        // aggregate a of the colour with i in N(a).  ~10-20 products instead of one per aggregate.  A response outside every reach
        // set means the reach was too short: fall back to one product per aggregate.
        std::vector<std::vector<int>> reach(nAgg);
        {
            std::vector<int> ballCells, seeds;
            std::vector<int> mark(nAgg, -1);
            for (int a = 0; a < nAgg; a++)
            {
                seeds.assign(cells.begin() + cnt[a], cells.begin() + cnt[a + 1]);
                G.ball(seeds.data(), (int)seeds.size(), coarseProbeReach, ballCells);
                for (int c : ballCells)
                    if (mark[aggOf[c]] != a)
                    {
                        mark[aggOf[c]] = a;
                        reach[a].push_back(aggOf[c]);
                    }
            }
        }
        std::vector<std::vector<int>> reachedBy(nAgg); // i -> the aggregates a with i in N(a)
        for (int a = 0; a < nAgg; a++)
            for (int i : reach[a]) reachedBy[i].push_back(a);
        std::vector<int> colour;
        const int nColours = detail::greedyColour(nAgg, [&](int a, std::vector<int>& out) {
            out.clear();
            for (int i : reach[a])
                for (int b : reachedBy[i]) out.push_back(b);
        }, colour);
        std::vector<int32_t> colour32(colour.begin(), colour.end());
        DevBuf<int32_t> dColour;
        dColour.upload(be, colour32);
        bool ok = true;
        std::vector<int> owner(nAgg);
        for (int k = 0; k < nColours && ok; k++)
        {
            be.launch(n, CoarseUnitColour{Cs.dAggOf.p, dColour.p, offP, nC, k, K.t2.p});
            matVecDev(K.t2.p, K.t3.p);
            coarseRestrict(K.t3.p);
            nProbes++;
            std::fill(owner.begin(), owner.end(), -1);
            for (int a = 0; a < nAgg; a++)
                if (colour[a] == k)
                    for (int i : reach[a]) owner[i] = a;
            if (wantAp)
            {
                std::vector<int32_t> o32(owner.begin(), owner.end());
                DevBuf<int32_t> dOwner;
                dOwner.upload(be, o32);
                extractAp(dOwner.p, -1);
                be.sync(); // dOwner goes out of scope
            }
            double big = 0.0;
            for (int i = 0; i < Kg; i++) big = std::max(big, std::fabs(Cs.hRc[i]));
            for (int i = 0; i < Kg && ok; i++)
            {
                if (owner[i] >= 0) Cs.lu[(size_t)i * Kg + owner[i]] = Cs.hRc[i];
                else if (std::fabs(Cs.hRc[i]) > 1e-12 * big) ok = false;
            }
        }
        if (!ok)
        {
            if (printInfo) fprintf(stderr, "[dab200] coarse space: probing reach %d too short, falling back to one product per aggregate\n", coarseProbeReach);
            std::fill(Cs.lu.begin(), Cs.lu.end(), 0.0);
            nProbes = 0;
            if (wantAp) be.zero(Cs.dApCount.p, sizeof(unsigned long long));
        }
        else if (printInfo)
            fprintf(stderr, "[dab200] coarse space: %d aggregates probed with %d coloured products\n", nAgg, nProbes);
    }
    if (nProbes == 0)
        for (int j = 0; j < Kg; j++)
        {
            const int local = (j >= Cs.aggBase && j < Cs.aggBase + nAgg) ? j - Cs.aggBase : -1;
            be.launch(n, CoarseUnit{Cs.dAggOf.p, offP, nC, local, K.t2.p});
            matVecDev(K.t2.p, K.t3.p);
            coarseRestrict(K.t3.p);
            for (int i = 0; i < Kg; i++) Cs.lu[(size_t)i * Kg + j] = Cs.hRc[i];
            extractAp(nullptr, j);
        }
    if (wantAp)
    {
        // COO -> CSR by row, entries of a row ordered by aggregate (the atomics fill the COO in no particular order: fix it)
        unsigned long long cnt = 0;
        be.d2h(&cnt, Cs.dApCount.p, sizeof(cnt));
        bool bad = (long long)cnt > Cs.apCap;
        std::vector<int32_t> row, agg;
        std::vector<double> val;
        if (!bad)
        {
            row.resize(cnt); agg.resize(cnt); val.resize(cnt);
            if (cnt)
            {
                be.d2h(row.data(), Cs.dApRow.p, cnt * sizeof(int32_t));
                be.d2h(agg.data(), Cs.dApAgg.p, cnt * sizeof(int32_t));
                be.d2h(val.data(), Cs.dApVal.p, cnt * sizeof(double));
            }
            for (size_t e = 0; e < cnt && !bad; e++)
                if (agg[e] < 0 || agg[e] >= Kg) bad = true; // a response outside every reach set: keep the exact product path
        }
        if (!bad)
        {
            std::vector<int32_t> ptr((size_t)n + 1, 0);
            for (size_t e = 0; e < cnt; e++) ptr[row[e] + 1]++;
            for (int r = 0; r < n; r++) ptr[r + 1] += ptr[r];
            std::vector<int32_t> pos(ptr.begin(), ptr.end() - 1), sAgg(cnt);
            std::vector<double> sVal(cnt);
            for (size_t e = 0; e < cnt; e++)
            {
                const int32_t q = pos[row[e]]++;
                sAgg[q] = agg[e];
                sVal[q] = val[e];
            }
            std::vector<std::pair<int32_t, double>> tmp;
            for (int r = 0; r < n; r++)
            {
                const int a = ptr[r], b = ptr[r + 1];
                if (b - a < 2) continue;
                tmp.clear();
                for (int e = a; e < b; e++) tmp.emplace_back(sAgg[e], sVal[e]);
                std::sort(tmp.begin(), tmp.end());
                for (int e = a; e < b; e++) { sAgg[e] = tmp[e - a].first; sVal[e] = tmp[e - a].second; }
            }
            Cs.dApPtr.upload(be, ptr);
            Cs.dApAggSorted.upload(be, sAgg);
            Cs.dApValSorted.upload(be, sVal);
            Cs.apValid = true;
            if (printInfo) fprintf(stderr, "[dab200] coarse space: sparse A*P with %llu entries (%.2f per row)\n", cnt, (double)cnt / n);
        }
        else if (printInfo)
            fprintf(stderr, "[dab200] coarse space: sparse A*P not usable (overflow or response outside the reach sets): matrix-free product kept\n");
        Cs.dApRow.release(); Cs.dApAgg.release(); Cs.dApVal.release();
    }
    Cs.factor(std::min(std::max(1, detail::hostThreads() / std::max(1, nRanks)), 32));
    {
        std::vector<double> invT;
        Cs.invertTransposed(invT, [&](int nItems, auto fn) {
            // small systems: one thread; the columns of the inverse are independent
            const int nt = nItems >= 256 ? std::max(1, detail::hostThreads() / std::max(1, nRanks)) : 1;
            if (nt == 1) fn(0, 0, nItems);
            else
            {
                std::vector<std::thread> th;
                for (int t = 0; t < nt; t++)
                    th.emplace_back([&, t]() { fn(t, (int)((int64_t)nItems * t / nt), (int)((int64_t)nItems * (t + 1) / nt)); });
                for (auto& x : th) x.join();
            }
        });
        Cs.dInvT.upload(be, invT);
    }
    Cs.valid = true;
    (void)offP;
}

// hRc = P^T v (global coarse vector on the host, summed over ranks)
inline void Solver::coarseRestrict(const double* v, bool toHost)
{
    Coarse& Cs = kry.coarse;
    const int offP = 3 * hm.nC;
    be.launch(Cs.nChunks, CoarseRestrict1{v + offP, Cs.dCells.p, Cs.dChunkStart.p, Cs.dPartial.p});
    be.zero(Cs.dRc.p, (size_t)Cs.nAggGlobal * sizeof(double));
    be.launch(Cs.nAggLocal, CoarseRestrict2{Cs.dPartial.p, Cs.dAggChunkOff.p, Cs.dRc.p + Cs.aggBase});
    comm.allreduceSum(be, Cs.dRc.p, Cs.nAggGlobal);
    if (toHost) be.d2h(Cs.hRc.data(), Cs.dRc.p, (size_t)Cs.nAggGlobal * sizeof(double));
}

// z = M^{-1} v  (external layout in and out).  With the coarse space: multiplicative two-level,
// z1 = P Ac^{-1} P^T v, z = z1 + ILU^{-1} (v - A z1).
inline void Solver::applyPC(const double* v, double* z)
{
    Krylov& K = kry;
    if (K.coarse.enabled && K.coarse.valid)
    {
        Coarse& Cs = K.coarse;
        const int n = nDof();
        // coarse solve on the device: yc = Ac^-1 rc as a GEMV with the explicit (transposed) inverse -- no host round trip
        coarseRestrict(v, false);
        be.launch(Cs.nAggGlobal, CoarseApply{Cs.dInvT.p, Cs.dRc.p, Cs.nAggGlobal, Cs.dYc.p});
        be.launch(n, CoarseProlong{Cs.dYc.p, Cs.dAggOf.p, 3 * hm.nC, hm.nC, Cs.aggBase, K.t2.p}); // z1
        if (Cs.apValid)
            be.launch(n, ApApply{Cs.dApPtr.p, Cs.dApAggSorted.p, Cs.dApValSorted.p, Cs.dYc.p, v, K.t3.p}); // t3 = v - (A P) yc
        else
        {
            matVecDev(K.t2.p, K.t3.p);
            kspExtraMatvecs++;
            be.launch(n, SubVec{v, K.t3.p}); // t3 = v - A z1
        }
        applyIlu(K.t3.p, z);
        be.launch(n, AxpyVec{K.t2.p, 1.0, z});
    }
    else
        applyIlu(v, z);
    // Richardson sweeps on the exact operator (the reference's optional "globalPCIters" wrapper, DALinearEqn.C:74-140):
    // z <- z + M^-1 (v - A z); a fixed linear operator, so plain (non-flexible) GMRES stays valid
    if (globalPCIters > 0)
    {
        const int n = nDof();
        if (K.t4.n < (size_t)n)
        {
            K.t4.alloc(be, n);
            K.t5.alloc(be, n);
        }
        for (int it = 0; it < globalPCIters; it++)
        {
            matVecDev(z, K.t4.p);
            kspExtraMatvecs++;
            be.launch(n, SubVec{v, K.t4.p}); // t4 = v - A z
            applyIlu(K.t4.p, K.t5.p);
            be.launch(n, AxpyVec{K.t5.p, richardsonOmega, z});
        }
    }
}

inline void Solver::applyIlu(const double* v, double* z)
{
    Krylov& K = kry;
    EllView A = K.view();
    be.launch(K.n, GatherVec{v, K.dPerm.p, K.t1.p});
    auto padded = [](int nCells, int lanes) { return (nCells * lanes + 31) / 32 * 32; }; // whole warps: see TriLowerColour
    if (pcBlockCells > 0)
    {
        // many small levels: four lanes per cell
        for (size_t k = 0; k < K.colours.size(); k++) be.launch(padded(K.colours[k].nCells, 4), TriLowerColour<4>{A, K.colours[k], K.t1.p});
        for (size_t k = K.colours.size(); k-- > 0;) be.launch(padded(K.colours[k].nCells, 4), TriUpperColour<4>{A, K.colours[k], K.t1.p});
    }
    else
    {
        for (size_t k = 0; k < K.colours.size(); k++) be.launch(padded(K.colours[k].nCells, 1), TriLowerColour<1>{A, K.colours[k], K.t1.p});
        for (size_t k = K.colours.size(); k-- > 0;) be.launch(padded(K.colours[k].nCells, 1), TriUpperColour<1>{A, K.colours[k], K.t1.p});
    }
    be.launch(K.n, ScatterVec{K.t1.p, K.dPerm.p, z});
}

// DALinearEqn::solveLinearEqn: GMRES(restart), right PC, zero initial guess, unpreconditioned norm
inline int Solver::solveLinearEqn(const double* rhs, double* sol, KspStats& st)
{
    Krylov& K = kry;
    // adjPCLag > 1 (reference mphys_dafoam.py:511-530): the caller decides when calcdRdWT refreshes the preconditioner; a
    // factorisation of an earlier design keeps being used in between
    if (!K.pcValid && !(K.pcFactored && adjPCLag > 1 && K.symbolic)) calcPC();
    ensureRecorded();
    if (kspType == "idrs") return solveIdrs(rhs, sol, st);
    const int n = nDof();
    const int m = std::max(1, std::min(gmresRestart, gmresMaxIters));
    K.ops.init(be, &comm, m + 2); // grow-only: a no-op when another solver already sized it larger
    if (K.vCap < m + 1 || K.V.n < (size_t)(m + 1) * n)
    {
        K.V.alloc(be, (size_t)(m + 1) * n, false);
        K.vCap = m + 1;
        K.w.alloc(be, n);
        K.z.alloc(be, n);
        K.xdev.alloc(be, n);
        K.bdev.alloc(be, n);
        if (K.hdev.n < (size_t)(m + 2)) K.hdev.alloc(be, m + 2); // grow-only: IDR(s) may keep using it with s > m + 2
        K.ops.init(be, &comm, m + 2);
    }
    be.h2d(K.bdev.p, rhs, (size_t)n * sizeof(double));
    be.zero(K.xdev.p, (size_t)n * sizeof(double));
    auto timer = be.timer();
    be.sync();
    timer.start();
    const long l0 = be.launches;
    const double bnorm = K.ops.norm2(K.bdev.p, n);
    st.r0 = bnorm;
    st.nMatvec = 0;
    kspExtraMatvecs = 0;
    const double tol = std::max(gmresRelTol * bnorm, gmresAbsTol);
    std::vector<double> H((size_t)(m + 1) * m, 0.0), cs(m, 0.0), sn(m, 0.0), g(m + 1, 0.0), yv(m, 0.0), hcol(m + 2, 0.0);
    int its = 0, nRefine = 0, nTrueRestarts = 0;
    double rnorm = bnorm;
    int reason = 0;
    if (bnorm == 0.0)
    {
        reason = 3;
    }
    while (reason == 0)
    {
        // r = b - A x (x = 0 on the first cycle)
        double beta;
        if (its == 0)
        {
            be.d2d(K.w.p, K.bdev.p, (size_t)n * sizeof(double));
            beta = bnorm;
        }
        else
        {
            matVecDev(K.xdev.p, K.w.p);
            st.nMatvec++;
            be.launch(n, SubVec{K.bdev.p, K.w.p});
            beta = K.ops.norm2(K.w.p, n);
        }
        rnorm = beta;
        if (rnorm <= tol) { reason = rnorm <= gmresRelTol * bnorm ? 2 : 3; break; }
        be.launch(n, ScaleCopy{K.w.p, 1.0 / beta, K.V.p});
        std::fill(g.begin(), g.end(), 0.0);
        g[0] = beta;
        int k = 0;
        for (; k < m && its < gmresMaxIters; k++, its++)
        {
            double* vk = K.V.p + (size_t)k * n;
            double* vk1 = K.V.p + (size_t)(k + 1) * n;
            applyPC(vk, K.z.p);
            matVecDev(K.z.p, vk1);
            st.nMatvec++;
            // classical Gram-Schmidt with refinement if needed (KSP_GMRES_CGS_REFINE_IFNEEDED)
            const double* d = K.ops.dots(K.V.p, n, k + 2, vk1, n); // V_0..V_k . w and w . w (V_{k+1} = w)
            for (int j = 0; j <= k; j++) hcol[j] = d[j];
            const double wn2 = d[k + 1];
            K.putCoeffs(be, hcol.data(), k + 1);
            be.launch(n, MultiAxpy{K.V.p, n, k + 1, K.hdev.p, vk1, 0});
            // ||w - V h||^2 = ||w||^2 - ||h||^2 (V orthonormal); refine -- and measure the norm explicitly -- only when
            // cancellation makes that estimate unreliable (the IFNEEDED criterion of the reference's KSP)
            double hn2 = 0.0;
            for (int j = 0; j <= k; j++) hn2 += hcol[j] * hcol[j];
            double nrm;
            // refine when the projection removed more than 3/4 of ||w||^2 (cancellation); looser than PETSc's IFNEEDED test
            // (||w_new|| < ||h||, which fires on ~85 % of the iterations here and doubles the basis traffic): convergence is
            // verified with the true residual below, so a slightly optimistic recurrence only costs a restart
            if (wn2 - hn2 < 0.25 * wn2 || useMGSO)
            {
                nRefine++;
                const double* d2 = K.ops.dots(K.V.p, n, k + 2, vk1, n);
                std::vector<double> h2(d2, d2 + k + 1);
                const double wn2b = d2[k + 1];
                K.putCoeffs(be, h2.data(), k + 1);
                be.launch(n, MultiAxpy{K.V.p, n, k + 1, K.hdev.p, vk1, 0});
                double h2n = 0.0;
                for (int j = 0; j <= k; j++)
                {
                    hcol[j] += h2[j];
                    h2n += h2[j] * h2[j];
                }
                nrm = (wn2b - h2n > 0.25 * wn2b) ? std::sqrt(wn2b - h2n) : K.ops.norm2(vk1, n);
            }
            else
                nrm = std::sqrt(wn2 - hn2);
            hcol[k + 1] = nrm;
            if (nrm > 0.0) be.launch(n, ScaleCopy{vk1, 1.0 / nrm, vk1});
            // Givens rotations
            for (int j = 0; j < k; j++)
            {
                const double t = cs[j] * hcol[j] + sn[j] * hcol[j + 1];
                hcol[j + 1] = -sn[j] * hcol[j] + cs[j] * hcol[j + 1];
                hcol[j] = t;
            }
            const double dd = std::hypot(hcol[k], hcol[k + 1]);
            cs[k] = dd > 0 ? hcol[k] / dd : 1.0;
            sn[k] = dd > 0 ? hcol[k + 1] / dd : 0.0;
            hcol[k] = dd;
            hcol[k + 1] = 0.0;
            g[k + 1] = -sn[k] * g[k];
            g[k] = cs[k] * g[k];
            for (int j = 0; j <= k; j++) H[(size_t)j * m + k] = hcol[j];
            rnorm = std::fabs(g[k + 1]);
            if (printInfo && (its % 50 == 0)) fprintf(stderr, "[dab200] GMRES %4d  residual %.6e\n", its, rnorm);
            if (rnorm <= tol || nrm == 0.0)
            {
                k++;
                its++;
                break;
            }
        }
        // y = H^{-1} g, x += M^{-1} (V y)
        for (int i = k - 1; i >= 0; i--)
        {
            double s = g[i];
            for (int j = i + 1; j < k; j++) s -= H[(size_t)i * m + j] * yv[j];
            yv[i] = s / H[(size_t)i * m + i];
        }
        K.putCoeffs(be, yv.data(), k);
        be.launch(n, MultiAxpy{K.V.p, n, k, K.hdev.p, K.w.p, 1});
        applyPC(K.w.p, K.z.p);
        be.launch(n, AxpyVec{K.z.p, 1.0, K.xdev.p});
        if (rnorm <= tol)
        {
            // the Givens recurrence says converged: verify with the true residual b - A x (classical Gram-Schmidt can
            // lose enough orthogonality for the recurrence to be optimistic); if it is not there yet, the loop restarts from x
            matVecDev(K.xdev.p, K.w.p);
            st.nMatvec++;
            be.launch(n, SubVec{K.bdev.p, K.w.p});
            rnorm = K.ops.norm2(K.w.p, n);
            if (rnorm <= tol * 1.0000001) reason = rnorm <= gmresRelTol * bnorm * 1.0000001 ? 2 : 3;
            else if (its >= gmresMaxIters) reason = -3;
            else nTrueRestarts++;
        }
        else if (its >= gmresMaxIters) reason = -3;
    }
    if (reason == -3)
    {
        // report the true residual, not the recurrence estimate, when the iteration budget ran out
        matVecDev(K.xdev.p, K.w.p);
        st.nMatvec++;
        be.launch(n, SubVec{K.bdev.p, K.w.p});
        rnorm = K.ops.norm2(K.w.p, n);
    }
    st.solveSec = timer.stopMs() * 1e-3;
    (void)l0;
    be.d2h(sol, K.xdev.p, (size_t)n * sizeof(double));
    st.nMatvec += kspExtraMatvecs;
    st.iterations = its;
    st.reason = reason;
    st.rn = rnorm;
    st.pcSec = K.pcSec;
    if (printInfo)
        fprintf(stderr, "[dab200] Main iteration %d KSP Residual norm %14.12e %.3f s (%d Gram-Schmidt refinements, %d true-residual restarts)\n", its, rnorm, st.solveSec, nRefine, nTrueRestarts);
    // reference success rule (DALinearEqn.C:422-434)
    const double absRatio = rnorm / gmresAbsTol;
    const double relRatio = bnorm > 0 ? rnorm / bnorm / gmresRelTol : 0.0;
    return (relRatio > gmresTolDiff && absRatio > gmresTolDiff) ? 1 : 0;
}

// IDR(s) (Sonneveld & van Gijzen; the bi-orthogonal variant of van Gijzen & Sonneveld, ACM TOMS Algorithm 913) with the same right
// preconditioner, stopping rule and statistics as the GMRES above.  An extension (adjEqnOption.kspType idrs; the reference's KSP is
// GMRES): 3s + 4 work vectors and O(s) vector updates per product instead of an orthogonalisation against the whole basis, which is
// 85 % of the GMRES time at 1M cells (DESIGN.md section 6).  `iterations` counts operator applications, like a GMRES iteration.
// The recurrence residual is checked against the true residual b - A x before returning; when they disagree the method restarts on
// the true residual.
inline int Solver::solveIdrs(const double* rhs, double* sol, KspStats& st)
{
    Krylov& K = kry;
    if (!K.pcValid && !(K.pcFactored && adjPCLag > 1 && K.symbolic)) calcPC();
    ensureRecorded();
    const int n = nDof(), s = idrS;
    if (K.idrS != s || K.idr.n < (size_t)(3 * s + 4) * n)
    {
        K.idr.alloc(be, (size_t)(3 * s + 4) * n, false);
        K.idrS = s;
        K.xdev.alloc(be, n);
        K.bdev.alloc(be, n);
        K.ops.init(be, &comm, std::max(gmresRestart, 32) + 2);
        K.vCap = 0; // the GMRES basis (if any) shares nothing with this workspace
        K.V.alloc(be, 1, false);
        K.idrShadowReady = false;
    }
    // the coefficient buffer and the dot-product workspace are shared with GMRES, which may have re-sized them since this
    // workspace was made (IDR(s), GMRES(m < s - 1), IDR(s) on one handle): both only grow
    if (K.hdev.n < (size_t)s) K.hdev.alloc(be, s);
    K.ops.init(be, &comm, s);
    double* P = K.idr.p;
    double* G = P + (size_t)s * n;
    double* U = G + (size_t)s * n;
    double* r = U + (size_t)s * n;
    double* t = r + n; // directly after r: dots(r, n, 2, t) = (r.t, t.t)
    double* v = t + n;
    double* z = v + n;
    // shadow space: fixed pseudo-random vectors, orthonormalised (modified Gram-Schmidt); kept between solves
    if (!K.idrShadowReady)
    {
        K.idrShadowReady = true;
        std::vector<double> h((size_t)n);
        for (int j = 0; j < s; j++)
        {
            uint64_t x = 0x9E3779B97F4A7C15ull * (uint64_t)(j + 1) + 0xD1B54A32D192ED03ull * (uint64_t)(rank + 1);
            for (int i = 0; i < n; i++)
            {
                x ^= x << 13; x ^= x >> 7; x ^= x << 17; // xorshift64
                h[i] = (double)(x >> 11) * (1.0 / 9007199254740992.0) - 0.5;
            }
            double* Pj = P + (size_t)j * n;
            be.h2d(Pj, h.data(), (size_t)n * sizeof(double));
            for (int i = 0; i < j; i++)
            {
                const double d = K.ops.dots(P + (size_t)i * n, n, 1, Pj, n)[0];
                be.launch(n, AxpyVec{P + (size_t)i * n, -d, Pj});
            }
            const double nr = K.ops.norm2(Pj, n);
            be.launch(n, ScaleCopy{Pj, 1.0 / nr, Pj});
        }
    }
    be.h2d(K.bdev.p, rhs, (size_t)n * sizeof(double));
    be.zero(K.xdev.p, (size_t)n * sizeof(double));
    auto timer = be.timer();
    be.sync();
    timer.start();
    const double bnorm = K.ops.norm2(K.bdev.p, n);
    st.r0 = bnorm;
    st.nMatvec = 0;
    kspExtraMatvecs = 0;
    const double tol = std::max(gmresRelTol * bnorm, gmresAbsTol);
    int its = 0, reason = bnorm == 0.0 ? 3 : 0, nRestarts = 0;
    double rnorm = bnorm;
    std::vector<double> M((size_t)s * s), f(s), c(s);
    be.d2d(r, K.bdev.p, (size_t)n * sizeof(double));
    while (reason == 0)
    {
        // (re)start from the current x and its true residual r
        be.zero(G, (size_t)2 * s * n * sizeof(double)); // G and U
        std::fill(M.begin(), M.end(), 0.0);
        for (int i = 0; i < s; i++) M[(size_t)i * s + i] = 1.0;
        double om = 1.0;
        bool breakdown = false;
        while (rnorm > tol && its < gmresMaxIters && !breakdown)
        {
            {
                const double* d = K.ops.dots(P, n, s, r, n);
                for (int i = 0; i < s; i++) f[i] = d[i];
            }
            for (int k = 0; k < s && rnorm > tol && its < gmresMaxIters; k++)
            {
                // lower-triangular solve M[k:,k:] c = f[k:]
                for (int i = k; i < s; i++)
                {
                    double a = f[i];
                    for (int j = k; j < i; j++) a -= M[(size_t)i * s + j] * c[j];
                    c[i] = a / M[(size_t)i * s + i];
                }
                K.putCoeffs(be, c.data() + k, s - k);
                be.d2d(v, r, (size_t)n * sizeof(double));
                be.launch(n, MultiAxpy{G + (size_t)k * n, n, s - k, K.hdev.p, v, 0}); // v = r - sum c_i G_i
                applyPC(v, z);
                be.launch(n, MultiAxpy{U + (size_t)k * n, n, s - k, K.hdev.p, t, 1}); // t = sum c_i U_i
                be.launch(n, AxpyVec{z, om, t});
                double* Uk = U + (size_t)k * n;
                double* Gk = G + (size_t)k * n;
                be.d2d(Uk, t, (size_t)n * sizeof(double));
                matVecDev(Uk, Gk);
                st.nMatvec++;
                its++;
                // bi-orthogonalise against P_0..P_{k-1}.  The textbook loop (alpha_i = p_i.g / mu_ii; g -= alpha_i g_i; u -= alpha_i u_i, one
                // dot product and host round trip per i) is a forward substitution in disguise: P^T G is lower triangular (= M), so with
                // d = P^T g taken ONCE from the unmodified g, alpha solves M[0:k,0:k] alpha = d[0:k] and the dots of the updated g with
                // the remaining shadow vectors are d_i - sum_j alpha_j M_ij.  One multi-dot + two multi-axpys per application instead of
                // k dots + 2k axpys + k synchronisations; identical in exact arithmetic.
                {
                    const double* d = K.ops.dots(P, n, s, Gk, n);
                    std::vector<double> dd(d, d + s), al(k > 0 ? k : 1, 0.0);
                    for (int i = 0; i < k; i++)
                    {
                        double a = dd[i];
                        for (int j = 0; j < i; j++) a -= M[(size_t)i * s + j] * al[j];
                        al[i] = a / M[(size_t)i * s + i];
                    }
                    if (k > 0)
                    {
                        K.putCoeffs(be, al.data(), k);
                        be.launch(n, MultiAxpy{G, n, k, K.hdev.p, Gk, 0}); // Gk -= sum_i al_i G_i
                        be.launch(n, MultiAxpy{U, n, k, K.hdev.p, Uk, 0}); // Uk -= sum_i al_i U_i
                    }
                    for (int i = k; i < s; i++)
                    {
                        double a = dd[i];
                        for (int j = 0; j < k; j++) a -= M[(size_t)i * s + j] * al[j];
                        M[(size_t)i * s + k] = a;
                    }
                }
                const double mkk = M[(size_t)k * s + k];
                if (!(std::fabs(mkk) > 1e-300) || !std::isfinite(mkk)) { breakdown = true; break; }
                const double beta = f[k] / mkk;
                be.launch(n, AxpyVec{Gk, -beta, r});
                be.launch(n, AxpyVec{Uk, beta, K.xdev.p});
                rnorm = K.ops.norm2(r, n);
                for (int i = k + 1; i < s; i++) f[i] -= beta * M[(size_t)i * s + k];
                if (printInfo && (its % 50 == 0)) fprintf(stderr, "[dab200] IDR(%d) %4d  residual %.6e\n", s, its, rnorm);
            }
            if (!(rnorm > tol) || its >= gmresMaxIters || breakdown) break;
            // dimension-reduction step: r <- (I - om A M^-1) r with the "maintaining the convergence" choice of om
            applyPC(r, z);
            matVecDev(z, t);
            st.nMatvec++;
            its++;
            const double* d = K.ops.dots(r, n, 2, t, n);
            const double tr = d[0], tt = d[1];
            if (!(tt > 0.0)) { breakdown = true; break; }
            om = tr / tt;
            const double rho = tr / (std::sqrt(tt) * rnorm);
            if (std::fabs(rho) < 0.7 && rho != 0.0) om *= 0.7 / std::fabs(rho);
            if (om == 0.0 || !std::isfinite(om)) { breakdown = true; break; }
            be.launch(n, AxpyVec{t, -om, r});
            be.launch(n, AxpyVec{z, om, K.xdev.p});
            rnorm = K.ops.norm2(r, n);
        }
        // true residual
        matVecDev(K.xdev.p, r);
        st.nMatvec++;
        be.launch(n, SubVec{K.bdev.p, r});
        const double rtrue = K.ops.norm2(r, n);
        const bool recurrenceSaysDone = rnorm <= tol;
        rnorm = rtrue;
        if (rnorm <= tol * 1.0000001) reason = rnorm <= gmresRelTol * bnorm * 1.0000001 ? 2 : 3;
        else if (its >= gmresMaxIters) reason = -3;
        else if (!std::isfinite(rnorm)) reason = -9;
        else
        {
            nRestarts++; // drifted recurrence or breakdown: restart on the true residual
            if (nRestarts > 50) reason = recurrenceSaysDone ? -3 : -5;
        }
    }
    st.solveSec = timer.stopMs() * 1e-3;
    be.d2h(sol, K.xdev.p, (size_t)n * sizeof(double));
    st.nMatvec += kspExtraMatvecs;
    st.iterations = its;
    st.reason = reason;
    st.rn = rnorm;
    st.pcSec = K.pcSec;
    if (printInfo)
        fprintf(stderr, "[dab200] Main iteration %d IDR(%d) Residual norm %14.12e %.3f s (%d restarts)\n", its, s, rnorm, st.solveSec, nRestarts);
    const double absRatio = rnorm / gmresAbsTol;
    const double relRatio = bnorm > 0 ? rnorm / bnorm / gmresRelTol : 0.0;
    return (relRatio > gmresTolDiff && absRatio > gmresTolDiff) ? 1 : 0;
}

// runFPAdj / solveAdjointFP (pyDASolvers.pyx:412-416; reference DASimpleFoam::runFPAdj, DASimpleFoam.C:189-909): a stationary
// (fixed-point) adjoint iteration psi <- psi + omega M^-T (dFdW - J^T psi) with the reference's controls and termination rule --
// zero start, adjEqnOption.fpMaxIters / fpRelTol / fpMinResTolDiff, the L2 norms of the adjoint residual per state block (U, p, [T],
// [nuTilda], phi) normalised by their values after the first sweep, all below fpRelTol => 0, else the relaxed fpRelTol*fpMinResTolDiff
// check => 0, else 1.  The approximate inverse M^-1 here is the engine's multicolour ILU(0) of the first-order Jacobian with the
// damping adjEqnOption.fpOmega (default 0.5; 1.0 diverges), NOT the reference's transposed SIMPLE operators: it converges where that
// splitting is convergent (small and medium cases; at 1M cells it is not, DESIGN.md section 6) -- Krylov stays the production path.
inline int Solver::solveFixedPoint(const double* rhs, double* sol, KspStats& st)
{
    Krylov& K = kry;
    if (!K.pcValid && !(K.pcFactored && adjPCLag > 1 && K.symbolic)) calcPC();
    ensureRecorded();
    const int n = nDof(), nC = hm.nC;
    if (K.w.n < (size_t)n)
    {
        K.w.alloc(be, n);
        K.z.alloc(be, n);
    }
    K.xdev.alloc(be, n);
    K.bdev.alloc(be, n);
    K.ops.init(be, &comm, 34);
    be.h2d(K.bdev.p, rhs, (size_t)n * sizeof(double));
    // state blocks of the vector layout
    std::vector<std::pair<int, int>> blocks{{0, 3 * nC}, {3 * nC, nC}};
    int off = 4 * nC;
    if (par.comp) { blocks.push_back({off, nC}); off += nC; }
    if (par.turb) { blocks.push_back({off, nC}); off += nC; }
    blocks.push_back({off, n - off});
    const int nb = (int)blocks.size();
    std::vector<double> init(nb, 0.0), nrm(nb, 0.0);
    auto timer = be.timer();
    be.sync();
    timer.start();
    st.nMatvec = 0;
    kspExtraMatvecs = 0;
    st.r0 = K.ops.norm2(K.bdev.p, n);
    auto residual = [&]() {
        matVecDev(K.xdev.p, K.w.p);
        st.nMatvec++;
        be.launch(n, SubVec{K.bdev.p, K.w.p});
        for (int b = 0; b < nb; b++) nrm[b] = K.ops.norm2(K.w.p + blocks[b].first, blocks[b].second);
    };
    auto allBelow = [&](double tol) {
        for (int b = 0; b < nb; b++)
            if (init[b] > 0.0 && !(nrm[b] / init[b] < tol)) return false;
        return true;
    };
    int conv = 1, cnt = 0;
    for (; cnt < fpMaxIters; cnt++)
    {
        residual();
        if (cnt >= 1)
        {
            if (cnt == 1) init = nrm;
            if (printInfo && cnt % 50 == 0)
            {
                fprintf(stderr, "[dab200] fixed-point adjoint step %d, normalised residuals:", cnt);
                for (int b = 0; b < nb; b++) fprintf(stderr, " %.3e", init[b] > 0 ? nrm[b] / init[b] : 0.0);
                fprintf(stderr, "\n");
            }
            if (allBelow(fpRelTol)) { conv = 0; break; }
            bool finite = true;
            for (int b = 0; b < nb; b++) finite = finite && std::isfinite(nrm[b]);
            if (!finite) break;
        }
        applyIlu(K.w.p, K.z.p); // ILU only: the multiplicative coarse correction is not a contraction as a stationary sweep (measured)
        be.launch(n, AxpyVec{K.z.p, fpOmega, K.xdev.p});
    }
    if (conv == 1)
    {
        residual();
        if (cnt >= 1 && allBelow(fpRelTol * fpMinResTolDiff)) conv = 0; // "Adjoint is still considered successful"
    }
    double tot = 0.0;
    for (int b = 0; b < nb; b++) tot += nrm[b] * nrm[b];
    st.solveSec = timer.stopMs() * 1e-3;
    be.d2h(sol, K.xdev.p, (size_t)n * sizeof(double));
    st.nMatvec += kspExtraMatvecs;
    st.iterations = cnt;
    st.reason = conv == 0 ? 2 : -3;
    st.rn = std::sqrt(tot);
    st.pcSec = K.pcSec;
    return conv;
}

} // namespace dab
