// Domain decomposition of the host mesh: recursive coordinate bisection of the cell centres and
// extraction of one rank's sub-mesh with a one-cell ghost layer.  Replaces, for the adjoint hot path, the
// reference's `decomposePar` subprocess (scotch; reference dafoam/pyDAFoam.py:1454-1480, 597-604) and
// OpenFOAM's processor patches: cut faces stay *internal* faces of the local mesh whose other cell is a
// ghost cell appended after the owned cells, so the gather kernels run unchanged and every inter-rank
// dependency becomes a ghost-cell copy (DESIGN.md section 7).
#pragma once
#include "mesh.hpp"
#include <algorithm>
#include <numeric>
#include <cstdlib>

namespace dab
{

struct HaloPlan
{
    std::vector<int> peers;                    // neighbour ranks, ascending
    std::vector<std::vector<int32_t>> sendCells; // per peer: owned local cells the peer holds as ghosts
    std::vector<int> recvCellStart, recvCellCount; // per peer: contiguous ghost slots [start, start+count)
    std::vector<std::vector<int32_t>> sendFaces; // per peer: local faces whose phi this rank owns and the peer needs
    std::vector<std::vector<int32_t>> recvFaces; // per peer: local (foreign) faces filled from the peer
    // cyclic patches: per peer and send cell, the signed transform the value undergoes on the way (0: none; +k: R_k v; -k: R_k^T v)
    std::vector<std::vector<int32_t>> sendXf;
    // couplings of this rank with itself (both cells of a cyclic face pair owned here): plain local copies, same ordering rules
    std::vector<int32_t> selfSendCells, selfSendXf, selfSendFaces, selfRecvFaces;
    int selfRecvStart = 0, selfRecvCount = 0;
    bool hasSelf() const { return selfRecvCount > 0 || !selfRecvFaces.empty(); }
};

struct Partition
{
    int rank = 0, nRanks = 1;
    int64_t nGlobalCells = 0;
    std::vector<int32_t> cellGlobal; // local (owned + ghost) -> global cell
    std::vector<int32_t> faceGlobal; // local face -> global face
    std::vector<uint8_t> faceOwned;  // 1 if the phi DOF of the local face belongs to this rank
    std::vector<int32_t> faceXf;     // k > 0: the local face is the neighbour-side copy of a face of cyclic transform k (geometry in that frame)
    HaloPlan halo;
};

// recursive coordinate bisection: part[c] in [0, nParts)
inline void rcbPartition(const HostMesh& g, int nParts, std::vector<int>& part)
{
    part.assign(g.nC, 0);
    std::vector<int> idx(g.nC);
    std::iota(idx.begin(), idx.end(), 0);
    struct Job { int lo, hi, p0, np; };
    std::vector<Job> stack{{0, g.nC, 0, nParts}};
    while (!stack.empty())
    {
        Job j = stack.back();
        stack.pop_back();
        if (j.np == 1)
        {
            for (int i = j.lo; i < j.hi; i++) part[idx[i]] = j.p0;
            continue;
        }
        double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
        for (int i = j.lo; i < j.hi; i++)
            for (int k = 0; k < 3; k++)
            {
                mn[k] = std::min(mn[k], g.C[k][idx[i]]);
                mx[k] = std::max(mx[k], g.C[k][idx[i]]);
            }
        int ax = 0;
        for (int k = 1; k < 3; k++)
            if (mx[k] - mn[k] > mx[ax] - mn[ax]) ax = k;
        const int npL = j.np / 2, npR = j.np - npL;
        const int mid = j.lo + (int)((int64_t)(j.hi - j.lo) * npL / j.np);
        std::nth_element(idx.begin() + j.lo, idx.begin() + mid, idx.begin() + j.hi,
                         [&](int a, int b) { return g.C[ax][a] < g.C[ax][b] || (g.C[ax][a] == g.C[ax][b] && a < b); });
        stack.push_back({j.lo, mid, j.p0, npL});
        stack.push_back({mid, j.hi, j.p0 + npL, npR});
    }
}

// build the local mesh of `rank` from the global mesh (geometry and wall distance already computed)
//
// Cyclic faces (g.cyc[f] = k > 0, mesh.hpp) are cut faces as well, also when both cells belong to this rank: the owner-side cell sees
// the neighbour as a ghost holding the neighbour's values transformed by +k, the neighbour-side cell sees the owner as a ghost
// transformed by -k, and the face appears twice in the local mesh -- once with the owner's geometry and the phi state (type B), once
// in the neighbour's frame as a foreign face filled by the face exchange (type D).  Reference role: cyclicFvPatchField::
// patchNeighbourField + the `transform()` of coupled patches inside every fvc:: operator; coupled-face indexing DAIndex.C:151-167.
inline void extractLocalMesh(const HostMesh& g, const std::vector<int>& part, int rank, int nRanks, HostMesh& l, Partition& P)
{
    P.rank = rank;
    P.nRanks = nRanks;
    P.nGlobalCells = g.nC;
    const bool anyCyc = g.hasCyclic();
    auto cycOf = [&](int f) { return anyCyc ? g.cyc[f] : 0; };
    std::vector<int32_t> g2l(g.nC, -1);
    // owned cells: first the interior ones (no ghost neighbour), then the ones along the cuts, each group
    // in global order -- kernels can then run the interior range while the ghost exchange is in flight
    std::vector<uint8_t> onCut(g.nC, 0);
    for (int f = 0; f < g.nIF; f++)
        if (part[g.own[f]] != part[g.nei[f]] || cycOf(f) != 0)
        {
            onCut[g.own[f]] = 1;
            onCut[g.nei[f]] = 1;
        }
    int nC = 0;
    for (int pass = 0; pass < 2; pass++)
    {
        for (int c = 0; c < g.nC; c++)
            if (part[c] == rank && onCut[c] == pass)
            {
                g2l[c] = nC++;
                P.cellGlobal.push_back(c);
            }
        if (pass == 0) l.nInterior = nC;
    }
    // ghost cells: (source rank, transform, global id); grouped by rank (this rank's own cyclic images last), then transform, then id
    struct Key
    {
        int q, xs, c;
        bool operator<(const Key& o) const { return q != o.q ? q < o.q : (xs != o.xs ? xs < o.xs : c < o.c); }
        bool operator==(const Key& o) const { return q == o.q && xs == o.xs && c == o.c; }
    };
    auto rankKey = [&](int q) { return q == rank ? nRanks : q; }; // self sorts after every peer
    std::vector<Key> ghosts, sends; // sends: (destination rank, transform at the receiver, my global cell)
    for (int f = 0; f < g.nIF; f++)
    {
        const int a = g.own[f], b = g.nei[f], k = cycOf(f);
        if (k == 0)
        {
            if (part[a] == rank && part[b] != rank) { ghosts.push_back({rankKey(part[b]), 0, b}); sends.push_back({rankKey(part[b]), 0, a}); }
            if (part[b] == rank && part[a] != rank) { ghosts.push_back({rankKey(part[a]), 0, a}); sends.push_back({rankKey(part[a]), 0, b}); }
        }
        else
        {
            if (part[a] == rank) { ghosts.push_back({rankKey(part[b]), +k, b}); sends.push_back({rankKey(part[b]), -k, a}); }
            if (part[b] == rank) { ghosts.push_back({rankKey(part[a]), -k, a}); sends.push_back({rankKey(part[a]), +k, b}); }
        }
    }
    std::sort(ghosts.begin(), ghosts.end());
    ghosts.erase(std::unique(ghosts.begin(), ghosts.end()), ghosts.end());
    std::sort(sends.begin(), sends.end());
    sends.erase(std::unique(sends.begin(), sends.end()), sends.end());
    int nT = nC;
    std::vector<int> ghostXs; // per ghost (index - nC)
    auto ghostSlot = [&](int q, int xs, int c) {
        const Key key{rankKey(q), xs, c};
        return nC + (int)(std::lower_bound(ghosts.begin(), ghosts.end(), key) - ghosts.begin());
    };
    P.halo.selfRecvStart = nC;
    for (const Key& gk : ghosts)
    {
        if (gk.q == nRanks)
        {
            if (P.halo.selfRecvCount == 0) P.halo.selfRecvStart = nT;
            P.halo.selfRecvCount++;
        }
        else
        {
            if (P.halo.peers.empty() || P.halo.peers.back() != gk.q)
            {
                P.halo.peers.push_back(gk.q);
                P.halo.recvCellStart.push_back(nT);
                P.halo.recvCellCount.push_back(0);
            }
            P.halo.recvCellCount.back()++;
        }
        nT++;
        P.cellGlobal.push_back(gk.c);
        ghostXs.push_back(gk.xs);
    }
    const int nPeers = (int)P.halo.peers.size();
    auto peerIndex = [&](int q) { return (int)(std::lower_bound(P.halo.peers.begin(), P.halo.peers.end(), q) - P.halo.peers.begin()); };
    // cells to send, in the order the receiver lists its ghosts (transform, then global id)
    P.halo.sendCells.assign(nPeers, {});
    P.halo.sendXf.assign(nPeers, {});
    for (const Key& sk : sends)
    {
        if (sk.q == nRanks)
        {
            P.halo.selfSendCells.push_back(g2l[sk.c]);
            P.halo.selfSendXf.push_back(sk.xs);
        }
        else
        {
            P.halo.sendCells[peerIndex(sk.q)].push_back(g2l[sk.c]);
            P.halo.sendXf[peerIndex(sk.q)].push_back(sk.xs);
        }
    }
    // faces: A (both owned, not cyclic), B (owner mine, neighbour ghost), D (owner ghost, neighbour mine), then boundary by patch
    std::vector<int> fa, fb, fd;
    for (int f = 0; f < g.nIF; f++)
    {
        const bool oa = part[g.own[f]] == rank, ob = part[g.nei[f]] == rank;
        if (cycOf(f) != 0)
        {
            if (oa) fb.push_back(f);
            if (ob) fd.push_back(f);
        }
        else if (oa && ob) fa.push_back(f);
        else if (oa) fb.push_back(f);
        else if (ob) fd.push_back(f);
    }
    std::vector<int> lf(fa);
    lf.insert(lf.end(), fb.begin(), fb.end());
    lf.insert(lf.end(), fd.begin(), fd.end());
    const int nIF = (int)lf.size();
    const int nA = (int)fa.size(), nB = (int)fb.size();
    l.patches.clear();
    for (size_t p = 0; p < g.patches.size(); p++)
    {
        PatchDef pd = g.patches[p];
        const int start = (int)lf.size();
        for (int i = 0; i < g.patches[p].size; i++)
        {
            const int f = g.patches[p].start + i;
            if (part[g.own[f]] == rank) lf.push_back(f);
        }
        pd.start = start;
        pd.size = (int)lf.size() - start;
        l.patches.push_back(pd);
    }
    const int nF = (int)lf.size();
    P.faceGlobal.assign(lf.begin(), lf.end());
    P.faceOwned.assign(nF, 1);
    P.halo.sendFaces.assign(nPeers, {});
    P.halo.recvFaces.assign(nPeers, {});
    for (int i = nA; i < nIF; i++)
    {
        const int f = lf[i];
        const int ra = part[g.own[f]], rb = part[g.nei[f]];
        if (i < nA + nB)
        {
            // B: ascending global id
            if (rb == rank) P.halo.selfSendFaces.push_back(i);
            else P.halo.sendFaces[peerIndex(rb)].push_back(i);
        }
        else
        {
            // D: ascending global id
            P.faceOwned[i] = 0;
            if (ra == rank) P.halo.selfRecvFaces.push_back(i);
            else P.halo.recvFaces[peerIndex(ra)].push_back(i);
        }
    }
    // topology
    l.points = g.points;
    l.nP = g.nP;
    l.nF = nF; l.nIF = nIF; l.nBF = nF - nIF; l.nC = nC; l.nCtot = nT;
    l.own.resize(nF);
    l.nei.resize(nIF);
    l.fOff.assign(1, 0);
    l.fLab.clear();
    for (int i = 0; i < nF; i++)
    {
        const int f = lf[i];
        const int k = i < nIF ? cycOf(f) : 0;
        if (i < nA || i >= nIF)
        {
            l.own[i] = g2l[g.own[f]];
            if (i < nIF) l.nei[i] = g2l[g.nei[f]];
        }
        else if (i < nA + nB)
        {
            l.own[i] = g2l[g.own[f]];
            l.nei[i] = ghostSlot(part[g.nei[f]], k, g.nei[f]);
        }
        else
        {
            l.own[i] = ghostSlot(part[g.own[f]], -k, g.own[f]);
            l.nei[i] = g2l[g.nei[f]];
        }
        for (int q = g.fOff[f]; q < g.fOff[f + 1]; q++) l.fLab.push_back(g.fLab[q]);
        l.fOff.push_back((int32_t)l.fLab.size());
    }
    l.xforms = g.xforms;
    l.cycAOff = g.cycAOff; l.cycA = g.cycA; l.cycBOff = g.cycBOff; l.cycB = g.cycB; l.cycXf = g.cycXf;
    P.faceXf.assign(nF, 0);
    for (int i = nA + nB; i < nIF; i++) P.faceXf[i] = cycOf(lf[i]);
    l.patchGeom = g.patchGeom;
    l.bPatch.assign(l.nBF, -1);
    for (size_t p = 0; p < l.patches.size(); p++)
        for (int i = 0; i < l.patches[p].size; i++) l.bPatch[l.patches[p].start - nIF + i] = (int32_t)p;
    // ELL cell -> faces for the owned cells
    std::vector<int> cnt(nC, 0);
    for (int i = 0; i < nF; i++)
    {
        if (l.own[i] < nC) cnt[l.own[i]]++;
        if (i < nIF && l.nei[i] < nC) cnt[l.nei[i]]++;
    }
    l.maxCF = nC ? *std::max_element(cnt.begin(), cnt.end()) : 0;
    l.cellFaces.assign((size_t)l.maxCF * nC, -1);
    std::fill(cnt.begin(), cnt.end(), 0);
    // ascending local face id, boundary ids >= nIF (cut faces are internal faces with a ghost neighbour): every row is
    // [internal..., boundary..., -1 padding], the order RevB's two passes over a row rely on
    for (int i = 0; i < nF; i++)
    {
        if (l.own[i] < nC) l.cellFaces[(size_t)cnt[l.own[i]]++ * nC + l.own[i]] = (i << 1);
        if (i < nIF && l.nei[i] < nC) l.cellFaces[(size_t)cnt[l.nei[i]]++ * nC + l.nei[i]] = (i << 1) | 1;
    }
    l.checkEllOrder();
    // geometry slices
    for (int k = 0; k < 3; k++)
    {
        l.Sf[k].resize(nF); l.Cf[k].resize(nF); l.corr[k].resize(nF); l.C[k].resize(nT);
    }
    l.magSf.resize(nF); l.w.resize(nF); l.delta.resize(nF); l.V.resize(nT); l.yWall.resize(nT);
    for (int i = 0; i < nF; i++)
    {
        const int f = lf[i];
        double sf[3] = {g.Sf[0][f], g.Sf[1][f], g.Sf[2][f]}, cf[3] = {g.Cf[0][f], g.Cf[1][f], g.Cf[2][f]};
        double co[3] = {g.corr[0][f], g.corr[1][f], g.corr[2][f]};
        if (i >= nA + nB && i < nIF && cycOf(f) != 0)
        {
            // the neighbour-side copy of a cyclic face: geometry in the neighbour's frame
            const HostMesh::CycXf& X = g.xforms[cycOf(f) - 1];
            const double s0[3] = {sf[0], sf[1], sf[2]}, c0[3] = {cf[0], cf[1], cf[2]}, o0[3] = {co[0], co[1], co[2]};
            HostMesh::xfVector(X, true, s0, sf);
            HostMesh::xfPoint(X, true, c0, cf);
            HostMesh::xfVector(X, true, o0, co);
        }
        for (int k = 0; k < 3; k++) { l.Sf[k][i] = sf[k]; l.Cf[k][i] = cf[k]; l.corr[k][i] = co[k]; }
        l.magSf[i] = g.magSf[f]; l.w[i] = g.w[f]; l.delta[i] = g.delta[f];
    }
    for (int c = 0; c < nT; c++)
    {
        const int gc = P.cellGlobal[c];
        double cc[3] = {g.C[0][gc], g.C[1][gc], g.C[2][gc]};
        const int xs = c >= nC ? ghostXs[c - nC] : 0;
        if (xs != 0)
        {
            const double c0[3] = {cc[0], cc[1], cc[2]};
            HostMesh::xfPoint(g.xforms[std::abs(xs) - 1], xs < 0, c0, cc);
        }
        for (int k = 0; k < 3; k++) l.C[k][c] = cc[k];
        l.V[c] = g.V[gc];
        l.yWall[c] = g.yWall[gc];
    }
}

} // namespace dab
