// CTA-resident ("tile") kernels of the transpose product y = diag(n) (dR/dW)^T x  (reference role:
// DASolver::dRdWTMatVecMultFunction, DASolver.C:1364-1409).  Same arithmetic as the cell-per-thread kernels -- the cell
// functions of rev_kernels.hpp, instantiated with a tile accessor -- with a different data path:
//
//   * one CTA owns a tile (tiles.hpp): a contiguous range of cells plus its halo rings;
//   * phase 0 stages every per-cell array a stage reads through a *neighbour* index into shared memory: the tile part is a
//     contiguous range (coalesced, sector-exact), the halo part a short gather through the tile's cell list;
//   * the stages then run from shared memory under tile-local indices; face arrays (read once per side, no reuse inside
//     a stage beyond what L1 gives) stay in global memory;
//   * ProdTileBC fuses RevB and RevC: RevB is evaluated on the tile and its first ring (the ring only for the gradient
//     adjoints RevC gathers), so the 17 doubles per cell that RevB hands to RevC never travel through HBM.
//
// HBM-bound fp64 gathers: no tensor cores.  The host build (DAB_HOSTSIM, tests only) runs the same phases tile by tile.
#pragma once
#include "rev_kernels.hpp"
#include "tiles.hpp"

namespace dab
{

// capacities compiled into the tile kernels (doubles per array are EXT*, shared memory is static per program)
constexpr int TILE_TMAX = 192; // cells per tile (= threads per CTA: 6 warps)
constexpr int TILE_EXT1 = 256; // tile + ring 1
constexpr int TILE_EXT2 = 320; // tile + rings 1, 2   (ProdTileBC: 101 888 B of shared memory -> 2 CTAs per SM)

// shared base of the tile accessors: topology of the current tile + face data from global memory
struct TAccBase
{
    MeshView m;     // face arrays / patch table (global ids); the per-cell pointers of this view are NOT used
    StateView s;    // global state (phi by face id; cell arrays only for own-cell reads by global id)
    PsiView x;      // global input vector
    double* sm;     // shared memory of the CTA
    const int32_t *tf, *tn; // this tile's local tables [maxCF][ln]
    int ln, c0, maxCF_;
    DAB_HD int maxCF() const { return maxCF_; }
    DAB_HD int nIF() const { return m.nIF; }
    DAB_HD FaceRef face(int c, int k) const { return faceOfE2(m.nIF, tf[(size_t)k * ln + c], tn[(size_t)k * ln + c]); }
    template <int NF>
    DAB_HD void faceRow(int c, int* e, int* n) const
    {
        _Pragma("unroll") for (int k = 0; k < NF; k++)
        {
            e[k] = tf[(size_t)k * ln + c];
            n[k] = tn[(size_t)k * ln + c];
        }
    }
    DAB_HD bool ghost(int) const { return false; } // tiles run on one GPU
    DAB_HD int patch(int f) const { return m.bPatch[f - m.nIF]; }
    DAB_HD void Sf(int f, double* v) const { v[0] = m.Sx[f]; v[1] = m.Sy[f]; v[2] = m.Sz[f]; }
    DAB_HD void kv(int f, double* v) const { v[0] = m.kx[f]; v[1] = m.ky[f]; v[2] = m.kz[f]; }
    DAB_HD void faceOff(int f, double* dO, double* dN) const { faceOffsets(m, f, dO, dN); }
    DAB_HD double magSf(int f) const { return m.magSf[f]; }
    DAB_HD double w(int f) const { return m.w[f]; }
    DAB_HD double delta(int f) const { return m.delta[f]; }
    DAB_HD double phi(int f) const { return s.phi[f]; }
    DAB_HD double xphi(int f) const { return x.phi[f]; }
    DAB_HD bool mrfCell(int) const { return false; }
    DAB_HD bool bcRefOn(int) const { return false; }
    DAB_HD bool bcRefAny() const { return false; }
    DAB_HD void setBcRef(int, int, double) const {}
    DAB_HD void addBcRef(int, int, double) const {}
};

// ---- RevA on a tile: neighbour-read arrays (x.p, V, grad p, p, rAU) in shared memory over tile + ring 1 -------------------
struct TAccA : TAccBase
{
    static constexpr int E1 = TILE_EXT1;
    enum { O_XP = 0, O_V = E1, O_GP = 2 * E1, O_P = 5 * E1, O_RAU = 6 * E1, SM_DOUBLES = 7 * E1 };
    RecordView r; // global record (own-cell reads)
    AdjView a;    // global reverse intermediates (outputs)
    int nTg, nCg; // global strides
    DAB_HD double V(int c) const { return sm[O_V + c]; }
    DAB_HD double xp(int c) const { return sm[O_XP + c]; }
    DAB_HD double gP(int c, int i) const { return sm[O_GP + i * E1 + c]; }
    DAB_HD double p(int c) const { return sm[O_P + c]; }
    DAB_HD double rAU(int c) const { return sm[O_RAU + c]; }
    // own-cell values straight from global memory (tile cells: c0 + c, coalesced)
    DAB_HD double U(int c, int j) const { return s.U[3 * (size_t)(c0 + c) + j]; }
    DAB_HD double xU(int c, int j) const { return x.U[3 * (size_t)(c0 + c) + j]; }
    DAB_HD double HbyA(int c, int j) const { return r.HbyA[(size_t)j * nTg + c0 + c]; }
    DAB_HD double D0(int c) const { return r.D0[c0 + c]; }
    DAB_HD void setMt(int c, int j, double v) const { a.mt[(size_t)j * nTg + c0 + c] = v; }
    DAB_HD void setDn(int c, double v) const { a.Dn[c0 + c] = v; }
    DAB_HD void setUdir(int c, int j, double v) const { a.Udir[(size_t)j * nCg + c0 + c] = v; }
    DAB_HD void setPdir(int c, double v) const { a.pdir[c0 + c] = v; }
    DAB_HD void setGPb(int c, int i, double v) const { a.gPb[(size_t)i * nTg + c0 + c] = v; }
};

template <int NF>
struct ProdTileA
{
    static constexpr int THREADS = TILE_TMAX;
    static constexpr int MAXREG = 80;
    static constexpr int PHASES = 2;
    static constexpr int SM_DOUBLES = TAccA::SM_DOUBLES;
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    AdjView a;
    PsiView x;
    TileView tv;
    DAB_HD void phase(int ph, int t, int tid, int nthr, double* sm) const
    {
        constexpr int E1 = TILE_EXT1;
        const int32_t* cum = tv.cum + (size_t)t * (tv.R + 1);
        const int n0 = cum[0], n1 = cum[1];
        const int c0 = t * tv.T;
        const int nTg = m.nCtot;
        if (ph == 0)
        {
            const int32_t* gid = tv.gid + (size_t)t * tv.ls;
            for (int l = tid; l < n1; l += nthr)
            {
                const int g = l < n0 ? c0 + l : gid[l];
                sm[TAccA::O_XP + l] = x.p[g];
                sm[TAccA::O_V + l] = m.V[g];
                for (int i = 0; i < 3; i++) sm[TAccA::O_GP + i * E1 + l] = r.gP[(size_t)i * nTg + g];
                sm[TAccA::O_P + l] = s.p[g];
                sm[TAccA::O_RAU + l] = r.rAU[g];
            }
            return;
        }
        TAccA A;
        A.m = m; A.s = s; A.x = x; A.sm = sm;
        A.tf = tv.tf + (size_t)t * tv.maxCF * tv.ln;
        A.tn = tv.tn + (size_t)t * tv.maxCF * tv.ln;
        A.ln = tv.ln; A.c0 = c0; A.maxCF_ = tv.maxCF;
        A.r = r; A.a = a; A.nTg = nTg; A.nCg = m.nC;
        for (int l = tid; l < n0; l += nthr) revACell<NF>(A, q, l);
    }
};

// ---- RevB + RevC on a tile ------------------------------------------------------------------------------------------------
struct TAccBC : TAccBase
{
    static constexpr int E1 = TILE_EXT1, E2 = TILE_EXT2, TM = TILE_TMAX;
    // tile + rings 1, 2 (read through a neighbour index by RevB on the tile and ring 1)
    enum
    {
        O_U = 0, O_NUT = 3 * E2, O_MT = 4 * E2, O_DN = 7 * E2, O_FLAG = 8 * E2, O_GU = 9 * E2, O_NT = 18 * E2, O_XNT = 19 * E2,
        O_V = 20 * E2, O_GNT = 21 * E2, END2 = 24 * E2,
        // tile + ring 1 (RevC reads the gradient adjoints of the neighbours)
        O_GPB = END2, O_GUB = END2 + 3 * E1, O_GNTB = END2 + 12 * E1, O_YW = END2 + 15 * E1, END1 = END2 + 16 * E1,
        // tile only (RevB -> RevC of the same cell)
        O_U2 = END1, O_NT2 = END1 + 3 * TM, O_NUTB = END1 + 4 * TM, SM_DOUBLES = END1 + 5 * TM
    };
    AdjView a;    // global: Udir, pdir of RevA (own-cell reads)
    double *yU, *yP, *yN, *yPhi;
    int nCg;
    DAB_HD double U(int c, int j) const { return sm[O_U + j * E2 + c]; }
    DAB_HD double nut(int c) const { return sm[O_NUT + c]; }
    DAB_HD double mt(int c, int j) const { return sm[O_MT + j * E2 + c]; }
    DAB_HD double Dn(int c) const { return sm[O_DN + c]; }
    DAB_HD double flag(int c) const { return sm[O_FLAG + c]; }
    DAB_HD double gU(int c, int i) const { return sm[O_GU + i * E2 + c]; }
    DAB_HD double nt(int c) const { return sm[O_NT + c]; }
    DAB_HD double xnt(int c) const { return sm[O_XNT + c]; }
    DAB_HD double V(int c) const { return sm[O_V + c]; }
    DAB_HD double gNt(int c, int i) const { return sm[O_GNT + i * E2 + c]; }
    DAB_HD double yWall(int c) const { return sm[O_YW + c]; }
    DAB_HD double gPb(int c, int i) const { return sm[O_GPB + i * E1 + c]; }
    DAB_HD double gUb(int c, int i) const { return sm[O_GUB + i * E1 + c]; }
    DAB_HD double gNtb(int c, int i) const { return sm[O_GNTB + i * E1 + c]; }
    DAB_HD double U2(int c, int j) const { return sm[O_U2 + j * TM + c]; }
    DAB_HD double nt2(int c) const { return sm[O_NT2 + c]; }
    DAB_HD double nutb(int c) const { return sm[O_NUTB + c]; }
    DAB_HD void setGUb(int c, int i, double v) const { sm[O_GUB + i * E1 + c] = v; }
    DAB_HD void setGNtb(int c, int i, double v) const { sm[O_GNTB + i * E1 + c] = v; }
    DAB_HD void setU2(int c, int j, double v) const { sm[O_U2 + j * TM + c] = v; }
    DAB_HD void setNt2(int c, double v) const { sm[O_NT2 + c] = v; }
    DAB_HD void setNutb(int c, double v) const { sm[O_NUTB + c] = v; }
    // own-cell reads / product rows by global id (tile cells)
    DAB_HD double Udir(int c, int j) const { return a.Udir[(size_t)j * nCg + c0 + c]; }
    DAB_HD double pdir(int c) const { return a.pdir[c0 + c]; }
    DAB_HD void setYU(int c, int j, double v) const { yU[3 * (size_t)(c0 + c) + j] = v; }
    DAB_HD void setYP(int c, double v) const { yP[c0 + c] = v; }
    DAB_HD void setYN(int c, double v) const { yN[c0 + c] = v; }
    DAB_HD void setYPhi(int f, double v) const { yPhi[f] = v; }
};

template <int NF, int FEAT>
struct ProdTileBC
{
    static constexpr int THREADS = TILE_TMAX;
    static constexpr int MAXREG = 168; // 2 CTAs x 6 warps x 168 registers = 63 K of the SM's 64 K
    static constexpr int PHASES = 3;
    static constexpr int SM_DOUBLES = TAccBC::SM_DOUBLES;
    MeshView m;
    Params q;
    StateView s;
    RecordView r;
    AdjView a;
    PsiView x;
    double* y;
    TileView tv;
    DAB_HD void phase(int ph, int t, int tid, int nthr, double* sm) const
    {
        constexpr int E1 = TILE_EXT1, E2 = TILE_EXT2;
        const int32_t* cum = tv.cum + (size_t)t * (tv.R + 1);
        const int n0 = cum[0], n1 = cum[1], n2 = cum[2];
        const int c0 = t * tv.T;
        const int nTg = m.nCtot;
        if (ph == 0)
        {
            const int32_t* gid = tv.gid + (size_t)t * tv.ls;
            for (int l = tid; l < n2; l += nthr)
            {
                const int g = l < n0 ? c0 + l : gid[l];
                for (int j = 0; j < 3; j++) sm[TAccBC::O_U + j * E2 + l] = s.U[3 * (size_t)g + j];
                sm[TAccBC::O_NUT + l] = r.nut[g];
                for (int j = 0; j < 3; j++) sm[TAccBC::O_MT + j * E2 + l] = a.mt[(size_t)j * nTg + g];
                sm[TAccBC::O_DN + l] = a.Dn[g];
                sm[TAccBC::O_FLAG + l] = r.flag[g];
                for (int i = 0; i < 9; i++) sm[TAccBC::O_GU + i * E2 + l] = r.gU[(size_t)i * nTg + g];
                sm[TAccBC::O_NT + l] = q.turb ? s.nt[g] : 0.0;
                sm[TAccBC::O_XNT + l] = q.turb ? x.nt[g] : 0.0;
                sm[TAccBC::O_V + l] = m.V[g];
                for (int i = 0; i < 3; i++) sm[TAccBC::O_GNT + i * E2 + l] = q.turb ? r.gNt[(size_t)i * nTg + g] : 0.0;
                if (l < n1)
                {
                    for (int i = 0; i < 3; i++) sm[TAccBC::O_GPB + i * E1 + l] = a.gPb[(size_t)i * nTg + g];
                    sm[TAccBC::O_YW + l] = m.yWall[g];
                }
            }
            return;
        }
        TAccBC A;
        A.m = m; A.s = s; A.x = x; A.sm = sm;
        A.tf = tv.tf + (size_t)t * tv.maxCF * tv.ln;
        A.tn = tv.tn + (size_t)t * tv.maxCF * tv.ln;
        A.ln = tv.ln; A.c0 = c0; A.maxCF_ = tv.maxCF;
        A.a = a; A.nCg = m.nC;
        const size_t nC = m.nC;
        A.yU = y; A.yP = y + 3 * nC; A.yN = y + 4 * nC; A.yPhi = y + (size_t)(q.turb ? 5 : 4) * nC;
        if (ph == 1)
        {
            // RevB: the tile's cells in full, the first ring for the gradient adjoints only
            for (int l = tid; l < n1; l += nthr) revBCell<NF, FEAT>(A, q, l, l >= n0);
            return;
        }
        for (int l = tid; l < n0; l += nthr) revCCell<NF>(A, q, l, 0);
    }
};

} // namespace dab
