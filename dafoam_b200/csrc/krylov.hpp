// On-device Krylov machinery replacing the reference's PETSc objects for the adjoint solve:
//   * dRdWTPC in "level-grouped ELL": rows ordered (cell colour, DOF slot, cell) so that every
//     (colour, slot) group is a contiguous, mutually independent row range stored column-major
//     (coalesced), replacing the PETSc AIJ Mat filled by DAPartDeriv::calcPartDerivMat
//     (reference src/adjoint/DAPartDeriv/DAPartDeriv.C:350-474) with DAJacCon connectivity levels
//     (reference src/adjoint/DAJacCon/DAJacCon.C:2039+) and DAColoring (reference DAColoring.C:32-784);
//   * ILU(0) factorisation and triangular solves, one kernel per cell colour, replacing
//     PCASM+PCILU (reference src/adjoint/DALinearEqn/DALinearEqn.C:142-310).  PETSc's RCM ordering gives
//     O(ni+nj) dependent wavefronts; the multicolour ordering gives ~10 fully parallel levels, which is
//     what keeps the triangular solves bandwidth-bound on a GPU;
//   * restarted GMRES, right preconditioning, unpreconditioned residual norm, classical Gram-Schmidt
//     with refinement if needed (reference DALinearEqn.C:74-140, 313-324).
#pragma once
#include "backend.hpp"
#include "views.hpp"
#include "comm.hpp"
#include <atomic>
#include <cmath>
#include <thread>
#include <cstdint>
#include <vector>

namespace dab
{

struct KspStats
{
    int iterations = 0, reason = 0;
    double r0 = 0, rn = 0, solveSec = 0, pcSec = 0;
    int nMatvec = 0;
};

// ---- device view of the level-grouped ELL matrix -------------------------------------------------------
struct EllView
{
    int n;
    const int64_t* rowBase;  // [n] offset of entry 0 of the row
    const int32_t* rowStride; // [n] distance between consecutive entries of the row (= rows in its group)
    const int32_t* rowLen;   // [n]
    const int32_t* diag;     // [n] entry index of the diagonal
    const int32_t* col;      // ELL columns (new numbering), -1 padding
    double* val;
    const float* valF = nullptr; // fp32 copy of the FACTORS (adjEqnOption.pcStorage "fp32"): what the triangular solves read
};

// one colour of the ordering: `nCells` cells, slot s occupies rows [slotStart[s], slotStart[s]+slotCount[s])
constexpr int MAXSLOT = 16;
struct ColourView
{
    int nCells, nSlots;
    int slotStart[MAXSLOT];
    int slotCount[MAXSLOT];
    long long slotBase[MAXSLOT]; // ELL offset of entry 0 of the slot's first row (the slot's rows are contiguous; entry stride = slotCount)
};

// ---- FD assembly -----------------------------------------------------------------------------------------
struct StatePtrs
{
    double *U, *p, *nt, *phi;
    int nC, turb;
    const double* magSf;
    double sU, sP, sNut, sPhi;
    int phiNorm = 1; // "phi" listed in normalizeStates: the FD perturbation of a face flux is scaled by |Sf| (DAPartDeriv.C:284-310), else by 1
    double* T = nullptr; // compressible: [U | p | T | nuTilda | phi]
    double sT = 1.0;
    DAB_HD double* at(int ext, double& scale) const
    {
        if (ext < 3 * nC) { scale = sU; return U + ext; }
        ext -= 3 * nC;
        if (ext < nC) { scale = sP; return p + ext; }
        ext -= nC;
        if (T)
        {
            if (ext < nC) { scale = sT; return T + ext; }
            ext -= nC;
        }
        if (turb)
        {
            if (ext < nC) { scale = sNut; return nt + ext; }
            ext -= nC;
        }
        scale = phiNorm ? sPhi * magSf[ext] : 1.0;
        return phi + ext;
    }
};

struct FdPerturb
{
    StatePtrs sp;
    const int32_t* list; // external state indices of this FD colour
    double eps;          // signed step
    DAB_HD void operator()(int i) const
    {
        double sc;
        double* q = sp.at(list[i], sc);
        *q += eps * sc;
    }
};

// A[row(state j)][col(residual r)] = (R1[r] - R0[r]) / eps
struct FdFill
{
    EllView A;
    const int32_t* list;  // external state indices of this FD colour
    const int32_t* iperm; // ext -> new
    const int32_t* perm;  // new -> ext
    const double *R0, *R1;
    double ieps;
    DAB_HD void operator()(int t) const
    {
        const int i = iperm[list[t]];
        const int64_t base = A.rowBase[i];
        const int64_t st = A.rowStride[i];
        const int len = A.rowLen[i];
        for (int e = 0; e < len; e++)
        {
            const int r = perm[A.col[base + e * st]];
            A.val[base + e * st] = (R1[r] - R0[r]) * ieps;
        }
    }
};

// ---- ILU(0) ---------------------------------------------------------------------------------------------
DAB_HD int ellFind(const EllView& A, int i, int j)
{
    const int64_t base = A.rowBase[i], st = A.rowStride[i];
    int lo = 0, hi = A.rowLen[i] - 1;
    while (lo <= hi)
    {
        const int mid = (lo + hi) >> 1;
        const int c = A.col[base + mid * st];
        if (c == j) return mid;
        if (c < j) lo = mid + 1;
        else hi = mid - 1;
    }
    return -1;
}

struct IluFactorColour
{
    EllView A;
    ColourView cv;
    double shift; // relative pivot guard (MAT_SHIFT_NONZERO role, reference DALinearEqn.C:262-264)
    DAB_HD void operator()(int t) const
    {
        for (int s = 0; s < cv.nSlots; s++)
        {
            if (t >= cv.slotCount[s]) break;
            const int i = cv.slotStart[s] + t;
            const int64_t bi = A.rowBase[i], si = A.rowStride[i];
            const int len = A.rowLen[i], di = A.diag[i];
            double rowMax = 0.0;
            for (int e = 0; e < len; e++)
            {
                const double v = fabs(A.val[bi + e * si]);
                rowMax = v > rowMax ? v : rowMax;
            }
            for (int e = 0; e < di; e++)
            {
                const int k = A.col[bi + e * si];
                const int64_t bk = A.rowBase[k], sk = A.rowStride[k];
                const int dk = A.diag[k], lk = A.rowLen[k];
                const double lik = A.val[bi + e * si] * A.val[bk + dk * sk]; // finished rows hold 1 / u_kk
                A.val[bi + e * si] = lik;
                if (lik == 0.0) continue;
                // both rows are sorted by column: one merge pass over (upper part of row k, row i right of entry e) instead of a binary
                // search in row i per entry of row k (1.64 s of the 5.7 s set-up at 1M cells went into this kernel)
                int pj = e + 1;
                for (int q = dk + 1; q < lk && pj < len; q++)
                {
                    const int j = A.col[bk + q * sk];
                    while (pj < len && A.col[bi + pj * si] < j) pj++;
                    if (pj < len && A.col[bi + pj * si] == j) A.val[bi + pj * si] -= lik * A.val[bk + q * sk];
                }
            }
            double d = A.val[bi + di * si];
            if (!(fabs(d) > shift * rowMax)) d = (d < 0.0 ? -1.0 : 1.0) * (rowMax > 0.0 ? shift * rowMax : 1.0);
            // the reciprocal is what gets stored: the eliminations above and the back substitution multiply instead of dividing (an
            // IEEE fp64 division per row sits in the dependency chain of the ~10 rows a thread solves one after the other)
            A.val[bi + di * si] = 1.0 / d;
        }
    }
};

// Triangular solves, one launch per colour.  LANES threads share a cell: the cell's rows (slots) are walked in order -- later rows
// of the cell read what its earlier rows produced -- and the entries of a row are dealt round-robin to the lanes, the partial sums
// combined with a shuffle butterfly.  With the multicolour ordering (~74k cells per launch at 1M cells) LANES = 1 is faster: the
// kernels are bound by the x[col] gathers, which coalesce across the consecutive cells of a warp, and splitting a row over lanes
// divides that coalescing by LANES.  With the block-natural ordering (levels of ~5k cells) 4 lanes win: there the launches are
// too small to fill the device.  The ordering picks the variant.

template <int TRI_LANES>
DAB_HD double triRowDot(const EllView& A, int64_t bi, int64_t si, int e0, int e1, int lane, const double* y)
{
    // (a 4-way unrolled version with independent partial sums was measured: lower solve -5 %, upper solve +20 % -- not kept)
    double acc = 0.0;
    if (A.valF)
        for (int e = e0 + lane; e < e1; e += TRI_LANES) acc += (double)A.valF[bi + e * si] * y[A.col[bi + e * si]];
    else
        for (int e = e0 + lane; e < e1; e += TRI_LANES) acc += A.val[bi + e * si] * y[A.col[bi + e * si]];
    return acc;
}

template <int TRI_LANES>
struct TriLowerColour // y = L^{-1} y (unit lower), in place; launched over nCells * TRI_LANES threads
{
    EllView A;
    ColourView cv;
    double* y;
    DAB_HD void operator()(int tt) const
    {
#if defined(__CUDA_ARCH__)
        // the launch is padded to whole warps and no thread leaves early: every lane of the warp takes part in every shuffle
        const int t = tt / TRI_LANES, lane = tt - t * TRI_LANES;
        for (int s = 0; s < cv.nSlots; s++)
        {
            const bool on = t < cv.slotCount[s];
            const int i = cv.slotStart[s] + t;
            double acc = 0.0;
            if (on) acc = triRowDot<TRI_LANES>(A, cv.slotBase[s] + t, cv.slotCount[s], 0, A.diag[i], lane, y);
            for (int o = 1; o < TRI_LANES; o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, TRI_LANES);
            if (on && lane == 0) y[i] -= acc;
            __syncwarp(); // the next row of this cell may read y[i]
        }
#else
        if (tt % TRI_LANES) return;
        const int t = tt / TRI_LANES;
        for (int s = 0; s < cv.nSlots; s++)
        {
            if (t >= cv.slotCount[s]) break;
            const int i = cv.slotStart[s] + t;
            const int64_t bi = A.rowBase[i], si = A.rowStride[i];
            double part[TRI_LANES];
            for (int l = 0; l < TRI_LANES; l++) part[l] = triRowDot<TRI_LANES>(A, bi, si, 0, A.diag[i], l, y);
            for (int o = 1; o < TRI_LANES; o <<= 1)
                for (int l = 0; l < TRI_LANES; l++)
                    if (!(l & o)) part[l] += part[l | o]; // same pairing as the device butterfly (lane 0's sum)
            y[i] -= part[0];
        }
#endif
    }
};

template <int TRI_LANES>
struct TriUpperColour // x = U^{-1} x, in place; launched over nCells * TRI_LANES threads
{
    EllView A;
    ColourView cv;
    double* x;
    DAB_HD void operator()(int tt) const
    {
#if defined(__CUDA_ARCH__)
        const int t = tt / TRI_LANES, lane = tt - t * TRI_LANES;
        for (int s = cv.nSlots - 1; s >= 0; s--)
        {
            const bool on = t < cv.slotCount[s];
            const int i = cv.slotStart[s] + t;
            int64_t bi = 0, si = 0;
            int di = 0;
            double acc = 0.0;
            if (on)
            {
                bi = cv.slotBase[s] + t; si = cv.slotCount[s]; di = A.diag[i];
                acc = triRowDot<TRI_LANES>(A, bi, si, di + 1, A.rowLen[i], lane, x);
            }
            for (int o = 1; o < TRI_LANES; o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, TRI_LANES);
            if (on && lane == 0) x[i] = (x[i] - acc) * (A.valF ? (double)A.valF[bi + di * si] : A.val[bi + di * si]); // the factor stores 1 / u_ii
            __syncwarp();
        }
#else
        if (tt % TRI_LANES) return;
        const int t = tt / TRI_LANES;
        for (int s = cv.nSlots - 1; s >= 0; s--)
        {
            if (t >= cv.slotCount[s]) continue;
            const int i = cv.slotStart[s] + t;
            const int64_t bi = A.rowBase[i], si = A.rowStride[i];
            const int di = A.diag[i];
            double part[TRI_LANES];
            for (int l = 0; l < TRI_LANES; l++) part[l] = triRowDot<TRI_LANES>(A, bi, si, di + 1, A.rowLen[i], l, x);
            for (int o = 1; o < TRI_LANES; o <<= 1)
                for (int l = 0; l < TRI_LANES; l++)
                    if (!(l & o)) part[l] += part[l | o];
            x[i] = (x[i] - part[0]) * (A.valF ? (double)A.valF[bi + di * si] : A.val[bi + di * si]);
        }
#endif
    }
};

// (Measured and removed: solving a colour in two steps -- one thread per ROW for the other colours' contributions, then one thread per
// cell for the in-cell substitution -- is slower: the ~10 rows of a cell gather the same x entries, which the per-cell thread
// re-reads from L1; spread over ten warps they come from L2 ten times.)
DAB_HD double ellVal(const EllView& A, int64_t o) { return A.valF ? (double)A.valF[o] : A.val[o]; }

// (Also measured and removed: accumulating the other-colour sums of ALL rows of a cell in lock step before the in-cell substitution --
// ~10 independent load chains per thread on paper; 16-slot accumulator/bound arrays spill at the 80-register budget and the solve takes
// 23.4 s instead of 7.6 s.  The plain row-after-row loop below is the fastest of the five variants tried.)
struct CvtToFloat // fp32 copy of the factors
{
    const double* src;
    float* dst;
    DAB_HD void operator()(int i) const { dst[i] = (float)src[i]; }
};

struct GatherVec // dst[i] = src[idx[i]]
{
    const double* src;
    const int32_t* idx;
    double* dst;
    DAB_HD void operator()(int i) const { dst[i] = src[idx[i]]; }
};
struct ScatterVec // dst[idx[i]] = src[i]
{
    const double* src;
    const int32_t* idx;
    double* dst;
    DAB_HD void operator()(int i) const { dst[idx[i]] = src[i]; }
};
struct JacobiApply
{
    const double *src, *dinv;
    double* dst;
    DAB_HD void operator()(int i) const { dst[i] = src[i] * dinv[i]; }
};

// ---- dense vector operations of GMRES ---------------------------------------------------------------------
struct MultiAxpy // w[i] -= sum_j h[j] * V[j*ld + i]   (sign = -1) or  w[i] = sum_j ... (assign)
{
    const double* V;
    int64_t ld;
    int k;
    const double* h;
    double* w;
    int assign;
    DAB_HD void operator()(int i) const
    {
        double s = 0.0;
        for (int j = 0; j < k; j++) s += h[j] * V[(int64_t)j * ld + i];
        w[i] = assign ? s : w[i] - s;
    }
};
struct ScaleCopy // dst = a * src
{
    const double* src;
    double a;
    double* dst;
    DAB_HD void operator()(int i) const { dst[i] = a * src[i]; }
};
struct AxpyVec // y += a*x
{
    const double* x;
    double a;
    double* y;
    DAB_HD void operator()(int i) const { y[i] += a * x[i]; }
};
struct SubVec // r = b - r
{
    const double* b;
    double* r;
    DAB_HD void operator()(int i) const { r[i] = b[i] - r[i]; }
};

#ifndef DAB_HOSTSIM
constexpr int DOT_TILE = 8;
constexpr int DOT_BLOCKS = 132 * 4; // four CTAs on each of an H100's 132 SMs: one even wave
constexpr int DOT_THREADS = 256;
// partial[b*k + j] = sum over block b's strided share of V_j . w   (deterministic two-pass reduction)
__global__ void __launch_bounds__(DOT_THREADS) multiDotPartial(const double* __restrict__ V, int64_t ld, int k, const double* __restrict__ w,
                                                               int n, double* __restrict__ partial)
{
    __shared__ double sm[DOT_THREADS / 32][DOT_TILE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j0 = 0; j0 < k; j0 += DOT_TILE)
    {
        const int nj = (k - j0) < DOT_TILE ? (k - j0) : DOT_TILE;
        double acc[DOT_TILE];
#pragma unroll
        for (int j = 0; j < DOT_TILE; j++) acc[j] = 0.0;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        {
            const double wi = w[i];
#pragma unroll
            for (int j = 0; j < DOT_TILE; j++)
                if (j < nj) acc[j] += V[(int64_t)(j0 + j) * ld + i] * wi;
        }
#pragma unroll
        for (int j = 0; j < DOT_TILE; j++)
        {
            double v = acc[j];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
            if (lane == 0) sm[warp][j] = v;
        }
        __syncthreads();
        if (threadIdx.x < nj)
        {
            double v = 0.0;
            for (int q = 0; q < DOT_THREADS / 32; q++) v += sm[q][threadIdx.x];
            partial[(int64_t)blockIdx.x * k + j0 + threadIdx.x] = v;
        }
        __syncthreads();
    }
}
__global__ void multiDotFinal(const double* __restrict__ partial, int nb, int k, double* __restrict__ out)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    double s = 0.0;
    for (int b = 0; b < nb; b++) s += partial[(int64_t)b * k + j];
    out[j] = s;
}
#endif

struct VecOps
{
    Backend* be = nullptr;
    Comm* comm = nullptr; // dot products are summed over the ranks (the MPI_Allreduce of the reference's KSP)
    DevBuf<double> partial, dOut;
    std::vector<double> hOut;
    int cap = 0; // vectors one dots() call may take; init() only ever grows it (GMRES, IDR(s) and the fixed-point solver share the object)
    void init(Backend& b, Comm* c, int maxK)
    {
        be = &b;
        comm = c;
        if (maxK <= cap) return;
        cap = maxK;
#ifndef DAB_HOSTSIM
        partial.alloc(b, (size_t)DOT_BLOCKS * (maxK + 2));
#endif
        dOut.alloc(b, maxK + 2);
        hOut.resize(maxK + 2);
    }
    // out[j] = V_j . w, j < k  (host result)
    const double* dots(const double* V, int64_t ld, int k, const double* w, int n)
    {
        if (k > cap) throw Error("VecOps::dots: more vectors than the workspace was initialised for");
#ifndef DAB_HOSTSIM
        multiDotPartial<<<DOT_BLOCKS, DOT_THREADS, 0, be->stream>>>(V, ld, k, w, n, partial.p);
        multiDotFinal<<<(k + 63) / 64, 64, 0, be->stream>>>(partial.p, DOT_BLOCKS, k, dOut.p);
        be->launches += 2;
        if (comm) comm->allreduceSum(*be, dOut.p, k);
        be->d2h(hOut.data(), dOut.p, (size_t)k * sizeof(double));
#else
        for (int j = 0; j < k; j++)
        {
            double s = 0.0;
            for (int i = 0; i < n; i++) s += V[(int64_t)j * ld + i] * w[i];
            hOut[j] = s;
        }
        be->launches += 2;
        if (comm && comm->active())
        {
            be->h2d(dOut.p, hOut.data(), (size_t)k * sizeof(double));
            comm->allreduceSum(*be, dOut.p, k);
            be->d2h(hOut.data(), dOut.p, (size_t)k * sizeof(double));
        }
#endif
        return hOut.data();
    }
    // out[j] = V_j . w left on the device (no host synchronisation); summed over the ranks
    void dotsDev(const double* V, int64_t ld, int k, const double* w, int n, double* out)
    {
        if (k > cap) throw Error("VecOps::dotsDev: more vectors than the workspace was initialised for");
#ifndef DAB_HOSTSIM
        multiDotPartial<<<DOT_BLOCKS, DOT_THREADS, 0, be->stream>>>(V, ld, k, w, n, partial.p);
        multiDotFinal<<<(k + 63) / 64, 64, 0, be->stream>>>(partial.p, DOT_BLOCKS, k, out);
#else
        for (int j = 0; j < k; j++)
        {
            double s = 0.0;
            for (int i = 0; i < n; i++) s += V[(int64_t)j * ld + i] * w[i];
            out[j] = s;
        }
#endif
        be->launches += 2;
        if (comm && comm->active()) comm->allreduceSum(*be, out, k);
    }
    double norm2(const double* w, int n) { return std::sqrt(dots(w, 0, 1, w, n)[0]); }
};

// ---- aggregated pressure coarse space (two-level correction) ----------------------------------------------
struct CoarseRestrict1 // partial[t] = sum of v_p over the cells of chunk t
{
    const double* vp; // pressure block of the vector
    const int32_t* cells;
    const int32_t* chunkStart; // [nChunks+1]
    double* partial;
    DAB_HD void operator()(int t) const
    {
        double s = 0.0;
        for (int i = chunkStart[t]; i < chunkStart[t + 1]; i++) s += vp[cells[i]];
        partial[t] = s;
    }
};
struct CoarseRestrict2 // rc[a] = sum of the partials of aggregate a
{
    const double* partial;
    const int32_t* aggChunkOff; // [nAgg+1]
    double* rc;
    DAB_HD void operator()(int a) const
    {
        double s = 0.0;
        for (int i = aggChunkOff[a]; i < aggChunkOff[a + 1]; i++) s += partial[i];
        rc[a] = s;
    }
};
struct CoarseProlong // z = 0 except z_p[c] = yc[agg[c]]
{
    const double* yc;
    const int32_t* aggOf;
    int offP, nC, aggBase;
    double* z;
    DAB_HD void operator()(int i) const
    {
        const int c = i - offP;
        z[i] = (c >= 0 && c < nC) ? yc[aggBase + aggOf[c]] : 0.0;
    }
};
struct CoarseUnit // x = indicator of the pressure DOFs of local aggregate a (a < 0: zero vector)
{
    const int32_t* aggOf;
    int offP, nC, a;
    double* x;
    DAB_HD void operator()(int i) const
    {
        const int c = i - offP;
        x[i] = (c >= 0 && c < nC && aggOf[c] == a) ? 1.0 : 0.0;
    }
};

struct CoarseUnitColour // x = indicator of the pressure DOFs of every local aggregate of probing colour k
{
    const int32_t* aggOf;
    const int32_t* aggColour;
    int offP, nC, k;
    double* x;
    DAB_HD void operator()(int i) const
    {
        const int c = i - offP;
        x[i] = (c >= 0 && c < nC && aggColour[aggOf[c]] == k) ? 1.0 : 0.0;
    }
};

// ---- sparse A*P: the product of the operator with a coarse-space vector, without a matrix-free product ------------------------------
// The multiplicative two-level step needs t = v - A z1 with z1 = P yc (piecewise-constant pressure per aggregate).  A (P e_a) is zero
// except within a few cells of the boundary of aggregate a (a constant pressure has no gradient inside), and the probing of the
// Galerkin operator computes exactly these columns: they are kept (COO while probing, CSR by row afterwards) and t = v - (AP) yc
// becomes one short sparse product per application instead of a full RevA+RevB+RevC (17 % of an IDR(s) application at 1M cells).
struct ApExtract
{
    const double* t;        // response A * (sum of unit aggregates of this probe)
    int nC, nCellStates, offPhi;
    const int32_t* aggOf;   // [nC] local aggregate of a cell
    const int32_t *own, *nei;
    const int32_t* srcOfAgg; // coloured probe: global index of the source aggregate whose reach contains local aggregate i (-1: none); or null
    int constSrc;            // one-aggregate probe: its global index
    unsigned long long* counter;
    long long cap;
    int32_t *outRow, *outAgg;
    double* outVal;
    DAB_HD void operator()(int r) const
    {
        const double v = t[r];
        if (v == 0.0) return;
        int c;
        if (r < 3 * nC) c = r / 3;
        else if (r < offPhi) c = (r - 3 * nC) % nC;
        else
        {
            const int f = r - offPhi;
            c = own[f] < nC ? own[f] : nei[f];
        }
        const int src = srcOfAgg ? srcOfAgg[aggOf[c]] : constSrc;
#if defined(__CUDA_ARCH__)
        const unsigned long long k = atomicAdd(counter, 1ull);
#else
        const unsigned long long k = (*counter)++;
#endif
        if ((long long)k < cap)
        {
            outRow[k] = r;
            outAgg[k] = src;
            outVal[k] = v;
        }
    }
};
struct ApApply // out = v - (A P) yc, rows in CSR
{
    const int32_t* ptr;
    const int32_t* agg;
    const double* val;
    const double* yc;
    const double* v;
    double* out;
    DAB_HD void operator()(int r) const
    {
        double s = 0.0;
        for (int e = ptr[r]; e < ptr[r + 1]; e++) s += val[e] * yc[agg[e]];
        out[r] = v[r] - s;
    }
};

struct Coarse
{
    bool enabled = false, valid = false;
    // sparse A*P (see ApExtract)
    bool apValid = false;
    long long apCap = 0;
    DevBuf<unsigned long long> dApCount;
    DevBuf<int32_t> dApRow, dApAgg, dApPtr, dApAggSorted;
    DevBuf<double> dApVal, dApValSorted;
    int nAggLocal = 0, nAggGlobal = 0, aggBase = 0, nChunks = 0;
    DevBuf<int32_t> dAggOf, dCells, dChunkStart, dAggChunkOff;
    DevBuf<double> dPartial, dRc, dYc;
    std::vector<double> lu;   // dense LU of the Galerkin coarse operator (row-major, nAggGlobal^2)
    std::vector<int> piv;
    std::vector<double> hRc;
    // LU with partial pivoting; nThreads > 1: the row updates of every elimination step are shared by persistent host threads
    // (spin barrier between steps) -- same arithmetic per entry as the serial loop, so the factors do not depend on the thread count
    void factor(int nThreads = 1)
    {
        const int n = nAggGlobal;
        piv.resize(n);
        if (nThreads > 1 && n >= 512)
        {
            factorThreaded(nThreads);
            return;
        }
        for (int k = 0; k < n; k++)
        {
            int p = k;
            double mx = std::fabs(lu[(size_t)k * n + k]);
            for (int i = k + 1; i < n; i++)
                if (std::fabs(lu[(size_t)i * n + k]) > mx) { mx = std::fabs(lu[(size_t)i * n + k]); p = i; }
            piv[k] = p;
            if (p != k)
                for (int j = 0; j < n; j++) std::swap(lu[(size_t)k * n + j], lu[(size_t)p * n + j]);
            const double d = lu[(size_t)k * n + k];
            if (d == 0.0) throw Error("coarse operator is singular");
            for (int i = k + 1; i < n; i++)
            {
                const double l = lu[(size_t)i * n + k] / d;
                lu[(size_t)i * n + k] = l;
                if (l != 0.0)
                    for (int j = k + 1; j < n; j++) lu[(size_t)i * n + j] -= l * lu[(size_t)k * n + j];
            }
        }
    }
    void factorThreaded(int nThreads)
    {
        const int n = nAggGlobal;
        std::atomic<int> arrived{0}, generation{0};
        std::atomic<bool> singular{false};
        auto barrier = [&]() {
            const int g = generation.load(std::memory_order_acquire);
            if (arrived.fetch_add(1, std::memory_order_acq_rel) + 1 == nThreads)
            {
                arrived.store(0, std::memory_order_relaxed);
                generation.store(g + 1, std::memory_order_release);
            }
            else
                while (generation.load(std::memory_order_acquire) == g) std::this_thread::yield();
        };
        auto worker = [&](int t) {
            for (int k = 0; k < n; k++)
            {
                if (t == 0)
                {
                    int p = k;
                    double mx = std::fabs(lu[(size_t)k * n + k]);
                    for (int i = k + 1; i < n; i++)
                        if (std::fabs(lu[(size_t)i * n + k]) > mx) { mx = std::fabs(lu[(size_t)i * n + k]); p = i; }
                    piv[k] = p;
                    if (p != k)
                        for (int j = 0; j < n; j++) std::swap(lu[(size_t)k * n + j], lu[(size_t)p * n + j]);
                    if (lu[(size_t)k * n + k] == 0.0) singular.store(true);
                }
                barrier();
                if (singular.load()) return;
                const double d = lu[(size_t)k * n + k];
                const int rows = n - (k + 1);
                const int b = k + 1 + (int)((int64_t)rows * t / nThreads), e = k + 1 + (int)((int64_t)rows * (t + 1) / nThreads);
                const double* rk = &lu[(size_t)k * n];
                for (int i = b; i < e; i++)
                {
                    double* ri = &lu[(size_t)i * n];
                    const double l = ri[k] / d;
                    ri[k] = l;
                    if (l != 0.0)
                        for (int j = k + 1; j < n; j++) ri[j] -= l * rk[j];
                }
                barrier();
            }
        };
        std::vector<std::thread> th;
        for (int t = 1; t < nThreads; t++) th.emplace_back(worker, t);
        worker(0);
        for (auto& x : th) x.join();
        if (singular.load()) throw Error("coarse operator is singular");
    }
    // explicit inverse, transposed (invT[j*n + i] = (A^-1)[i][j]): applied on the device as a coalesced GEMV (CoarseApply), so a
    // preconditioner application needs no host round trip.  Columns are independent: solved on host threads.
    DevBuf<double> dInvT;
    template <class ParallelFor>
    void invertTransposed(std::vector<double>& invT, ParallelFor pfor) const
    {
        const int n = nAggGlobal;
        invT.assign((size_t)n * n, 0.0);
        pfor(n, [&](int, int b, int e) {
            std::vector<double> x(n);
            for (int j = b; j < e; j++)
            {
                std::fill(x.begin(), x.end(), 0.0);
                x[j] = 1.0;
                // P b, then L y = P b and U x = y with row-wise (contiguous) sweeps
                for (int k = 0; k < n; k++) std::swap(x[k], x[piv[k]]);
                int first = 0;
                while (first < n && x[first] == 0.0) first++;
                for (int i = first + 1; i < n; i++)
                {
                    const double* row = &lu[(size_t)i * n];
                    double s2 = x[i];
                    for (int k = first; k < i; k++) s2 -= row[k] * x[k];
                    x[i] = s2;
                }
                for (int i = n - 1; i >= 0; i--)
                {
                    const double* row = &lu[(size_t)i * n];
                    double s2 = x[i];
                    for (int k = i + 1; k < n; k++) s2 -= row[k] * x[k];
                    x[i] = s2 / row[i];
                }
                for (int i = 0; i < n; i++) invT[(size_t)j * n + i] = x[i]; // column j of A^-1 = row j of invT
            }
        });
    }
    void solve(double* b) const
    {
        const int n = nAggGlobal;
        for (int k = 0; k < n; k++)
        {
            std::swap(b[k], b[piv[k]]);
            for (int i = k + 1; i < n; i++) b[i] -= lu[(size_t)i * n + k] * b[k];
        }
        for (int i = n - 1; i >= 0; i--)
        {
            double s = b[i];
            for (int j = i + 1; j < n; j++) s -= lu[(size_t)i * n + j] * b[j];
            b[i] = s / lu[(size_t)i * n + i];
        }
    }
};

struct Krylov
{
    bool pcValid = false;
    bool pcFactored = false; // a factorisation exists (possibly of an earlier state: adjPCLag)
    int pcAssemblies = 0;
    bool symbolic = false;
    double pcSec = 0.0;
    int n = 0;
    // ordering
    std::vector<int32_t> perm, iperm;       // new -> ext, ext -> new
    std::vector<ColourView> colours;
    DevBuf<int32_t> dPerm, dIPerm;
    // matrix
    std::vector<int64_t> rowBase;
    std::vector<int32_t> rowStride, rowLen, diag;
    DevBuf<int64_t> dRowBase;
    DevBuf<int32_t> dRowStride, dRowLen, dDiag, dCol;
    DevBuf<double> dVal, dDinv;
    DevBuf<float> dValF; // fp32 copy of the ILU factors (pcStorage fp32): halves the value traffic of every application
    bool useF32 = false;
    std::vector<double> hValAssembled; // host copy of the assembled (unfactorised) values when writeJacobians asks for dRdWTPC
    int64_t nnz = 0, ellSize = 0;
    // FD colours
    std::vector<int32_t> fdList, fdStart;
    DevBuf<int32_t> dFdList;
    // work
    DevBuf<double> R0, R1, t1, t2, t3, t4, t5;
    Coarse coarse;
    // GMRES workspace
    DevBuf<double> V, w, z, xdev, bdev, hdev;
    int vCap = 0;
    // hdev <- count host coefficients.  GMRES (m + 1 per cycle) and IDR(s) (s) share the buffer on one handle, so a copy larger
    // than it is an error rather than a write past the allocation
    void putCoeffs(Backend& be, const double* h, int count)
    {
        if ((size_t)count > hdev.n) throw Error("Krylov coefficient buffer holds " + std::to_string(hdev.n) + " values, " + std::to_string(count) + " needed");
        be.h2d(hdev.p, h, (size_t)count * sizeof(double));
    }
    DevBuf<double> idr; // IDR(s) workspace: P(s) | G(s) | U(s) | r | t | v | z
    int idrS = 0;
    bool idrShadowReady = false;
    VecOps ops;
    EllView view()
    {
        EllView e;
        e.n = n; e.rowBase = dRowBase.p; e.rowStride = dRowStride.p; e.rowLen = dRowLen.p; e.diag = dDiag.p;
        e.col = dCol.p; e.val = dVal.p;
        e.valF = useF32 && dValF.n ? dValF.p : nullptr;
        return e;
    }
};

} // namespace dab
