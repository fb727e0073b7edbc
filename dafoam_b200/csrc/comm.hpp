// Inter-rank communication of the adjoint path: ghost-cell / ghost-face copies between pipeline stages and
// the all-reduce of the GMRES dot products.  Replaces OpenFOAM's Pstream processor-patch exchange and the
// PETSc VecScatter/MPI_Allreduce of the reference (SURVEY.md section 2.3).  Product build: NCCL grouped
// ncclSend/ncclRecv on the solver's stream over NVLink; the test-only host build takes two callbacks so that
// the same host logic can be driven by torch.distributed/gloo on CPUs.
#pragma once
#include "backend.hpp"
#include "partition.hpp"
#include "views.hpp"

#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
#include <dlfcn.h>
#include <nccl.h>
#endif

namespace dab
{

#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
// NCCL is bound at run time (dlopen of libnccl.so.2) so that a process that also imports torch shares torch's
// bundled NCCL instead of pulling a second copy in by link order.
struct NcclApi
{
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    static NcclApi& get()
    {
        static NcclApi a;
        if (!a.lib)
        {
            a.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
            if (!a.lib) throw Error(std::string("cannot load libnccl.so.2: ") + dlerror());
            auto sym = [&](const char* n) {
                void* p = dlsym(a.lib, n);
                if (!p) throw Error(std::string("libnccl.so.2 lacks ") + n);
                return p;
            };
            a.GetUniqueId = (decltype(a.GetUniqueId))sym("ncclGetUniqueId");
            a.CommInitRank = (decltype(a.CommInitRank))sym("ncclCommInitRank");
            a.CommDestroy = (decltype(a.CommDestroy))sym("ncclCommDestroy");
            a.Send = (decltype(a.Send))sym("ncclSend");
            a.Recv = (decltype(a.Recv))sym("ncclRecv");
            a.AllReduce = (decltype(a.AllReduce))sym("ncclAllReduce");
            a.GroupStart = (decltype(a.GroupStart))sym("ncclGroupStart");
            a.GroupEnd = (decltype(a.GroupEnd))sym("ncclGroupEnd");
            a.GetErrorString = (decltype(a.GetErrorString))sym("ncclGetErrorString");
        }
        return a;
    }
};
#endif

extern "C"
{
    // per peer p: sendBufs[p] (sendCounts[p] doubles) goes to peers[p]; recvBufs[p] receives recvCounts[p] doubles
    typedef void (*dab_exchange_fn)(void* ctx, int nPeers, const int* peers, const double* const* sendBufs, const int* sendCounts,
                                    double* const* recvBufs, const int* recvCounts);
    typedef void (*dab_allreduce_fn)(void* ctx, double* buf, int n);
}

struct Comm
{
    int rank = 0, size = 1;
    dab_exchange_fn cbExchange = nullptr;
    dab_allreduce_fn cbAllreduce = nullptr;
    void* cbCtx = nullptr;
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
    ncclComm_t nccl = nullptr;
#endif
    bool active() const { return size > 1; }

    void initNccl(Backend& be, int rank_, int size_, const void* uid)
    {
        rank = rank_;
        size = size_;
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
        if (!uid) throw Error("dab_create: n_ranks > 1 needs an NCCL unique id");
        ncclUniqueId id;
        memcpy(&id, uid, sizeof(id));
        NcclApi& N = NcclApi::get();
        ncclResult_t r = N.CommInitRank(&nccl, size, id, rank);
        if (r != ncclSuccess) throw Error(std::string("ncclCommInitRank: ") + N.GetErrorString(r));
        {
            // NCCL builds its channels lazily on the first collective: pay that second here, not inside the first timed solve
            double* w = (double*)be.alloc(8 * sizeof(double));
            be.zero(w, 8 * sizeof(double));
            N.AllReduce(w, w, 8, ncclDouble, ncclSum, nccl, be.stream);
            be.sync();
            be.free(w);
        }
#else
        (void)be;
        (void)uid;
        if (!cbExchange) throw Error("multi-rank creation needs NCCL (product build) or communication callbacks (test build)");
#endif
    }

    void destroy()
    {
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
        if (nccl) NcclApi::get().CommDestroy(nccl);
        nccl = nullptr;
#endif
    }

    void exchange(Backend& be, const std::vector<int>& peers, const std::vector<const double*>& sendBufs, const std::vector<int>& sendCounts,
                  const std::vector<double*>& recvBufs, const std::vector<int>& recvCounts)
    {
        if (!active() || peers.empty()) return;
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
        NcclApi& N = NcclApi::get();
        N.GroupStart();
        for (size_t p = 0; p < peers.size(); p++)
        {
            if (sendCounts[p] > 0) N.Send(sendBufs[p], (size_t)sendCounts[p], ncclDouble, peers[p], nccl, be.stream);
            if (recvCounts[p] > 0) N.Recv(recvBufs[p], (size_t)recvCounts[p], ncclDouble, peers[p], nccl, be.stream);
        }
        ncclResult_t r = N.GroupEnd();
        if (r != ncclSuccess) throw Error(std::string("nccl halo exchange: ") + N.GetErrorString(r));
        be.launches++;
#else
        be.sync();
        cbExchange(cbCtx, (int)peers.size(), peers.data(), sendBufs.data(), sendCounts.data(), recvBufs.data(), recvCounts.data());
#endif
    }

    // in-place sum over ranks of n doubles in device memory
    void allreduceSum(Backend& be, double* dev, int n)
    {
        if (!active()) return;
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
        NcclApi& N = NcclApi::get();
        ncclResult_t r = N.AllReduce(dev, dev, (size_t)n, ncclDouble, ncclSum, nccl, be.stream);
        if (r != ncclSuccess) throw Error(std::string("ncclAllReduce: ") + N.GetErrorString(r));
        be.launches++;
#else
        be.sync();
        cbAllreduce(cbCtx, dev, n);
#endif
    }
};

// ---- pack / unpack kernels ---------------------------------------------------------------------------------
// component k of an exchanged item at `cell`, as the receiver must see it.  xs != 0: the value crosses a cyclic patch pair whose
// transform is R = Rtab[|xs| - 1] (xs < 0: the inverse, R^T): 3-component items are vectors (v' = R v), 9-component items rank-2
// tensors (T' = R T R^T; gradients and their adjoints), everything else is a scalar.  Ttab != nullptr marks a 3-component item as a
// position (cell centres): x' = R x + t with t = Ttab[3 (|xs| - 1)], inverse x' = R^T (x - t) (HostMesh::xfPoint, the same operation
// order).  Role of OpenFOAM's cyclicFvPatchField::patchNeighbourField -> transform(forwardT(), pnf).
DAB_HD double haloValue(const double* arr, int64_t cell, int cellStride, int compStride, int ncomp, int k, int xs, const double* Rtab,
                        const double* Ttab = nullptr)
{
    const double* a = arr + cell * cellStride;
    if (xs == 0 || (ncomp != 3 && ncomp != 9)) return a[(int64_t)k * compStride];
    const double* M = Rtab + 9 * ((xs < 0 ? -xs : xs) - 1);
    const bool inv = xs < 0;
    if (ncomp == 3 && Ttab)
    {
        const double* t = Ttab + 3 * ((xs < 0 ? -xs : xs) - 1);
        if (!inv) return M[3 * k] * a[0] + M[3 * k + 1] * a[compStride] + M[3 * k + 2] * a[2 * (int64_t)compStride] + t[k];
        return M[k] * (a[0] - t[0]) + M[3 + k] * (a[compStride] - t[1]) + M[6 + k] * (a[2 * (int64_t)compStride] - t[2]);
    }
    if (ncomp == 3)
    {
        double v = 0.0;
        for (int m = 0; m < 3; m++) v += (inv ? M[3 * m + k] : M[3 * k + m]) * a[(int64_t)m * compStride];
        return v;
    }
    const int r = k / 3, c = k - 3 * r;
    double v = 0.0;
    for (int i = 0; i < 3; i++)
    {
        const double mri = inv ? M[3 * i + r] : M[3 * r + i];
        for (int j = 0; j < 3; j++) v += mri * (inv ? M[3 * j + c] : M[3 * c + j]) * a[(int64_t)(3 * i + j) * compStride];
    }
    return v;
}
struct HaloPack
{
    const double* arr;
    int cellStride, compStride, ncomp;
    const int32_t* idx;     // [nSend] local indices to send (concatenated over peers)
    const int32_t* segOff;  // [nSend] start of the element's peer segment
    const int32_t* segCnt;  // [nSend] size of the element's peer segment
    int nSend, sumComp, compBase;
    double* buf;
    const int32_t* xf = nullptr; // [nSend] signed cyclic transform of the element (nullptr: none anywhere)
    const double* Rtab = nullptr;
    const double* Ttab = nullptr; // translations: the item is a position (see haloValue)
    DAB_HD void operator()(int i) const
    {
        const int k = i / nSend, j = i - k * nSend;
        const int64_t o = (int64_t)segOff[j] * sumComp + (int64_t)(compBase + k) * segCnt[j] + (j - segOff[j]);
        buf[o] = haloValue(arr, idx[j], cellStride, compStride, ncomp, k, xf ? xf[j] : 0, Rtab, Ttab);
    }
};
// couplings of a rank with itself (cyclic patch pair inside one sub-mesh): ghost slot <- transformed value of the local cell
struct SelfCopy
{
    double* arr;
    int cellStride, compStride, ncomp;
    const int32_t *src, *dst, *xf; // [n]; xf may be nullptr (faces)
    int n;
    const double* Rtab;
    const double* Ttab; // translations: the item is a position (see haloValue)
    DAB_HD void operator()(int i) const
    {
        const int k = i / n, j = i - k * n;
        arr[(int64_t)dst[j] * cellStride + (int64_t)k * compStride] = haloValue(arr, src[j], cellStride, compStride, ncomp, k, xf ? xf[j] : 0, Rtab, Ttab);
    }
};
struct HaloUnpack
{
    double* arr;
    int cellStride, compStride, ncomp;
    const int32_t* idx;     // [nRecv] local indices to fill
    const int32_t* segOff;
    const int32_t* segCnt;
    int nRecv, sumComp, compBase;
    const double* buf;
    DAB_HD void operator()(int i) const
    {
        const int k = i / nRecv, j = i - k * nRecv;
        const int64_t o = (int64_t)segOff[j] * sumComp + (int64_t)(compBase + k) * segCnt[j] + (j - segOff[j]);
        arr[(int64_t)idx[j] * cellStride + (int64_t)k * compStride] = buf[o];
    }
};

// ---- peer-memory ghost exchange (CUDA build, one process per GPU on one NVLink/NVSwitch node) ---------------------------------------
// Instead of pack -> grouped ncclSend/ncclRecv -> unpack, the pack kernel of the sending rank writes its values STRAIGHT INTO the
// receiving rank's window over NVLink (the window is cudaMalloc'ed by the receiver and mapped here through CUDA IPC), a one-warp
// kernel then publishes an epoch flag per peer (system-scope release), and the receiver's unpack kernel spins on its own flags
// (system-scope acquire) before it scatters the window into the ghost slots: the transfer is part of the producing kernel, no
// collective call and no NCCL launch latency on the path of a product (4 exchanges per product: 8 launches instead of ~20).
// Two parities of the window alternate, so a sender may run one exchange ahead of the receiver; every rank issues the same
// sequence of exchanges (SPMD), which is what makes the epoch counters agree.  NCCL stays for the all-reduces and as the fallback
// when IPC mapping is not available (DAB_P2P=0 forces it).
constexpr int P2P_MAXPEER = 32, P2P_CAP = 32, P2P_MAXITEMS = 8;
struct P2pItems
{
    int n, sumComp;
    double* arr[P2P_MAXITEMS];
    int cellStride[P2P_MAXITEMS], compStride[P2P_MAXITEMS], ncomp[P2P_MAXITEMS], compBase[P2P_MAXITEMS];
    bool position[P2P_MAXITEMS];
};
struct P2pDst
{
    double* base[P2P_MAXPEER];      // per peer: start of my segment in the peer's window (this set, this parity)
    long long* flag[P2P_MAXPEER];   // per peer: my flag slot in the peer's window
};
#if !defined(DAB_HOSTSIM)
struct P2pPack
{
    P2pItems it;
    P2pDst dst;
    const int32_t *idx, *segOff, *segCnt, *peerOf; // [nSend]
    int nSend;
    const int32_t* xf;  // [nSend] signed cyclic transform (nullptr: none anywhere)
    const double *Rtab, *Ttab;
    __device__ void operator()(int t) const
    {
        const int kk = t / nSend, j = t - kk * nSend;
        int a = 0;
        while (a + 1 < it.n && kk >= it.compBase[a + 1]) a++;
        const int k = kk - it.compBase[a];
        const double v = haloValue(it.arr[a], idx[j], it.cellStride[a], it.compStride[a], it.ncomp[a], k, xf ? xf[j] : 0, Rtab,
                                   it.position[a] ? Ttab : nullptr);
        dst.base[peerOf[j]][(int64_t)kk * segCnt[j] + (j - segOff[j])] = v;
    }
};
__global__ void p2pSignal(P2pDst dst, int nPeers, long long epoch)
{
    const int p = (int)threadIdx.x;
    if (p < nPeers)
    {
        __threadfence_system(); // the pack kernel before this one in the stream has completed: publish after its stores
        *(volatile long long*)dst.flag[p] = epoch;
        __threadfence_system();
    }
}
struct P2pUnpackArgs
{
    P2pItems it;
    const double* win;           // my window, this set, this parity
    const long long* flags;      // my flag slots [nPeers]
    const int32_t *idx, *segOff, *segCnt; // [nRecv]
    int nRecv, nPeers;
    long long epoch;
};
__global__ void __launch_bounds__(128) p2pUnpack(P2pUnpackArgs a, int n)
{
    // every block first waits until all peers have published this epoch (flags live in local memory: cheap to poll)
    if ((int)threadIdx.x < a.nPeers)
    {
        const volatile long long* f = a.flags + threadIdx.x;
        while (*f < a.epoch) { }
        __threadfence_system();
    }
    __syncthreads();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int kk = t / a.nRecv, j = t - kk * a.nRecv;
    int q = 0;
    while (q + 1 < a.it.n && kk >= a.it.compBase[q + 1]) q++;
    const int k = kk - a.it.compBase[q];
    const double v = a.win[(int64_t)a.segOff[j] * a.it.sumComp + (int64_t)kk * a.segCnt[j] + (j - a.segOff[j])];
    a.it.arr[q][(int64_t)a.idx[j] * a.it.cellStride[q] + (int64_t)k * a.it.compStride[q]] = v;
}
#endif

// one index set (cells or faces) exchanged with every peer
struct HaloSet
{
    int nSend = 0, nRecv = 0;
    std::vector<int> sendOffPeer, sendCntPeer, recvOffPeer, recvCntPeer; // per peer
    DevBuf<int32_t> dSendIdx, dSendSegOff, dSendSegCnt, dRecvIdx, dRecvSegOff, dRecvSegCnt;
    DevBuf<double> sendBuf, recvBuf;
    DevBuf<int32_t> dSendPeer; // [nSend] index of the element's peer
    DevBuf<int32_t> dSendXf;   // [nSend] signed cyclic transform, allocated only when some element has one
    const int32_t* xfPtr() const { return dSendXf.n ? dSendXf.p : nullptr; }
    // couplings of the rank with itself (cyclic pairs inside the sub-mesh)
    int nSelf = 0;
    DevBuf<int32_t> dSelfSrc, dSelfDst, dSelfXf;
    long long epoch = 0;       // peer-memory path: exchanges done on this set (parity = epoch & 1)
    int capComp = 0;
#ifndef DAB_HOSTSIM
    cudaEvent_t evPack = nullptr, evDone = nullptr;
#endif
    bool pending = false;

    void buildSelf(Backend& be, const std::vector<int32_t>& src, const std::vector<int32_t>& dst, const std::vector<int32_t>& xf)
    {
        if (src.size() != dst.size()) throw Error("cyclic self-coupling: send / receive lists differ in size");
        nSelf = (int)src.size();
        if (!nSelf) return;
        dSelfSrc.upload(be, src);
        dSelfDst.upload(be, dst);
        if (!xf.empty()) dSelfXf.upload(be, xf);
    }
    void build(Backend& be, const std::vector<std::vector<int32_t>>& send, const std::vector<std::vector<int32_t>>& recv,
               const std::vector<std::vector<int32_t>>* sendXf = nullptr)
    {
        if (sendXf)
        {
            std::vector<int32_t> sx;
            bool any = false;
            for (const auto& v : *sendXf)
                for (int32_t x : v) { sx.push_back(x); any = any || x != 0; }
            if (any) dSendXf.upload(be, sx);
        }
        std::vector<int32_t> si, so, sc, ri, ro, rc, sp;
        for (size_t p = 0; p < send.size(); p++)
        {
            sendOffPeer.push_back((int)si.size());
            sendCntPeer.push_back((int)send[p].size());
            for (int32_t c : send[p])
            {
                sp.push_back((int32_t)p);
                si.push_back(c);
                so.push_back(sendOffPeer.back());
                sc.push_back((int32_t)send[p].size());
            }
            recvOffPeer.push_back((int)ri.size());
            recvCntPeer.push_back((int)recv[p].size());
            for (int32_t c : recv[p])
            {
                ri.push_back(c);
                ro.push_back(recvOffPeer.back());
                rc.push_back((int32_t)recv[p].size());
            }
        }
        nSend = (int)si.size();
        nRecv = (int)ri.size();
        dSendIdx.upload(be, si); dSendSegOff.upload(be, so); dSendSegCnt.upload(be, sc); dSendPeer.upload(be, sp);
        dRecvIdx.upload(be, ri); dRecvSegOff.upload(be, ro); dRecvSegCnt.upload(be, rc);
    }
    void reserve(Backend& be, int sumComp)
    {
        if (sumComp <= capComp) return;
        sendBuf.alloc(be, (size_t)nSend * sumComp + 1, false);
        recvBuf.alloc(be, (size_t)nRecv * sumComp + 1, false);
        capComp = sumComp;
    }
};

struct HaloItem
{
    double* arr;
    int ncomp, cellStride, compStride;
    bool position = false; // a 3-component position: crosses a cyclic pair with the translation as well (haloValue)
};

struct Halo
{
    Comm* comm = nullptr;
    Backend* be = nullptr;
    std::vector<int> peers;
    HaloSet cells, faces;
    long exchanges = 0;
    // peer-memory windows (see P2pPack): p2p == false -> NCCL send/recv
    bool p2p = false;
    double* win = nullptr;               // my window (cudaMalloc)
    std::vector<double*> peerWin;        // per peer: the peer's window mapped through CUDA IPC
    size_t myData[2][2] = {{0, 0}, {0, 0}}, myFlag[2][2] = {{0, 0}, {0, 0}};     // [set][parity] offsets (doubles) in my window
    std::vector<size_t> peerData[2][2], peerFlag[2][2];                         // the same offsets in each peer's window
    std::vector<int> peerRecvOff[2];     // [set][peer]: where my segment starts in the peer's receive list
    std::vector<int> myIdxInPeer;        // my index in the peer's peer list (flag slot)

    static size_t windowLayout(size_t nRecvCells, size_t nRecvFaces, size_t data[2][2], size_t flag[2][2])
    {
        size_t off = 0;
        const size_t nr[2] = {nRecvCells, nRecvFaces};
        for (int st = 0; st < 2; st++)
            for (int q = 0; q < 2; q++)
            {
                data[st][q] = off;
                off += nr[st] * P2P_CAP;
            }
        for (int st = 0; st < 2; st++)
            for (int q = 0; q < 2; q++)
            {
                flag[st][q] = off;
                off += P2P_MAXPEER;
            }
        return off;
    }

    void setupP2P()
    {
        p2p = false;
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
        if (!comm || !comm->active()) return;
        if (const char* e = getenv("DAB_P2P"))
            if (atoi(e) == 0) return;
        const int nP = (int)peers.size(), R = comm->size, me = comm->rank;
        // every decision below must be the same on all ranks: problems are summed over the ranks before anybody acts on them
        double bad = (nP > P2P_MAXPEER) ? 1.0 : 0.0;
        // 1. table of everybody's receive layout: row r = [nPeers, nRecvCells, nRecvFaces, (peerRank, recvOffCells, recvOffFaces) x nPeers]
        const int RW = 4 + 3 * P2P_MAXPEER;
        std::vector<double> tab((size_t)R * RW, 0.0);
        if (bad == 0.0)
        {
            double* row = &tab[(size_t)me * RW];
            row[0] = nP; row[1] = cells.nRecv; row[2] = faces.nRecv;
            for (int p = 0; p < nP; p++)
            {
                row[4 + 3 * p] = peers[p];
                row[5 + 3 * p] = cells.recvOffPeer[p];
                row[6 + 3 * p] = faces.recvOffPeer[p];
            }
        }
        // 2. my window + its IPC handle (one byte per double: exact through a sum with zeros)
        size_t nW = windowLayout(cells.nRecv, faces.nRecv, myData, myFlag);
        cudaIpcMemHandle_t hnd;
        memset(&hnd, 0, sizeof(hnd));
        if (cudaMalloc((void**)&win, (nW + 2) * sizeof(double)) != cudaSuccess) { bad = 1.0; win = nullptr; cudaGetLastError(); }
        if (win)
        {
            cudaMemset(win, 0, (nW + 2) * sizeof(double));
            cudaDeviceSynchronize();
            if (cudaIpcGetMemHandle(&hnd, win) != cudaSuccess) { bad = 1.0; cudaGetLastError(); }
        }
        const int HB = (int)sizeof(cudaIpcMemHandle_t);
        std::vector<double> hv((size_t)R * HB + 1, 0.0);
        for (int i = 0; i < HB; i++) hv[(size_t)me * HB + i] = (double)((const unsigned char*)&hnd)[i];
        hv[(size_t)R * HB] = bad;
        DevBuf<double> dTab, dH;
        dTab.upload(*be, tab);
        dH.upload(*be, hv);
        comm->allreduceSum(*be, dTab.p, (int)tab.size());
        comm->allreduceSum(*be, dH.p, (int)hv.size());
        be->d2h(tab.data(), dTab.p, tab.size() * sizeof(double));
        be->d2h(hv.data(), dH.p, hv.size() * sizeof(double));
        bool ok = hv[(size_t)R * HB] == 0.0;
        // 3. map the peers' windows, find my segment in their layout
        peerWin.assign(nP, nullptr);
        myIdxInPeer.assign(nP, -1);
        for (int st = 0; st < 2; st++)
        {
            peerRecvOff[st].assign(nP, 0);
            for (int q = 0; q < 2; q++) { peerData[st][q].assign(nP, 0); peerFlag[st][q].assign(nP, 0); }
        }
        double bad2 = 0.0;
        if (ok)
            for (int p = 0; p < nP; p++)
            {
                const int r = peers[p];
                const double* row = &tab[(size_t)r * RW];
                const int rp = (int)row[0];
                for (int i = 0; i < rp; i++)
                    if ((int)row[4 + 3 * i] == me)
                    {
                        myIdxInPeer[p] = i;
                        peerRecvOff[0][p] = (int)row[5 + 3 * i];
                        peerRecvOff[1][p] = (int)row[6 + 3 * i];
                    }
                if (myIdxInPeer[p] < 0) bad2 = 1.0;
                size_t d[2][2], f[2][2];
                windowLayout((size_t)row[1], (size_t)row[2], d, f);
                for (int st = 0; st < 2; st++)
                    for (int q = 0; q < 2; q++) { peerData[st][q][p] = d[st][q]; peerFlag[st][q][p] = f[st][q]; }
                cudaIpcMemHandle_t ph;
                for (int i = 0; i < HB; i++) ((unsigned char*)&ph)[i] = (unsigned char)hv[(size_t)r * HB + i];
                void* mapped = nullptr;
                if (cudaIpcOpenMemHandle(&mapped, ph, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { bad2 = 1.0; cudaGetLastError(); }
                peerWin[p] = (double*)mapped;
            }
        else
            bad2 = 1.0;
        DevBuf<double> dB;
        std::vector<double> b1(1, bad2);
        dB.upload(*be, b1);
        comm->allreduceSum(*be, dB.p, 1);
        be->d2h(b1.data(), dB.p, sizeof(double));
        p2p = b1[0] == 0.0;
        if (getenv("DAB_SETUP_INFO"))
            fprintf(stderr, "[dab200] halo exchange: %s (rank %d, %d peers)\n", p2p ? "peer-memory windows over NVLink (CUDA IPC)" : "NCCL send/recv", me, nP);
#endif
    }

#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
    // one exchange through the peer windows on the backend's current stream: pack into the peers, publish, wait + unpack
    void runP2P(HaloSet& hs, int st, const std::vector<HaloItem>& items, int sumComp)
    {
        hs.epoch++;
        const int q = (int)(hs.epoch & 1), nP = (int)peers.size();
        P2pItems it;
        it.n = (int)items.size();
        it.sumComp = sumComp;
        int base = 0;
        for (int i = 0; i < it.n; i++)
        {
            it.arr[i] = items[i].arr; it.cellStride[i] = items[i].cellStride; it.compStride[i] = items[i].compStride;
            it.ncomp[i] = items[i].ncomp; it.compBase[i] = base; it.position[i] = items[i].position;
            base += items[i].ncomp;
        }
        P2pDst dst;
        for (int p = 0; p < nP; p++)
        {
            dst.base[p] = peerWin[p] + peerData[st][q][p] + (size_t)peerRecvOff[st][p] * sumComp;
            dst.flag[p] = (long long*)(peerWin[p] + peerFlag[st][q][p]) + myIdxInPeer[p];
        }
        if (hs.nSend > 0) be->launch(hs.nSend * sumComp, P2pPack{it, dst, hs.dSendIdx.p, hs.dSendSegOff.p, hs.dSendSegCnt.p, hs.dSendPeer.p, hs.nSend, hs.xfPtr(), dRtab.p, dTtab.p});
        p2pSignal<<<1, 32, 0, be->stream>>>(dst, nP, hs.epoch);
        const int n = hs.nRecv * sumComp;
        if (n > 0)
        {
            P2pUnpackArgs a{it, win + myData[st][q], (const long long*)(win + myFlag[st][q]), hs.dRecvIdx.p, hs.dRecvSegOff.p, hs.dRecvSegCnt.p,
                            hs.nRecv, nP, hs.epoch};
            p2pUnpack<<<(n + 127) / 128, 128, 0, be->stream>>>(a, n);
        }
        DAB_CUDA_CHECK(cudaGetLastError());
        be->launches += 2;
    }
    bool useP2P(const std::vector<HaloItem>& items, int sumComp) const { return p2p && sumComp <= P2P_CAP && (int)items.size() <= P2P_MAXITEMS; }
#endif

    DevBuf<double> dRtab; // rotation matrices of the cyclic transforms, 9 doubles each
    DevBuf<double> dTtab; // their translations, 3 doubles each
    bool remote() const { return comm && comm->active(); }
    bool any() const { return remote() || cells.nSelf > 0 || faces.nSelf > 0; }

    void build(Backend& b, Comm& c, const HaloPlan& plan, const std::vector<HostMesh::CycXf>& xforms)
    {
        be = &b;
        comm = &c;
        peers = plan.peers;
        std::vector<double> R(9 * xforms.size() + 1, 0.0), T(3 * xforms.size() + 1, 0.0);
        for (size_t k = 0; k < xforms.size(); k++)
        {
            for (int a = 0; a < 9; a++) R[9 * k + a] = xforms[k].R[a];
            for (int a = 0; a < 3; a++) T[3 * k + a] = xforms[k].t[a];
        }
        dRtab.upload(b, R);
        dTtab.upload(b, T);
        std::vector<std::vector<int32_t>> recvCells(plan.peers.size());
        for (size_t p = 0; p < plan.peers.size(); p++)
            for (int i = 0; i < plan.recvCellCount[p]; i++) recvCells[p].push_back(plan.recvCellStart[p] + i);
        cells.build(b, plan.sendCells, recvCells, &plan.sendXf);
        faces.build(b, plan.sendFaces, plan.recvFaces);
        std::vector<int32_t> selfDst;
        for (int i = 0; i < plan.selfRecvCount; i++) selfDst.push_back(plan.selfRecvStart + i);
        cells.buildSelf(b, plan.selfSendCells, selfDst, plan.selfSendXf);
        faces.buildSelf(b, plan.selfSendFaces, plan.selfRecvFaces, {});
        setupP2P();
    }

    // ghost slots of the rank's own cyclic images: on the launching stream, in order with the producers of the values
    void runSelf(HaloSet& hs, const std::vector<HaloItem>& items)
    {
        if (hs.nSelf == 0) return;
        for (const auto& it : items)
            be->launch(hs.nSelf * it.ncomp, SelfCopy{it.arr, it.cellStride, it.compStride, it.ncomp, hs.dSelfSrc.p, hs.dSelfDst.p,
                                                     hs.dSelfXf.n ? hs.dSelfXf.p : nullptr, hs.nSelf, dRtab.p, it.position ? dTtab.p : nullptr});
    }

    void run(HaloSet& hs, const std::vector<HaloItem>& items)
    {
        runSelf(hs, items);
        if (!remote()) return;
        int sumComp = 0;
        for (const auto& it : items) sumComp += it.ncomp;
#if !defined(DAB_HOSTSIM) && defined(DAB_WITH_NCCL)
        if (useP2P(items, sumComp))
        {
            runP2P(hs, &hs == &faces ? 1 : 0, items, sumComp);
            exchanges++;
            return;
        }
#endif
        hs.reserve(*be, sumComp);
        int base = 0;
        for (const auto& it : items)
        {
            be->launch(hs.nSend * it.ncomp, HaloPack{it.arr, it.cellStride, it.compStride, it.ncomp, hs.dSendIdx.p, hs.dSendSegOff.p,
                                                     hs.dSendSegCnt.p, hs.nSend, sumComp, base, hs.sendBuf.p, hs.xfPtr(), dRtab.p,
                                                     it.position ? dTtab.p : nullptr});
            base += it.ncomp;
        }
        std::vector<const double*> sb;
        std::vector<double*> rb;
        std::vector<int> sc, rc;
        for (size_t p = 0; p < peers.size(); p++)
        {
            sb.push_back(hs.sendBuf.p + (size_t)hs.sendOffPeer[p] * sumComp);
            rb.push_back(hs.recvBuf.p + (size_t)hs.recvOffPeer[p] * sumComp);
            sc.push_back(hs.sendCntPeer[p] * sumComp);
            rc.push_back(hs.recvCntPeer[p] * sumComp);
        }
        comm->exchange(*be, peers, sb, sc, rb, rc);
        base = 0;
        for (const auto& it : items)
        {
            be->launch(hs.nRecv * it.ncomp, HaloUnpack{it.arr, it.cellStride, it.compStride, it.ncomp, hs.dRecvIdx.p, hs.dRecvSegOff.p,
                                                       hs.dRecvSegCnt.p, hs.nRecv, sumComp, base, hs.recvBuf.p});
            base += it.ncomp;
        }
        exchanges++;
    }
    void exchangeCells(const std::vector<HaloItem>& items) { run(cells, items); }
    void exchangeFaces(const std::vector<HaloItem>& items) { run(faces, items); }

    // asynchronous variant: pack on the compute stream, exchange + unpack on the communication stream; the caller
    // launches work that does not touch ghost slots in between and calls finish() before the work that does
    void start(HaloSet& hs, const std::vector<HaloItem>& items)
    {
#ifdef DAB_HOSTSIM
        run(hs, items);
#else
        runSelf(hs, items);
        if (!remote()) return;
        if (!hs.evPack)
        {
            cudaEventCreateWithFlags(&hs.evPack, cudaEventDisableTiming);
            cudaEventCreateWithFlags(&hs.evDone, cudaEventDisableTiming);
        }
        int sumComp = 0;
        for (const auto& it : items) sumComp += it.ncomp;
        if (useP2P(items, sumComp))
        {
            // everything of this exchange goes to the communication stream (after what the compute stream has produced so far): the
            // interior kernels of the next stage overlap the NVLink stores and the wait for the peers
            cudaEventRecord(hs.evPack, be->stream);
            std::swap(be->stream, be->stream2);
            cudaStreamWaitEvent(be->stream, hs.evPack, 0);
            runP2P(hs, &hs == &faces ? 1 : 0, items, sumComp);
            cudaEventRecord(hs.evDone, be->stream);
            std::swap(be->stream, be->stream2);
            hs.pending = true;
            exchanges++;
            return;
        }
        hs.reserve(*be, sumComp);
        int base = 0;
        for (const auto& it : items)
        {
            be->launch(hs.nSend * it.ncomp, HaloPack{it.arr, it.cellStride, it.compStride, it.ncomp, hs.dSendIdx.p, hs.dSendSegOff.p,
                                                     hs.dSendSegCnt.p, hs.nSend, sumComp, base, hs.sendBuf.p, hs.xfPtr(), dRtab.p,
                                                     it.position ? dTtab.p : nullptr});
            base += it.ncomp;
        }
        cudaEventRecord(hs.evPack, be->stream);
        std::swap(be->stream, be->stream2); // everything below goes to the communication stream
        cudaStreamWaitEvent(be->stream, hs.evPack, 0);
        std::vector<const double*> sb;
        std::vector<double*> rb;
        std::vector<int> sc, rc;
        for (size_t p = 0; p < peers.size(); p++)
        {
            sb.push_back(hs.sendBuf.p + (size_t)hs.sendOffPeer[p] * sumComp);
            rb.push_back(hs.recvBuf.p + (size_t)hs.recvOffPeer[p] * sumComp);
            sc.push_back(hs.sendCntPeer[p] * sumComp);
            rc.push_back(hs.recvCntPeer[p] * sumComp);
        }
        comm->exchange(*be, peers, sb, sc, rb, rc);
        base = 0;
        for (const auto& it : items)
        {
            be->launch(hs.nRecv * it.ncomp, HaloUnpack{it.arr, it.cellStride, it.compStride, it.ncomp, hs.dRecvIdx.p, hs.dRecvSegOff.p,
                                                       hs.dRecvSegCnt.p, hs.nRecv, sumComp, base, hs.recvBuf.p});
            base += it.ncomp;
        }
        cudaEventRecord(hs.evDone, be->stream);
        std::swap(be->stream, be->stream2);
        hs.pending = true;
        exchanges++;
#endif
    }
    void finish()
    {
#ifndef DAB_HOSTSIM
        for (HaloSet* hs : {&cells, &faces})
            if (hs->pending)
            {
                cudaStreamWaitEvent(be->stream, hs->evDone, 0);
                hs->pending = false;
            }
#endif
    }
};

} // namespace dab
