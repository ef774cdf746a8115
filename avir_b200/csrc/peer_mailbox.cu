// peer_mailbox.cu -- NCCL through dlopen and the IPC-mapped halo mailboxes of the row-sharded calls
// (peer_mailbox.h; used by engine.cu and lancir.cu).

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstring>
#include <mutex>
#include <vector>

#include "peer_mailbox.h"

namespace avb {

Nccl* nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, []() {
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) {
            n.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (n.lib) break;
        }
        if (!n.lib) return;
        n.GetUniqueId = (int (*)(void*))dlsym(n.lib, "ncclGetUniqueId");
        n.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(n.lib, "ncclCommInitRank");
        n.CommDestroy = (int (*)(void*))dlsym(n.lib, "ncclCommDestroy");
        n.Send = (int (*)(const void*, size_t, int, int, void*, cudaStream_t))dlsym(n.lib, "ncclSend");
        n.Recv = (int (*)(void*, size_t, int, int, void*, cudaStream_t))dlsym(n.lib, "ncclRecv");
        n.GroupStart = (int (*)())dlsym(n.lib, "ncclGroupStart");
        n.GroupEnd = (int (*)())dlsym(n.lib, "ncclGroupEnd");
        n.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(n.lib, "ncclAllGather");
        n.GetErrorString = (const char* (*)(int))dlsym(n.lib, "ncclGetErrorString");
    });
    if (!n.lib || !n.GetUniqueId || !n.CommInitRank || !n.Send || !n.Recv || !n.GroupStart ||
        !n.GroupEnd)
        return nullptr;
    return &n;
}

int peer_boxes_open(void* comm, int rank, int nranks, size_t bytes, size_t header, cudaStream_t st, PeerBoxes* h) {
    Nccl* nc = nccl();
    if (!nc) return fail(AVIRB200_ERR_NCCL, "libnccl.so.2 not loadable");
    bool ok = nc->AllGather != nullptr;
    cudaIpcMemHandle_t mine;
    std::memset(&mine, 0, sizeof mine);
    // its own allocation (the driver carves small requests out of shared blocks, and an IPC handle
    // names the whole block): at least 2 MiB, in multiples of 2 MiB
    const size_t box_bytes = align_up(bytes, 2u << 20);
    if (ok) ok = cudaMalloc(&h->box, box_bytes) == cudaSuccess;
    if (ok) ok = cudaMemset(h->box, 0, header) == cudaSuccess;
    if (ok) ok = cudaHostAlloc(&h->h_seq, 64 * sizeof(unsigned), cudaHostAllocPortable) == cudaSuccess;
    if (ok) ok = cudaIpcGetMemHandle(&mine, h->box) == cudaSuccess;
    // (an IPC handle names the allocation the pointer lies in; importers add the pointer's offset in it)
    unsigned long long box_off = 0;
    if (ok) {
        typedef int (*RangeFn)(unsigned long long*, size_t*, unsigned long long);
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        unsigned long long base = 0;
        size_t len = 0;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess && f != nullptr &&
            reinterpret_cast<RangeFn>(f)(&base, &len, (unsigned long long)(uintptr_t)h->box) == 0)
            box_off = (unsigned long long)(uintptr_t)h->box - base;
        else
            cudaGetLastError();
    }
    // all-gather (handle, ok, offset) records
    const size_t rec = sizeof(cudaIpcMemHandle_t) + 16;
    std::vector<char> hostrec((size_t)nranks * rec, 0);
    char* drec = nullptr;
    if (cudaMalloc(&drec, (size_t)nranks * rec) != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_ALLOC, "halo setup"); }
    std::memcpy(&hostrec[(size_t)rank * rec], &mine, sizeof mine);
    hostrec[(size_t)rank * rec + sizeof mine] = ok ? 1 : 0;
    std::memcpy(&hostrec[(size_t)rank * rec + sizeof mine + 8], &box_off, 8);
    cudaMemcpyAsync(drec + (size_t)rank * rec, &hostrec[(size_t)rank * rec], rec, cudaMemcpyHostToDevice, st);
    int nr = nc->AllGather ? nc->AllGather(drec + (size_t)rank * rec, drec, rec, /*ncclChar*/ 0, comm, st) : 1;
    cudaError_t ce = cudaMemcpyAsync(hostrec.data(), drec, (size_t)nranks * rec, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    cudaFree(drec);
    if (nr != 0 || ce != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_NCCL, "halo setup: handle exchange failed"); }
    bool all_ok = true;
    for (int q = 0; q < nranks; ++q) all_ok = all_ok && hostrec[(size_t)q * rec + sizeof mine] == 1;
    // second round: can every rank map its neighbours?
    bool mapped = all_ok;
    if (all_ok && rank > 0) {
        cudaIpcMemHandle_t hh;
        std::memcpy(&hh, &hostrec[(size_t)(rank - 1) * rec], sizeof hh);
        mapped = mapped && cudaIpcOpenMemHandle((void**)&h->box_up, hh, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
        unsigned long long off = 0;
        std::memcpy(&off, &hostrec[(size_t)(rank - 1) * rec + sizeof hh + 8], 8);
        if (mapped) h->box_up += off;
        h->off_up = off;
    }
    if (all_ok && rank + 1 < nranks) {
        cudaIpcMemHandle_t hh;
        std::memcpy(&hh, &hostrec[(size_t)(rank + 1) * rec], sizeof hh);
        mapped = mapped && cudaIpcOpenMemHandle((void**)&h->box_down, hh, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
        unsigned long long off = 0;
        std::memcpy(&off, &hostrec[(size_t)(rank + 1) * rec + sizeof hh + 8], 8);
        if (mapped) h->box_down += off;
        h->off_down = off;
    }
    cudaGetLastError();
    std::vector<char> flags((size_t)nranks, 0);
    char* dflag = nullptr;
    if (cudaMalloc(&dflag, (size_t)nranks) != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_ALLOC, "halo setup"); }
    flags[rank] = mapped ? 1 : 0;
    cudaMemcpyAsync(dflag + rank, &flags[rank], 1, cudaMemcpyHostToDevice, st);
    nr = nc->AllGather(dflag + rank, dflag, 1, 0, comm, st);
    ce = cudaMemcpyAsync(flags.data(), dflag, (size_t)nranks, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    cudaFree(dflag);
    if (nr != 0 || ce != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_NCCL, "halo setup: status exchange failed"); }
    bool every = true;
    for (int q = 0; q < nranks; ++q) every = every && flags[q] == 1;
    h->usable = every;
    return 0;
}

void peer_boxes_close(PeerBoxes* h) {
    if (h->box_up) cudaIpcCloseMemHandle(h->box_up - h->off_up);
    if (h->box_down) cudaIpcCloseMemHandle(h->box_down - h->off_down);
    h->box_up = h->box_down = nullptr;
    cudaFreeHost(h->h_seq);
    h->h_seq = nullptr;
}

} // namespace avb
