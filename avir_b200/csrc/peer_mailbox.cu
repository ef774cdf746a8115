// peer_mailbox.cu -- the band partition, NCCL through dlopen and the halo exchange of the row-sharded calls
// (peer_mailbox.h; used by engine.cu and lancir.cu), and the C ABI's communicator functions.

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstring>
#include <mutex>
#include <vector>

#include "peer_mailbox.h"

namespace avb {

namespace {

int split(int len, int r, int nranks) { return (int)((long long)len * r / nranks); }

// The process's NCCL, or nullptr when libnccl.so.2 cannot be loaded.
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

int loaded(Nccl** nc) {
    *nc = nccl();
    return *nc ? 0 : fail(AVIRB200_ERR_NCCL, "libnccl.so.2 not loadable");
}

} // namespace

int shard_split(int src_h, int dst_h, int rank, int nranks, avirb200_shard_info* info) {
    if (nranks < 1 || rank < 0 || rank >= nranks) return fail(AVIRB200_ERR_BAD_ARG, "bad rank");
    info->src_row0 = split(src_h, rank, nranks);
    info->src_rows = split(src_h, rank + 1, nranks) - info->src_row0;
    info->dst_row0 = split(dst_h, rank, nranks);
    info->dst_rows = split(dst_h, rank + 1, nranks) - info->dst_row0;
    if (info->dst_rows <= 0 || info->src_rows <= 0) return fail(AVIRB200_ERR_UNSUPPORTED, "image has fewer rows than ranks");
    return 0;
}

int shard_halos(int need_lo, int need_end, int src_h, int rank, int nranks, avirb200_shard_info* info) {
    // (the band always contains the rank's own rows: they are produced locally anyway)
    const int own_end = info->src_row0 + info->src_rows;
    const int a = need_lo < info->src_row0 ? need_lo : info->src_row0;
    const int b = need_end > own_end ? need_end : own_end;
    info->need_row0 = a;
    info->need_rows = b - a;
    info->halo_up = info->src_row0 - a;
    info->halo_down = b - own_end;
    if ((rank > 0 && info->halo_up > info->src_row0 - split(src_h, rank - 1, nranks)) ||
        (rank + 1 < nranks && info->halo_down > split(src_h, rank + 2, nranks) - own_end))
        return fail(AVIRB200_ERR_UNSUPPORTED, "halo exceeds the neighbouring band (too many ranks)");
    return 0;
}

int comm_nccl(void* comm, Nccl** nc) {
    if (comm == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "sharded resize needs a communicator");
    return loaded(nc);
}

int PeerExchange::open(void* comm, int rank, int nranks, size_t bytes, size_t header, cudaStream_t st) {
    if (comm == comm_ && rank == rank_ && nranks == nranks_) return 0;
    Nccl* nc = nullptr;
    int r = loaded(&nc);
    if (r != 0) return r;
    // (the pushes of the last communicator's calls read the ring and write the mailboxes unmapped below)
    if (stream != nullptr) CUDA_TRY(cudaStreamSynchronize(stream));
    unmap();
    box = nullptr;
    usable = false;
    comm_ = comm; rank_ = rank; nranks_ = nranks;
    seq_ = 0;
    bool ok = nc->AllGather != nullptr;
    cudaIpcMemHandle_t mine;
    std::memset(&mine, 0, sizeof mine);
    // its own allocation (the driver carves small requests out of shared blocks, and an IPC handle
    // names the whole block): at least 2 MiB, in multiples of 2 MiB
    const size_t box_bytes = align_up(bytes, 2u << 20);
    if (ok) ok = cudaMalloc(&box, box_bytes) == cudaSuccess;
    if (ok) ok = cudaMemset(box, 0, header) == cudaSuccess;
    if (ok) ok = pin() == 0;
    if (ok) ok = cudaIpcGetMemHandle(&mine, box) == cudaSuccess;
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
            reinterpret_cast<RangeFn>(f)(&base, &len, (unsigned long long)(uintptr_t)box) == 0)
            box_off = (unsigned long long)(uintptr_t)box - base;
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
    auto map = [&](int q, char** p, unsigned long long* off) {
        cudaIpcMemHandle_t hh;
        std::memcpy(&hh, &hostrec[(size_t)q * rec], sizeof hh);
        mapped = mapped && cudaIpcOpenMemHandle((void**)p, hh, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
        std::memcpy(off, &hostrec[(size_t)q * rec + sizeof hh + 8], 8);
        if (mapped) *p += *off;
    };
    if (all_ok && rank > 0) map(rank - 1, &box_up, &off_up_);
    if (all_ok && rank + 1 < nranks) map(rank + 1, &box_down, &off_down_);
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
    usable = every;
    return 0;
}

PeerExchange::Call PeerExchange::next_call() {
    const unsigned s = ++seq_;
    words_[s & 63u] = s;
    return {s, (int)(s & 1u), &words_[s & 63u]};
}

int PeerExchange::fork(cudaStream_t st) {
    if (stream == nullptr) CUDA_TRY(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    if (forked_ == nullptr) CUDA_TRY(cudaEventCreateWithFlags(&forked_, cudaEventDisableTiming));
    if (pushed_ == nullptr) CUDA_TRY(cudaEventCreateWithFlags(&pushed_, cudaEventDisableTiming));
    CUDA_TRY(cudaEventRecord(forked_, st));
    CUDA_TRY(cudaStreamWaitEvent(stream, forked_, 0));
    return 0;
}

int PeerExchange::join(cudaStream_t st) {
    CUDA_TRY(cudaEventRecord(pushed_, stream));
    CUDA_TRY(cudaStreamWaitEvent(st, pushed_, 0));
    return 0;
}

int PeerExchange::pin() {
    if (words_ == nullptr) {
        CUDA_TRY(cudaHostAlloc(&words_, 65 * sizeof(unsigned), cudaHostAllocPortable));
        words_[64] = 1;
    }
    return 0;
}

void PeerExchange::unmap() {
    if (box_up) cudaIpcCloseMemHandle(box_up - off_up_);
    if (box_down) cudaIpcCloseMemHandle(box_down - off_down_);
    box_up = box_down = nullptr;
}

void PeerExchange::close() {
    unmap();
    cudaFreeHost(words_);
    words_ = nullptr;
    if (stream) cudaStreamDestroy(stream);
    if (forked_) cudaEventDestroy(forked_);
    if (pushed_) cudaEventDestroy(pushed_);
    stream = nullptr;
    forked_ = pushed_ = nullptr;
}

int push_rows(void* dst, size_t dst_pitch, const void* src, size_t src_pitch, size_t width, int rows, void* flag,
              const unsigned* word, cudaStream_t st) {
    if (dst_pitch == width && src_pitch == width)
        CUDA_TRY(cudaMemcpyAsync(dst, src, (size_t)rows * width, cudaMemcpyDefault, st));
    else
        CUDA_TRY(cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, width, rows, cudaMemcpyDefault, st));
    if (flag != nullptr) CUDA_TRY(cudaMemcpyAsync(flag, word, 4, cudaMemcpyDefault, st));
    return 0;
}

} // namespace avb

extern "C" {

int avirb200_comm_unique_id(void* id128) {
    avb::Nccl* nc = nullptr;
    if (const int r = avb::loaded(&nc)) return r;
    NCCL_TRY(nc->GetUniqueId(id128));
    return 0;
}

int avirb200_comm_create(const void* id128, int rank, int nranks, void** comm_out) {
    avb::Nccl* nc = nullptr;
    if (const int r = avb::loaded(&nc)) return r;
    avb::Id128 id;
    std::memcpy(&id, id128, sizeof id);
    NCCL_TRY(nc->CommInitRank(comm_out, nranks, id, rank));
    return 0;
}

void avirb200_comm_destroy(void* comm) {
    avb::Nccl* nc = avb::nccl();
    if (nc && nc->CommDestroy && comm) nc->CommDestroy(comm);
}

} // extern "C"
