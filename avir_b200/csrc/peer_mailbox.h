// peer_mailbox.h -- what the row-sharded calls of both resizers (engine.cu: AVIR, lancir.cu: CLancIR) share:
// NCCL loaded through dlopen (no link-time dependency), and a rank's halo mailbox in device memory with its
// two neighbours' mailboxes mapped through CUDA IPC.  Each resizer lays out its own mailbox.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include <string>

#include "avirb200.h"
#include "host_util.h"

namespace avb {

struct Id128 { char b[128]; }; // ncclUniqueId (passed by value)

struct Nccl {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, Id128, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};

// The process's NCCL, or nullptr when libnccl.so.2 cannot be loaded.
Nccl* nccl();

// A rank's mailbox and its neighbours' (nullptr where there is no neighbour), and the pinned ring of
// sequence numbers the flag copies read.  usable: every rank of the communicator mapped its neighbours.
struct PeerBoxes {
    char* box = nullptr;
    char* box_up = nullptr;   // rank-1's mailbox, mapped
    char* box_down = nullptr; // rank+1's mailbox, mapped
    unsigned long long off_up = 0, off_down = 0; // the neighbours' mailboxes inside their allocations
    unsigned* h_seq = nullptr; // 64 entries
    bool usable = false;
};

// Collective over `comm` (every rank makes it): allocates this rank's mailbox of `bytes` in its own
// 2 MiB-rounded block with its first `header` bytes zeroed, all-gathers the IPC handles and offsets, maps
// the neighbours' mailboxes and all-gathers whether every rank could.  pb->usable stays false on EVERY rank
// when any rank could not; the error return is for a failed exchange only.
int peer_boxes_open(void* comm, int rank, int nranks, size_t bytes, size_t header, cudaStream_t st, PeerBoxes* pb);

// Unmaps the neighbours' mailboxes and frees the ring.  The mailbox itself is NOT freed: a neighbour process
// may still have it mapped (plans are destroyed without a collective), and freeing exported memory before
// every importer has closed it is undefined behaviour (CUDA IPC).  A few MB per sharded plan stay allocated
// until the process ends.
void peer_boxes_close(PeerBoxes* pb);

} // namespace avb

#define NCCL_TRY(expr)                                                                  \
    do {                                                                                \
        int r_ = (expr);                                                                \
        if (r_ != 0)                                                                    \
            return avb::fail(AVIRB200_ERR_NCCL, std::string(#expr) + ": " +             \
                                               (nc->GetErrorString ? nc->GetErrorString(r_) \
                                                                   : "nccl error"));     \
    } while (0)
