// peer_mailbox.h -- what the row-sharded calls of both resizers (engine.cu: AVIR, lancir.cu: CLancIR) share:
// the band partition, NCCL loaded through dlopen (no link-time dependency), and the halo exchange: a rank's
// mailbox in device memory with its two neighbours' mailboxes mapped through CUDA IPC, the call sequence
// number, the exchange stream and the copy-engine push of rows and flags.  Each resizer lays out its own mailbox.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include <string>

#include "avirb200.h"
#include "host_util.h"

namespace avb {

// The bands of rank `rank` of `nranks`, source rows [src_h r / n, src_h (r + 1) / n) and destination rows
// [dst_h r / n, dst_h (r + 1) / n), into src_* and dst_*.  AVIRB200_ERR_BAD_ARG for a rank outside [0, nranks),
// AVIRB200_ERR_UNSUPPORTED when either band is empty.
int shard_split(int src_h, int dst_h, int rank, int nranks, avirb200_shard_info* info);

// Joins the source rows [need_lo, need_end) a band reads with its own source band (shard_split's) into need_* and
// halo_*.  AVIRB200_ERR_UNSUPPORTED when a halo is larger than the neighbouring band.
int shard_halos(int need_lo, int need_end, int src_h, int rank, int nranks, avirb200_shard_info* info);

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

// What a sharded call of more than one rank needs: a communicator (AVIRB200_ERR_BAD_ARG when null), then the
// process's NCCL in *nc (AVIRB200_ERR_NCCL when libnccl.so.2 cannot be loaded).
int comm_nccl(void* comm, Nccl** nc);

// A rank's side of the exchange with its two neighbours.  Each plan holds one; the plan's sharded calls use it
// under the plan's mutex.
struct PeerExchange {
    char* box = nullptr;      // this rank's mailbox
    char* box_up = nullptr;   // rank-1's mailbox, mapped (nullptr without that neighbour)
    char* box_down = nullptr; // rank+1's
    bool usable = false;      // every rank of the communicator mapped its neighbours
    cudaStream_t stream = nullptr; // the exchange stream, between fork() and join()

    // One call: its sequence number, its mailbox slot (call parity) and the pinned word the flag copies read.
    struct Call { unsigned seq; int slot; const unsigned* word; };

    // Collective over `comm` (every rank makes it) when comm, rank or nranks differ from the last open, else
    // nothing: allocates this rank's mailbox of `bytes` in its own 2 MiB-rounded block with its first `header`
    // bytes zeroed, all-gathers the IPC handles and offsets, maps the neighbours' mailboxes and all-gathers
    // whether every rank could.  `usable` stays false on EVERY rank when any rank could not; the error return is
    // for a failed exchange only.
    int open(void* comm, int rank, int nranks, size_t bytes, size_t header, cudaStream_t st);
    // The next call's numbers (after an open that left the exchange usable).
    Call next_call();
    // The exchange stream starts after everything enqueued on `st` so far (created with the events on first use).
    int fork(cudaStream_t st);
    // `st` waits for everything enqueued on the exchange stream so far.
    int join(cudaStream_t st);
    // The pinned words (created on first use): [0, 64) the ring of sequence numbers next_call() writes, so that
    // up to 64 calls' flag copies may be pending; [64] the constant 1.
    int pin();
    const unsigned* one() const { return words_ + 64; }
    // Unmaps the neighbours' mailboxes and frees the pinned words, stream and events.  The mailbox itself is NOT
    // freed: a neighbour process may still have it mapped (plans are destroyed without a collective), and
    // freeing exported memory before every importer has closed it is undefined behaviour (CUDA IPC).  A few MB
    // per sharded plan stay allocated until the process ends.
    void close();

private:
    void* comm_ = nullptr;
    int rank_ = -1, nranks_ = 0; // nranks_ 0: never opened
    unsigned seq_ = 0;
    unsigned long long off_up_ = 0, off_down_ = 0; // the neighbours' mailboxes inside their allocations
    cudaEvent_t forked_ = nullptr, pushed_ = nullptr;
    unsigned* words_ = nullptr;
    void unmap();
};

// On `st`: `rows` rows of `width` bytes from `src` (rows `src_pitch` bytes apart) to `dst` (`dst_pitch` apart),
// one linear copy when both pitches equal the width; then, when `flag` is given, the 4-byte `word` into it.
int push_rows(void* dst, size_t dst_pitch, const void* src, size_t src_pitch, size_t width, int rows, void* flag,
              const unsigned* word, cudaStream_t st);

} // namespace avb

#define NCCL_TRY(expr)                                                                  \
    do {                                                                                \
        int r_ = (expr);                                                                \
        if (r_ != 0)                                                                    \
            return avb::fail(AVIRB200_ERR_NCCL, std::string(#expr) + ": " +             \
                                               (nc->GetErrorString ? nc->GetErrorString(r_) \
                                                                   : "nccl error"));     \
    } while (0)
