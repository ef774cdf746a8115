// host_util.h -- host helpers shared by the library's sources (engine.cu, lancir.cu, fast_host.cuh):
// error reporting, element sizes, alignment.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

#include <string>

#include "avirb200.h"

namespace avb {

// Stores `msg` as this thread's avirb200_last_error() and returns `code` (engine.cu).
int fail(int code, const std::string& msg);

// Bytes of one element of an avirb200_dtype.
inline size_t elem_size(int t) { return t == AVIRB200_U8 ? 1 : (t == AVIRB200_U16 ? 2 : (t == AVIRB200_F64 ? 8 : 4)); }

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

} // namespace avb

#define CUDA_TRY(expr)                                                                       \
    do {                                                                                     \
        cudaError_t e_ = (expr);                                                             \
        if (e_ != cudaSuccess)                                                               \
            return avb::fail(e_ == cudaErrorMemoryAllocation ? AVIRB200_ERR_ALLOC            \
                                                             : (e_ == cudaErrorNoDevice ||   \
                                                                e_ == cudaErrorInsufficientDriver \
                                                                    ? AVIRB200_ERR_NO_DEVICE \
                                                                    : AVIRB200_ERR_CUDA),    \
                             std::string(#expr) + ": " + cudaGetErrorString(e_));            \
    } while (0)
