// pass_request.h -- one pass of a call as every kernel family's builder reads it: the engine's entry points
// describe their passes with it, and run_pass (engine.cu), stream_params (stream_types.h), fast_pass
// (fast_host.cuh) and the generic kernel's parameters are all filled from it.  Pure host code without CUDA
// calls: the lockstep emulation used by the CPU tests (tests/emul) builds requests too, through
// stream_fill_row_params / stream_fill_col_params.
//
// Positions are along the pass's axis: source columns and intermediate columns for the row pass,
// intermediate rows and destination rows for the column pass.
#pragma once

#include <stddef.h>

#include "avirb200.h"

namespace avs {
struct StreamLink;
}

namespace avb {

struct PassRequest {
    bool is_v = false;        // the column pass
    int lines = 0;            // rows (row pass) or the intermediate's pixel columns (column pass)
    int out0 = 0, out1 = 0;   // final outputs [out0, out1) to produce
    // source: the buffer's position 0 is global position src_base; it holds positions [src_lo, src_hi)
    const void* src = nullptr;
    size_t src_pitch = 0;     // elements between lines
    int src_type = AVIRB200_F32;
    int src_base = 0, src_lo = 0, src_hi = 0;
    // destination: the buffer's position 0 receives output dst_base
    void* dst = nullptr;
    size_t dst_pitch = 0;
    int dst_type = AVIRB200_F32;
    int dst_base = 0;
    // widened 1..3-channel plans: where the 4-channel copy of the source (row pass) or of the
    // destination (column pass) goes
    void* scratch4 = nullptr;
    // row pass on the streaming kernel only: just the first seg_top and the last seg_bot lines, in one launch
    int seg_top = 0, seg_bot = 0;
    // sharded calls, fused halo exchange (streaming kernel only): the band's link -- the row pass also
    // sends its boundary lines through it, the column pass reads the neighbours' lines from it
    const avs::StreamLink* link = nullptr;
};

// The row pass of `rows` whole source lines into every column of the intermediate rows at `mid`.
inline PassRequest row_request(const avirb200_plan_desc& d, const void* src, size_t src_pitch, int rows, float* mid,
                               size_t mid_pitch) {
    PassRequest q;
    q.lines = rows;
    q.out1 = d.dst_w;
    q.src = src;
    q.src_pitch = src_pitch;
    q.src_type = d.in_type;
    q.src_hi = d.src_w;
    q.dst = mid;
    q.dst_pitch = mid_pitch;
    return q;
}

// The column pass over `cols` intermediate columns: destination rows [out0, out1) into `dst` (its row 0 =
// row out0) from the intermediate rows [mid_lo, mid_hi) the buffer at `mid` holds (its row 0 = row mid_lo).
inline PassRequest col_request(const avirb200_plan_desc& d, int cols, const float* mid, size_t mid_pitch, int mid_lo,
                               int mid_hi, void* dst, size_t dst_pitch, int out0, int out1) {
    PassRequest q;
    q.is_v = true;
    q.lines = cols;
    q.out0 = out0;
    q.out1 = out1;
    q.src = mid;
    q.src_pitch = mid_pitch;
    q.src_base = q.src_lo = mid_lo;
    q.src_hi = mid_hi;
    q.dst = dst;
    q.dst_pitch = dst_pitch;
    q.dst_type = d.out_type;
    q.dst_base = out0;
    return q;
}

} // namespace avb
