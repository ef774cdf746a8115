// pass_config.h -- how the generic pass kernel lays a tile out in shared memory: lines per block, outputs
// per tile, the two ping-pong buffers and their pitch.  Host arithmetic only (no CUDA call): the engine
// calls it at plan creation and for every band or window range; tests/emul/config_emul.cpp runs the same
// code on the CPU.
#pragma once

#include <stddef.h>

#include "avirb200.h"
#include "device_plan.h"

namespace avb {

struct PassConfig {
    int lines_per_block = 0;
    int tile_out = 0;
    int span_a = 0; // rows of buffer 0: the source tile and the outputs of odd steps (inputs of even steps)
    int span_b = 0; // rows of buffer 1: the outputs of even steps
    int pitch = 0;  // floats per row: lines x channels, odd (bank-conflict-free column walks)
    size_t smem = 0;
};

// The shared memory a block of the generic kernel prefers to stay within (several blocks per SM).
const size_t kGenericSmemPreferred = 100 * 1024;

// The kernels' view of an axis descriptor, with the descriptor's (host) table pointers: what the
// range arithmetic reads.
inline DevAxis host_axis_view(const avirb200_axis_desc& ad) {
    DevAxis d = {};
    d.src_len = ad.src_len; d.dst_len = ad.dst_len; d.nsteps = ad.nsteps;
    int lo = 0, hi = ad.src_len;
    for (int i = 0; i < ad.nsteps && i < AVIRB200_MAX_STEPS; ++i) {
        const avirb200_step_desc& s = ad.steps[i];
        DevStep& ds = d.steps[i];
        ds.kind = s.kind; ds.resample = s.resample; ds.latency = s.latency; ds.edge = s.edge;
        ds.in_len = s.in_len; ds.out_len = s.out_len; ds.ntaps = s.ntaps; ds.order = s.order;
        ds.upsampled = s.upsampled; ds.skip_odd = s.skip_odd; ds.zero_start = s.zero_start;
        ds.nphases = s.nphases;
        ds.out_prefix = s.out_prefix; ds.out_suffix = s.out_suffix;
        ds.in_prefix = s.in_prefix; ds.in_suffix = s.in_suffix;
        ds.n_prefix_dc = s.n_prefix_dc; ds.n_suffix_dc = s.n_suffix_dc;
        ds.in_lo = lo; ds.in_hi = hi;
        ds.taps = s.taps; ds.src_pos = s.src_pos; ds.phase = s.phase; ds.frac = s.frac;
        ds.prefix_dc = s.prefix_dc; ds.suffix_dc = s.suffix_dc;
        const Range od = step_output_domain(ds);
        lo = od.a; hi = od.b + 1;
    }
    return d;
}

// Source range a final-output range needs, through the whole chain (host side).
inline Range chain_source_range(const DevAxis& hd, Range out, int* max_span) {
    Range r = out;
    int span = r.b - r.a + 1;
    for (int i = hd.nsteps - 1; i >= 0; --i) {
        r = step_input_range(hd.steps[i], r, hd.steps[i].src_pos);
        span = imax(span, r.b - r.a + 1);
    }
    if (max_span) *max_span = span;
    return r;
}

// Accumulates the rows each buffer needs for the final outputs [j0, j1]: the range step i reads lives
// in buffer i & 1 (the source tile in buffer 0), the final outputs in buffer nsteps & 1.
inline void generic_tile_spans(const DevAxis& hd, int j0, int j1, int& span_a, int& span_b) {
    Range r{j0, j1};
    for (int i = hd.nsteps;; --i) {
        const int n = r.b - r.a + 1;
        if (i & 1) span_b = imax(span_b, n); else span_a = imax(span_a, n);
        if (i == 0) break;
        r = step_input_range(hd.steps[i - 1], r, hd.steps[i - 1].src_pos);
    }
}

// The generic kernel's layout for the final outputs [out0, out1).  With 64 / channels lines per block,
// the longest tile whose two buffers, sized by the larger span, stay within kGenericSmemPreferred;
// failing that one output per tile, with the buffers sized by their own spans and the lines per block
// halved until they fit max_smem (the device's per-block opt-in limit).  The result's smem exceeds
// max_smem only when one output of one line does not fit: the plan is then refused.  Each output's
// arithmetic does not depend on the layout.
inline PassConfig choose_generic_config(const DevAxis& hd, int channels, int out0, int out1, size_t max_smem) {
    static const int cand[] = {1024, 768, 512, 384, 256, 192, 128, 96, 64, 48, 32, 24, 16, 12, 8, 4, 2, 1};
    PassConfig c;
    c.lines_per_block = imax(1, 64 / channels);
    c.pitch = (c.lines_per_block * channels) | 1;
    for (int t : cand) {
        int sa = 0, sb = 0;
        for (int j0 = out0; j0 < out1; j0 += t) generic_tile_spans(hd, j0, imin(j0 + t, out1) - 1, sa, sb);
        c.tile_out = t;
        c.span_a = sa;
        c.span_b = sb;
        if (2ull * imax(sa, sb) * c.pitch * sizeof(float) <= kGenericSmemPreferred) break;
    }
    for (;;) {
        c.pitch = (c.lines_per_block * channels) | 1;
        c.smem = (size_t)(c.span_a + c.span_b) * c.pitch * sizeof(float);
        if (c.smem <= max_smem || c.lines_per_block == 1) break;
        c.lines_per_block /= 2;
    }
    return c;
}

} // namespace avb
