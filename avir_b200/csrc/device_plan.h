// device_plan.h -- device-side mirror of the C-ABI plan descriptor (avirb200.h) and the
// range arithmetic shared by host launch code and kernels.
#pragma once

#include <stdint.h>

#include "avirb200.h"

#if defined(__CUDACC__)
#define AVB_HD __host__ __device__ __forceinline__
#else
#define AVB_HD inline
#endif

namespace avb {

struct DevStep {
    int kind, resample, latency, edge;
    int in_len, out_len, ntaps, order;
    int upsampled, skip_odd, zero_start, nphases;
    int out_prefix, out_suffix, in_prefix, in_suffix;
    int n_prefix_dc, n_suffix_dc;
    int in_lo, in_hi; // valid index range [in_lo, in_hi) of this step's INPUT line
    const float* taps;
    const int* src_pos;
    const int* phase;
    const float* frac;
    const float* prefix_dc;
    const float* suffix_dc;
};

struct DevAxis {
    int src_len, dst_len, nsteps;
    DevStep steps[AVIRB200_MAX_STEPS];
};

struct Range {
    int a, b; // inclusive
};

// What every kernel family does to a pixel on the way in (sRGB linearisation: row pass) and on the way out
// (gamma, rounding, bit-depth truncation, clamping: column pass).
struct PixelStage {
    int gamma_in, gamma_out, alpha_index;
    float in_gamma_mult, out_gamma_mult;
    const float* srgb_lut; // 256 floats (u8 input), device memory
    int round_mode;
    float tr_mul, tr_mul_inv, pk_out;
};

inline PixelStage pixel_stage(const avirb200_plan_desc& d, const float* srgb_lut) {
    PixelStage s;
    s.gamma_in = (d.use_gamma & 1) ? 1 : 0;
    s.gamma_out = (d.use_gamma & 2) ? 1 : 0;
    s.alpha_index = d.alpha_index;
    s.in_gamma_mult = d.in_gamma_mult;
    s.out_gamma_mult = d.out_gamma_mult;
    s.srgb_lut = srgb_lut;
    s.round_mode = d.round_mode;
    s.tr_mul = d.tr_mul;
    s.tr_mul_inv = d.tr_mul_inv;
    s.pk_out = d.pk_out;
    return s;
}

AVB_HD int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }
AVB_HD int imin(int a, int b) { return a < b ? a : b; }
AVB_HD int imax(int a, int b) { return a > b ? a : b; }

// Input indices (of the step's own input line) needed to produce outputs [o.a, o.b].
// src_pos must be readable from the caller's address space.
AVB_HD Range step_input_range(const DevStep& s, Range o, const int* src_pos) {
    Range r;
    if (s.kind == AVIRB200_STEP_FIR) {
        r.a = (o.a - s.edge) * s.resample - s.latency;
        r.b = (o.b - s.edge) * s.resample - s.latency + s.ntaps - 1;
    } else if (s.kind == AVIRB200_STEP_RESIZE) {
        const int d21 = s.ntaps / 2 - 1;
        r.a = src_pos[o.a] - d21;
        r.b = src_pos[o.b] - d21 + s.ntaps - 1;
        if (s.upsampled) {
            r.a >>= 1;
            r.b >>= 1;
        }
    } else {
        const int R = s.resample;
        r.a = floordiv(o.a + s.latency - (s.ntaps - 1) + R - 1, R);
        r.b = floordiv(o.b + s.latency, R);
        const int pfx = -s.in_prefix * R;
        const int sfx = (s.in_len + s.in_suffix) * R - s.latency;
        if (o.a < pfx + s.n_prefix_dc && o.b >= pfx) r.a = imin(r.a, 0);
        if (o.a < sfx + s.n_suffix_dc && o.b >= sfx) r.b = imax(r.b, s.in_len - 1);
    }
    r.a = imin(imax(r.a, s.in_lo), s.in_hi - 1);
    r.b = imin(imax(r.b, s.in_lo), s.in_hi - 1);
    return r;
}

// Valid index range of a step's OUTPUT line.
AVB_HD Range step_output_domain(const DevStep& s) {
    Range r;
    if (s.kind == AVIRB200_STEP_UPSAMPLE) {
        r.a = -s.out_prefix;
        r.b = s.out_len + s.out_suffix - 1;
    } else {
        r.a = 0;
        r.b = s.out_len - 1;
    }
    return r;
}

} // namespace avb
