// fast_kernel.cuh -- specialised pass kernel for 4-channel images (sm_90a), device side.
//
// Same job as generic_pass.cuh (one kernel = one whole 1-D filtering chain for a tile of
// lines, every intermediate in shared memory) with the structure the FP32 pipe needs to be
// the limiter, because the bit-exact contract forbids FMA: each tap costs a separate
// multiply and add, so every other instruction in the inner loops competes for issue slots.
//
//   * lane = one channel PAIR (float2) of one line; a warp = the 32 lanes (16 lines) of ONE
//     position, so positions/taps/phases are warp-uniform: no divergence, tap reads are
//     shared-memory broadcasts, input reads are conflict-free 256-byte rows;
//   * register blocking: a thread produces 4 consecutive outputs from one register window
//     of inputs (window loads amortised over 4 x taps products) -- fully unrolled templates
//     for the chains of the BASELINE configs, plain loops for everything else; the variant
//     is dispatched once per step per warp, not per output;
//   * order-1 interpolation taps c0 + c1*x are row/column-invariant: they are formed once on
//     the host (same two float operations upstream performs) into an "effective phase"
//     table, so the kernels always run order-0 arithmetic;
//   * edge replication is materialised: a tile covers the UNCLAMPED index range its
//     consumer reads, out-of-domain positions hold the clamped sample, so inner loops
//     carry no index clamps;
//   * the source tile is staged with cp.async (16-byte LDGSTS, no register round trip, all
//     of a thread's copies in flight at once) while the tap rows of every step are staged
//     alongside.
//
// Arithmetic order is upstream's (see generic_pass.cuh / oracle/avir_port.c); tests run
// every case through both kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "device_plan.h"
#include "generic_pass.cuh"

namespace avb {

constexpr int kFastLanes = 32;      // lane pairs per position = 16 lines x 2
constexpr int kFastLines = 16;
constexpr int kFastThreads = 384;
constexpr int kFastBlocksPerSM = 1;
constexpr int kTileRec = 20; // ints per host-built tile record (see fast_host.cuh)
constexpr int kFastWarps = kFastThreads / 32;
constexpr int kFastMaxSteps = 4;
constexpr int kFastPitch = kFastLanes + 2; // float2 units: 272 bytes (16-byte aligned rows)

enum FastVariant : int {
    kVarSimple = 0,
    kVarResizeDil24D2,   // float8_dil, FL 24, source step 2            (cfg3 mirror dil)
    kVarResizeDil56D4,   // float8_dil, FL 56, source step 4            (cfg5)
    kVarResizeDil32D2,
    kVarResizeInl18D2,   // interleaved, FL 18, source step 2           (cfg3 float4, cfg4)
    kVarResizeInl24D2,
    kVarFirDil8R1,       // float8_dil 8-tap (7 + pad) correction       (cfg3/cfg5 dil)
    kVarFirInl7R1,       // interleaved 7-tap (L = 3), R = 1            (LPF k=2, correction)
    kVarFirInl15R2,      // interleaved 15-tap (L = 7), R = 2           (cfg4 decimator)
    kVarResize2Inl24,    // interleaved FL 24 over the virtual 2X line, skip-odd (cfg2, k = 0.5)
};

struct FastStep {
    int kind, variant;
    int resample, latency, edge, ntaps, ntaps_pad;
    int out_len;
    int in_lo, in_hi;    // valid domain of the input line
    int upsampled, skip_odd, zero_start;
    int n_eff;           // RESIZE: rows in `taps` (distinct effective phases)
    const float* taps;   // FIR: ntaps floats; RESIZE: [n_eff][ntaps_pad]
    const int* src_pos;  // RESIZE
    const int* eff;      // RESIZE: per-output row of `taps`
};

struct FastAxis {
    int nsteps, src_len, dst_len;
    FastStep s[kFastMaxSteps];
};

struct FastParams {
    FastAxis ax;
    int is_v;
    int n_lines;          // rows (H) or pixel columns (V) in this launch
    int tile_out;
    int out0, out1;
    int span_a, span_b;   // shared rows of the two ping-pong buffers
    int tap_off[kFastMaxSteps]; // float offset of each step's staged taps
    int taps_floats;            // total staged tap floats (integer-source raw tiles start behind)
    const int* tile_ranges;     // per tile: (a, b) of the source tile and of every step's output
    int uniform_taps[kFastMaxSteps]; // resize step whose outputs all share one effective phase
    int rtaps_step;                  // the step whose single effective phase is in rtaps (-1: none)
    float rtaps[64];                 // that phase: constant-bank operands for the blocked loops
    int debug;                       // always 0 (perf experiments of round 1: 1 = skip the arithmetic, 2 = skip source staging)
    const void* src;
    long long src_pitch;  // elements
    int src_type;
    int src_row_base;     // source position held by the buffer's position 0 (column pass: row; row pass: column)
    void* dst;
    long long dst_pitch;
    int dst_type;
    int dst_row_base;     // final output stored at the destination's position 0 (column pass: row; row pass: column)
    PixelStage px;
};

// ---- host+device range arithmetic (unclamped: tiles materialise edge replicas) ----------------

AVB_HD Range fast_input_range(const FastStep& s, Range o, const int* src_pos) {
    // o must lie inside the step's output domain
    Range r;
    if (s.kind == AVIRB200_STEP_FIR) {
        r.a = (o.a - s.edge) * s.resample - s.latency;
        r.b = (o.b - s.edge) * s.resample - s.latency + s.ntaps - 1;
    } else {
        const int d21 = s.ntaps / 2 - 1;
        r.a = src_pos[o.a] - d21;
        r.b = src_pos[o.b] - d21 + s.ntaps - 1;
        if (s.upsampled) {
            r.a >>= 1;
            r.b >>= 1;
        }
    }
    return r;
}

AVB_HD Range clampr(Range r, int lo, int hi) {
    Range c;
    c.a = imin(imax(r.a, lo), hi - 1);
    c.b = imin(imax(r.b, lo), hi - 1);
    return c;
}

#if defined(__CUDACC__)

// ---- small device helpers ------------------------------------------------------------------------

// The two channels a lane owns travel as one pair.  Upstream multiplies and adds separately
// (two roundings per tap), so every product and sum is its own IEEE FMUL / FADD (sm_90 has no
// packed FP32 instructions; __fmul_rn / __fadd_rn are never contracted into an FFMA).
__device__ __forceinline__ float2 f2mul(float t, float2 x) {
    return make_float2(__fmul_rn(t, x.x), __fmul_rn(t, x.y));
}
__device__ __forceinline__ float2 f2add(float2 a, float2 b) {
    return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2hadd8(const float2* v) {
    return f2add(f2add(f2add(v[0], v[4]), f2add(v[1], v[5])),
                 f2add(f2add(v[2], v[6]), f2add(v[3], v[7])));
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem));
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// Integer destinations: round (the class's own round()), clamp (avir.h:4392-4419).
__device__ __forceinline__ float epilogue_round_c4(const FastParams& p, float v) {
    if (p.px.tr_mul == 1.0f) v = round_out(v, p.px.round_mode);
    else v = __fmul_rn(round_out(__fmul_rn(v, p.px.tr_mul_inv), p.px.round_mode), p.px.tr_mul);
    return v < 0.0f ? 0.0f : (v > p.px.pk_out ? p.px.pk_out : v);
}

// Output stage for one element (gamma -> round -> clamp), 4-channel images.
__device__ __forceinline__ float epilogue_value_c4(const FastParams& p, float v, int c) {
    if (p.px.gamma_out) {
        if (c == p.px.alpha_index) v = __fmul_rn(v, p.px.out_gamma_mult);
        else v = __fmul_rn(lin2srgb(v), p.px.out_gamma_mult);
    }
    if (p.dst_type != AVIRB200_F32) v = epilogue_round_c4(p, v);
    return v;
}

// ---- blocked step routines: M outputs from one register window ----------------------------------
// `x0` points at the thread's lane in the row of the first input position of output 0; rows
// are kFastPitch float2 apart.  `tp` = staged taps of output 0 (FLP floats per output).

template <int SUM, int FL, int FLP, int D, int M, bool UNI>
__device__ __forceinline__ void resize_blocked(const FastParams& p, const float2* x0, const float* tp,
                                               int tstride, int zero_start, float2* out) {
    constexpr int W = FL + (M - 1) * D;
    float2 x[W];
#pragma unroll
    for (int w = 0; w < W; ++w) x[w] = x0[w * kFastPitch];
#pragma unroll
    for (int m = 0; m < M; ++m) {
        const float* t = tp + m * tstride;
        float2 r;
        if (SUM == AVIRB200_SUM_DIL8) {
            float2 ln[8];
#pragma unroll
            for (int g = 0; g < FL / 8; ++g) {
                float tt[8];
                if (UNI) {
                    // one effective phase for the whole axis: taps are kernel parameters, i.e.
                    // constant-bank operands of the multiplies (no loads, no registers)
#pragma unroll
                    for (int q = 0; q < 8; ++q) tt[q] = p.rtaps[g * 8 + q];
                } else {
                    const float4 ta = *reinterpret_cast<const float4*>(t + g * 8);
                    const float4 tb = *reinterpret_cast<const float4*>(t + g * 8 + 4);
                    tt[0] = ta.x; tt[1] = ta.y; tt[2] = ta.z; tt[3] = ta.w;
                    tt[4] = tb.x; tt[5] = tb.y; tt[6] = tb.z; tt[7] = tb.w;
                }
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float2 v = f2mul(tt[q], x[m * D + g * 8 + q]);
                    ln[q] = (g == 0) ? v : f2add(ln[q], v);
                }
            }
            r = f2hadd8(ln);
        } else {
#pragma unroll
            for (int i = 0; i < FL; i += 2) {
                float2 t2;
                if (UNI) t2 = make_float2(p.rtaps[i], p.rtaps[i + 1]);
                else t2 = *reinterpret_cast<const float2*>(t + i);
                const float2 v0 = f2mul(t2.x, x[m * D + i]);
                r = (i == 0) ? v0 : f2add(r, v0);
                r = f2add(r, f2mul(t2.y, x[m * D + i + 1]));
            }
        }
        if (zero_start) r = f2add(r, make_float2(0.0f, 0.0f));
        out[m] = r;
    }
}

// De-interleaved RESIZE with long filters: group-major so that only 8 + (M-1)*D inputs and
// M x 8 lane accumulators are live at a time (a full register window would not fit).
template <int FL, int FLP, int D, int M>
__device__ __forceinline__ void resize_dil_groupmajor(const float2* x0, const float* tp, int tstride,
                                                      int zero_start, float2* out) {
    constexpr int W = 8 + (M - 1) * D;
    float2 ln[M][8];
#pragma unroll
    for (int g = 0; g < FL / 8; ++g) {
        float2 x[W];
#pragma unroll
        for (int w = 0; w < W; ++w) x[w] = x0[(g * 8 + w) * kFastPitch];
#pragma unroll
        for (int m = 0; m < M; ++m) {
            const float* t = tp + m * tstride + g * 8;
            const float4 ta = *reinterpret_cast<const float4*>(t);
            const float4 tb = *reinterpret_cast<const float4*>(t + 4);
            const float tt[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float2 v = f2mul(tt[q], x[m * D + q]);
                ln[m][q] = (g == 0) ? v : f2add(ln[m][q], v);
            }
        }
    }
#pragma unroll
    for (int m = 0; m < M; ++m) {
        float2 r = f2hadd8(ln[m]);
        if (zero_start) r = f2add(r, make_float2(0.0f, 0.0f));
        out[m] = r;
    }
}

// Interleaved RESIZE over the virtual 2X zero-stuffed line, upstream's doResize2
// (avir.h:4114-4328): only the 12 taps that land on real samples are accumulated; consecutive
// outputs advance by one virtual position, i.e. alternate between the even and the odd taps.
// ODD = parity of output 0's first virtual position; x0 = sample (p0 + parity) / 2.  Taps are
// the kernel-parameter constants (single effective phase).
template <bool ODD>
__device__ __forceinline__ void resize2_blocked(const FastParams& p, const float2* x0, int zero_start,
                                                float2* out) {
    constexpr int W = ODD ? 13 : 14;
    float2 x[W];
#pragma unroll
    for (int w = 0; w < W; ++w) x[w] = x0[w * kFastPitch];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
        constexpr int dummy = 0;
        (void)dummy;
        const int fo = ODD ? ((m & 1) ? 0 : 1) : (m & 1);
        const int base = ODD ? (m >> 1) : ((m + 1) >> 1);
        float2 r = f2mul(p.rtaps[fo], x[base]);
#pragma unroll
        for (int t = 1; t < 12; ++t) r = f2add(r, f2mul(p.rtaps[fo + 2 * t], x[base + t]));
        if (zero_start) r = f2add(r, make_float2(0.0f, 0.0f));
        out[m] = r;
    }
}

// FIR.  INL: folded symmetric form around the centre tap; DIL: full padded filter.
// `tt` = the NT taps in registers.
template <int SUM, int NT, int R, int M>
__device__ __forceinline__ void fir_blocked(const float2* x0, const float* tt, float2* out) {
    constexpr int W = NT + (M - 1) * R;
    float2 x[W];
#pragma unroll
    for (int w = 0; w < W; ++w) x[w] = x0[w * kFastPitch];
#pragma unroll
    for (int m = 0; m < M; ++m) {
        if (SUM == AVIRB200_SUM_DIL8) {
            float2 ln[8];
#pragma unroll
            for (int g = 0; g < NT / 8; ++g) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float2 v = f2mul(tt[g * 8 + q], x[m * R + g * 8 + q]);
                    ln[q] = (g == 0) ? v : f2add(ln[q], v);
                }
            }
            out[m] = f2hadd8(ln);
        } else {
            constexpr int L = NT / 2;
            float2 s = f2mul(tt[L], x[m * R + L]);
#pragma unroll
            for (int i = 1; i <= L; ++i)
                s = f2add(s, f2mul(tt[L + i], f2add(x[m * R + L + i], x[m * R + L - i])));
            out[m] = s;
        }
    }
}

// ---- plain-loop step routine: any geometry, one output ------------------------------------------
// `xb` = the thread's lane in the row of input position 0 of the tile-relative frame, i.e.
// xb[(n - tile_a) * kFastPitch] is sample n.

template <int SUM>
__device__ float2 step_simple(const FastStep& s, const float2* xb, int tile_a, int j, const float* tp) {
    if (s.kind == AVIRB200_STEP_FIR) {
        if (SUM == AVIRB200_SUM_INL) {
            const int L = s.latency;
            const float2* c = xb + ((j - s.edge) * s.resample - tile_a) * kFastPitch;
            float2 sum = f2mul(tp[L], c[0]);
            for (int i = 1; i <= L; ++i)
                sum = f2add(sum, f2mul(tp[L + i], f2add(c[i * kFastPitch], c[-i * kFastPitch])));
            return sum;
        }
        const float2* c = xb + ((j - s.edge) * s.resample - s.latency - tile_a) * kFastPitch;
        float2 ln[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) ln[q] = f2mul(tp[q], c[q * kFastPitch]);
        for (int i = 8; i < s.ntaps; i += 8) {
#pragma unroll
            for (int q = 0; q < 8; ++q) ln[q] = f2add(ln[q], f2mul(tp[i + q], c[(i + q) * kFastPitch]));
        }
        return f2hadd8(ln);
    }
    const int FL = s.ntaps;
    const int p = __ldg(s.src_pos + j) - (FL / 2 - 1);
    float2 r = make_float2(0.0f, 0.0f);
    if (SUM == AVIRB200_SUM_INL) {
        bool first = true;
        if (s.upsampled) {
            // only even virtual positions hold samples; upstream's doResize2 skips the rest
            for (int i = (p & 1); i < FL; i += 2) {
                const float2 v = f2mul(tp[i], xb[(((p + i) >> 1) - tile_a) * kFastPitch]);
                r = first ? v : f2add(r, v);
                first = false;
            }
        } else {
            const float2* c = xb + (p - tile_a) * kFastPitch;
            for (int i = 0; i < FL; ++i) {
                const float2 v = f2mul(tp[i], c[i * kFastPitch]);
                r = first ? v : f2add(r, v);
                first = false;
            }
        }
    } else {
        const float2* c = xb + (p - tile_a) * kFastPitch;
        float2 ln[8];
        for (int i = 0; i < FL; i += 8) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float2 v = f2mul(tp[i + q], c[(i + q) * kFastPitch]);
                ln[q] = (i == 0) ? v : f2add(ln[q], v);
            }
        }
        r = f2hadd8(ln);
    }
    if (s.zero_start) r = f2add(r, make_float2(0.0f, 0.0f));
    return r;
}

// ---- where a step's outputs go -----------------------------------------------------------------------
// TO_GLOBAL = last step of the column pass: output stage + store to the destination image;
// otherwise the shared tile of the step's output.

struct Sink {
    float2* ob;          // shared tile: row (j - oa), this thread's lane
    int oa;
    unsigned char* gp;   // image element (dst row 0, this thread's pixel / channel pair)
    size_t grow;         // bytes between image rows
    int grow_base;       // dst_row_base
    bool gok;
};

// EPI 1 = destination is float and there is no output gamma: the value is stored as is.
// EPI 2 = integer destination without output gamma: round, clamp, narrow -- and none of the
// double-precision sRGB code in the kernel (inlined at every store site it slowed the whole
// kernel down, see DESIGN.md section 4.3).  EPI 0 = everything, decided at run time.
template <bool TO_GLOBAL, int EPI>
__device__ __forceinline__ void sink_store(const FastParams& p, const Sink& k, int j, float2 v, int c0) {
    if (!TO_GLOBAL) {
        k.ob[(j - k.oa) * kFastPitch] = v;
        return;
    }
    if (EPI == 1) {
        if (k.gok) *reinterpret_cast<float2*>(k.gp + (size_t)(j - k.grow_base) * k.grow) = v;
        return;
    }
    if (EPI == 2) {
        if (!k.gok) return;
        unsigned char* g2 = k.gp + (size_t)(j - k.grow_base) * k.grow;
        // (no bit-depth truncation, fast_launch(): one rounding conversion per sample, clamp and
        // narrow in integers, selects and predicated stores instead of branches)
        const int pk = (int)p.px.pk_out;
        const int a = imin(imax(round_out_int(v.x, p.px.round_mode), 0), pk);
        const int b = imin(imax(round_out_int(v.y, p.px.round_mode), 0), pk);
        const bool narrow = (p.dst_type == AVIRB200_U8);
        if (narrow) *reinterpret_cast<unsigned short*>(g2) = (unsigned short)(a | (b << 8));
        if (!narrow) *reinterpret_cast<unsigned*>(g2) = (unsigned)a | ((unsigned)b << 16);
        return;
    }
    v.x = epilogue_value_c4(p, v.x, c0);
    v.y = epilogue_value_c4(p, v.y, c0 + 1);
    if (!k.gok) return;
    unsigned char* g = k.gp + (size_t)(j - k.grow_base) * k.grow;
    if (p.dst_type == AVIRB200_F32) *reinterpret_cast<float2*>(g) = v;
    else if (p.dst_type == AVIRB200_U8)
        *reinterpret_cast<uchar2*>(g) = make_uchar2((unsigned char)v.x, (unsigned char)v.y);
    else
        *reinterpret_cast<ushort2*>(g) = make_ushort2((unsigned short)v.x, (unsigned short)v.y);
}

// ---- one step for one warp ------------------------------------------------------------------------------

// VAR / CT: compile-time step variant and constant-tap flag of the chain-specialised kernels
// (-1 = decide at run time from the step record: the chain-generic kernel).
template <int SUM, bool TO_GLOBAL, int VAR, int CT, int EPI>
__device__ __forceinline__ void run_step(const FastParams& p, const FastStep& s, const float2* xb,
                                         int tile_a, const Range out, const Range dom,
                                         const float* stp, int uni, bool const_taps_rt, int sp_first,
                                         int spacing_ok, const Sink& k, int warp, int c0) {
    const int variant = (VAR >= 0) ? VAR : s.variant;
    const bool const_taps = (CT >= 0) ? (CT == 1) : const_taps_rt;
    // balanced split of the tile's outputs over the warps, in units of 4
    const int on = out.b - out.a + 1;
    const int units = (on + 3) >> 2;
    const int jb = out.a + 4 * ((units * warp) / kFastWarps);
    const int je = imin(out.a + 4 * ((units * (warp + 1)) / kFastWarps), out.a + on);
    if (jb >= je) return;

    // region [bl, bh) the blocked routine may cover: in-domain, whole quads, right geometry
    const int bl = imax(jb, dom.a), bh = imin(je, dom.b + 1);
    int nq = 0, p0 = 0;
    if (variant != kVarSimple && bh - bl >= 4) {
        nq = (bh - bl) >> 2;
        if (s.kind == AVIRB200_STEP_RESIZE) {
            // the host checked the tile's in-domain outputs for the uniform source step the
            // templates assume (spacing_ok = that step, 0 = irregular) and tabulated the first
            // position, so no position look-ups are needed here
            const int D = (variant == kVarResizeDil56D4) ? 4 : (variant == kVarResize2Inl24 ? 1 : 2);
            if (variant == kVarResize2Inl24 && !const_taps) nq = 0;
            if (spacing_ok != D) nq = 0;
            p0 = sp_first + (bl - dom.a) * D - (s.ntaps / 2 - 1);
        } else {
            p0 = (bl - s.edge) * s.resample - s.latency; // first input of output bl (both forms)
        }
    }
    const int tstr = uni ? 0 : s.ntaps_pad; // RESIZE: staged row (j - dom.a), or one shared row

    auto simple_one = [&](int j) {
        const int jj = imin(imax(j, dom.a), dom.b); // edge replica: value of the clamped output
        const float* tp = (s.kind == AVIRB200_STEP_FIR) ? stp : stp + (size_t)(jj - dom.a) * tstr;
        sink_store<TO_GLOBAL, EPI>(p, k, j, step_simple<SUM>(s, xb, tile_a, jj, tp), c0);
    };

    int j = jb;
    const int head_end = (nq > 0) ? bl : je;
    for (; j < head_end; ++j) simple_one(j);
    if (nq > 0) {
        const float2* x0 = xb + (p0 - tile_a) * kFastPitch;
        if (variant == kVarResize2Inl24) x0 = xb + (((p0 + (p0 & 1)) >> 1) - tile_a) * kFastPitch;
        const float* tp = stp + (size_t)(bl - dom.a) * tstr;
        float2 o4[4];
#define AVB_QUAD_LOOP(CALL, XSTEP, TSTEP)                                                         \
    for (int q = 0; q < nq; ++q) {                                                                \
        CALL;                                                                                     \
        _Pragma("unroll") for (int m = 0; m < 4; ++m) sink_store<TO_GLOBAL, EPI>(p, k, j + m, o4[m], c0); \
        j += 4;                                                                                   \
        x0 += (XSTEP) * kFastPitch;                                                               \
        tp += (TSTEP);                                                                            \
    }
#define AVB_RESIZE_CASE(SUMM, FL, FLP)                                                                          \
    if (const_taps) {                                                                                           \
        AVB_QUAD_LOOP((resize_blocked<SUMM, FL, FLP, 2, 4, true>(p, x0, tp, 0, s.zero_start, o4)), 8, 0)        \
    } else {                                                                                                    \
        AVB_QUAD_LOOP((resize_blocked<SUMM, FL, FLP, 2, 4, false>(p, x0, tp, tstr, s.zero_start, o4)), 8, 4 * tstr) \
    }
        switch (variant) {
        case kVarResizeDil24D2: AVB_RESIZE_CASE(AVIRB200_SUM_DIL8, 24, 24) break;
        case kVarResizeDil32D2: AVB_RESIZE_CASE(AVIRB200_SUM_DIL8, 32, 32) break;
        case kVarResizeInl18D2: AVB_RESIZE_CASE(AVIRB200_SUM_INL, 18, 20) break;
        case kVarResizeInl24D2: AVB_RESIZE_CASE(AVIRB200_SUM_INL, 24, 24) break;
        case kVarResize2Inl24:
            if (p0 & 1) {
                AVB_QUAD_LOOP((resize2_blocked<true>(p, x0, s.zero_start, o4)), 2, 0)
            } else {
                AVB_QUAD_LOOP((resize2_blocked<false>(p, x0, s.zero_start, o4)), 2, 0)
            }
            break;
        case kVarResizeDil56D4:
            AVB_QUAD_LOOP((resize_dil_groupmajor<56, 56, 4, 2>(x0, tp, tstr, s.zero_start, o4),
                           resize_dil_groupmajor<56, 56, 4, 2>(x0 + 8 * kFastPitch, tp + 2 * tstr, tstr, s.zero_start, o4 + 2)),
                          16, 4 * tstr)
            break;
        case kVarFirDil8R1: {
            float tt[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) tt[i] = stp[i];
            AVB_QUAD_LOOP((fir_blocked<AVIRB200_SUM_DIL8, 8, 1, 4>(x0, tt, o4)), 4, 0)
            break;
        }
        case kVarFirInl7R1: {
            float tt[7];
#pragma unroll
            for (int i = 0; i < 7; ++i) tt[i] = stp[i];
            AVB_QUAD_LOOP((fir_blocked<AVIRB200_SUM_INL, 7, 1, 4>(x0, tt, o4)), 4, 0)
            break;
        }
        case kVarFirInl15R2: {
            float tt[15];
#pragma unroll
            for (int i = 0; i < 15; ++i) tt[i] = stp[i];
            AVB_QUAD_LOOP((fir_blocked<AVIRB200_SUM_INL, 15, 2, 4>(x0, tt, o4)), 8, 0)
            break;
        }
        default:
            break;
        }
#undef AVB_RESIZE_CASE
#undef AVB_QUAD_LOOP
        for (; j < je; ++j) simple_one(j);
    }
}

// ---- source tile staging ----

template <bool IS_V>
__device__ __forceinline__ void stage_source(const FastParams& p, float2* buf, const int* tr,
                                             int line0, int nlines, int tid) {
    const int a = tr[0], n = tr[1] - a + 1; // tile record (shared memory)
    if (IS_V) {
        // a "line" is a pixel column; 16 pixels = 64 contiguous floats of a row
        const float* src = static_cast<const float*>(p.src);
        const int q = imin(tid & 15, nlines - 1); // pixel within the strip (float4)
        const int r0 = tid >> 4;                  // 16 rows per sweep
        float2* d = buf + r0 * kFastPitch + (tid & 15) * 2;
        if (a >= 0 && a + n <= p.ax.src_len) {
            // interior tile: no edge replication, pointers advance by constants
            const float4* g = reinterpret_cast<const float4*>(src + (size_t)(a + r0 - p.src_row_base) * p.src_pitch) + line0 + q;
            const size_t gstep = (size_t)(kFastThreads / 16) * (p.src_pitch / 4);
            for (int pos = r0; pos < n; pos += kFastThreads / 16) {
                cp_async16(d, g);
                d += (kFastThreads / 16) * kFastPitch;
                g += gstep;
            }
        } else {
            for (int pos = r0; pos < n; pos += kFastThreads / 16) {
                const int y = imin(imax(a + pos, 0), p.ax.src_len - 1) - p.src_row_base;
                cp_async16(d, reinterpret_cast<const float4*>(src + (size_t)y * p.src_pitch) + line0 + q);
                d += (kFastThreads / 16) * kFastPitch;
            }
        }
        return;
    }
    const int px = tid & 31; // 32 consecutive positions per sweep
    const int r0 = tid >> 5; // 8 rows per sweep
    for (int r = r0; r < kFastLines; r += kFastThreads / 32) {
        const size_t rowoff = (size_t)(line0 + imin(r, nlines - 1)) * p.src_pitch;
        if (p.src_type == AVIRB200_F32) {
            const float4* srow = reinterpret_cast<const float4*>(static_cast<const float*>(p.src) + rowoff) - p.src_row_base;
            float2* d = buf + px * kFastPitch + r * 2;
            if (a >= 0 && a + n <= p.ax.src_len) {
                const float4* g = srow + a + px; // interior tile: constant strides
                for (int pos = px; pos < n; pos += 32) {
                    cp_async16(d, g);
                    d += 32 * kFastPitch;
                    g += 32;
                }
            } else {
                for (int pos = px; pos < n; pos += 32) {
                    const int x = imin(imax(a + pos, 0), p.ax.src_len - 1);
                    cp_async16(d, srow + x);
                    d += 32 * kFastPitch;
                }
            }
        } else {
            for (int pos = px; pos < n; pos += 32) {
                const int x = imin(imax(a + pos, 0), p.ax.src_len - 1) - p.src_row_base;
                float4 v;
                if (p.src_type == AVIRB200_U8) {
                    const uchar4 b = __ldg(reinterpret_cast<const uchar4*>(static_cast<const unsigned char*>(p.src) + rowoff) + x);
                    v = make_float4((float)b.x, (float)b.y, (float)b.z, (float)b.w);
                    if (p.px.gamma_in) {
                        const int ai = p.px.alpha_index;
                        v.x = (ai == 0) ? __fmul_rn(v.x, p.px.in_gamma_mult) : p.px.srgb_lut[b.x];
                        v.y = p.px.srgb_lut[b.y];
                        v.z = p.px.srgb_lut[b.z];
                        v.w = (ai == 3) ? __fmul_rn(v.w, p.px.in_gamma_mult) : p.px.srgb_lut[b.w];
                    }
                } else {
                    const ushort4 b = __ldg(reinterpret_cast<const ushort4*>(static_cast<const unsigned short*>(p.src) + rowoff) + x);
                    v = make_float4((float)b.x, (float)b.y, (float)b.z, (float)b.w);
                    if (p.px.gamma_in) {
                        const int ai = p.px.alpha_index;
                        v.x = (ai == 0) ? __fmul_rn(v.x, p.px.in_gamma_mult) : srgb2lin(v.x, p.px.in_gamma_mult);
                        v.y = srgb2lin(v.y, p.px.in_gamma_mult);
                        v.z = srgb2lin(v.z, p.px.in_gamma_mult);
                        v.w = (ai == 3) ? __fmul_rn(v.w, p.px.in_gamma_mult) : srgb2lin(v.w, p.px.in_gamma_mult);
                    }
                }
                *reinterpret_cast<float4*>(buf + pos * kFastPitch + r * 2) = v;
            }
        }
    }
}

// ---- integer sources (row pass): raw pixels stream in asynchronously, converted in shared memory --
// Raw layout: [position][line] of one pixel (uchar4 / ushort4).

template <int BYTES>
__device__ __forceinline__ void cp_async_small(void* smem, const void* gmem) {
    const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(sa), "l"(gmem), "n"(BYTES));
}

__device__ __forceinline__ void stage_raw(const FastParams& p, unsigned char* raw, const int* tr, int line0,
                                          int nlines, int tid) {
    const int a = tr[0], n = tr[1] - a + 1;
    const int px = tid & 31, r0 = tid >> 5;
    const int pb = (p.src_type == AVIRB200_U8) ? 4 : 8; // bytes per pixel
    for (int r = r0; r < kFastLines; r += kFastThreads / 32) {
        const unsigned char* srow = static_cast<const unsigned char*>(p.src) +
                                    (size_t)(line0 + imin(r, nlines - 1)) * p.src_pitch * (pb / 4);
        for (int pos = px; pos < n; pos += 32) {
            const int x = imin(imax(a + pos, 0), p.ax.src_len - 1) - p.src_row_base;
            unsigned char* d = raw + ((size_t)pos * kFastLines + r) * pb;
            if (pb == 4) cp_async_small<4>(d, srow + (size_t)x * 4);
            else cp_async_small<8>(d, srow + (size_t)x * 8);
        }
    }
}

// packScanline on the staged raw tile (avir.h:2777-2971): (float) cast, or sRGB linearisation.
__device__ __forceinline__ void convert_raw(const FastParams& p, const unsigned char* raw, float2* buf,
                                            const float* lut, int n, int tid) {
    for (int idx = tid; idx < n * kFastLines; idx += kFastThreads) {
        const int pos = idx >> 4, r = idx & (kFastLines - 1);
        float4 v;
        if (p.src_type == AVIRB200_U8) {
            const uchar4 b = reinterpret_cast<const uchar4*>(raw)[idx];
            v = make_float4((float)b.x, (float)b.y, (float)b.z, (float)b.w);
            if (p.px.gamma_in) {
                const int ai = p.px.alpha_index;
                v.x = (ai == 0) ? __fmul_rn(v.x, p.px.in_gamma_mult) : lut[b.x];
                v.y = lut[b.y];
                v.z = lut[b.z];
                v.w = (ai == 3) ? __fmul_rn(v.w, p.px.in_gamma_mult) : lut[b.w];
            }
        } else {
            const ushort4 b = reinterpret_cast<const ushort4*>(raw)[idx];
            v = make_float4((float)b.x, (float)b.y, (float)b.z, (float)b.w);
            if (p.px.gamma_in) {
                const int ai = p.px.alpha_index;
                v.x = (ai == 0) ? __fmul_rn(v.x, p.px.in_gamma_mult) : srgb2lin(v.x, p.px.in_gamma_mult);
                v.y = srgb2lin(v.y, p.px.in_gamma_mult);
                v.z = srgb2lin(v.z, p.px.in_gamma_mult);
                v.w = (ai == 3) ? __fmul_rn(v.w, p.px.in_gamma_mult) : srgb2lin(v.w, p.px.in_gamma_mult);
            }
        }
        *reinterpret_cast<float4*>(buf + pos * kFastPitch + r * 2) = v;
    }
}

// ---- the kernel ------------------------------------------------------------------------------------------
// One block = one tile: 16 lines x tile_out final outputs.  blockIdx.x walks along the line so
// that concurrently resident blocks share their halo reads through L2.
//
// Tile record (host-built, kTileRec ints):
//   [0..9]   (a, b) of the source tile and of every step's output tile
//   [10..13] first source position of each resize step's in-domain outputs
//   [14..17] uniform source step of those outputs (0 = irregular)

// NS/V0..V2/CTS: chain known at compile time (steps, their variants, which step has its taps
// in the kernel parameters); NS = -1 is the chain-generic kernel.  Specialising removes the
// per-step variant dispatch, the indexed parameter loads and most of the code the generic
// kernel drags through the instruction cache.
template <int SUM, bool IS_V, int NS, int V0, int V1, int V2, int CTS, int EPI>
__global__ void __launch_bounds__(kFastThreads, kFastBlocksPerSM)
fast_pass_kernel(const __grid_constant__ FastParams p) {
    // Persistent: a block walks over tiles (tile index = line block * tiles_per_line + tile
    // along the line, strided by the grid, so concurrently running blocks work on neighbouring
    // tiles and share halos through L2).  The source of the NEXT tile streams into the second
    // source buffer (cp.async) while the current tile computes, so HBM stays busy during the
    // arithmetic instead of the whole GPU alternating between a load phase and a math phase.
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // integer sources are converted into the float tile every iteration, so only their raw
    // pixel tiles are double-buffered and one float source buffer suffices
    const bool one_a = !IS_V && (p.src_type != AVIRB200_F32);
    float2* bufA0 = reinterpret_cast<float2*>(smem_raw);
    float2* bufA1 = one_a ? bufA0 : bufA0 + (size_t)p.span_a * kFastPitch;
    float2* bufB = bufA1 + (size_t)p.span_a * kFastPitch;
    float* stap = reinterpret_cast<float*>(bufB + (size_t)p.span_b * kFastPitch);
    // integer sources: two raw pixel tiles behind the taps (16-byte aligned: taps are padded)
    unsigned char* raw0 = reinterpret_cast<unsigned char*>(stap + p.taps_floats);
    unsigned char* raw1 = raw0 + (size_t)p.span_a * kFastLines * 8;
    __shared__ __align__(16) int srec[3][kTileRec];
    __shared__ float slut[256];

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int warp = tid >> 5;
    const int ns = (NS > 0) ? NS : p.ax.nsteps;
    const int tiles_x = (p.out1 - p.out0 + p.tile_out - 1) / p.tile_out;
    const int total = tiles_x * ((p.n_lines + kFastLines - 1) / kFastLines);
    const bool async_src = IS_V || (p.src_type == AVIRB200_F32);
    const bool raw_src = !IS_V && (p.src_type != AVIRB200_F32);
    const int G = gridDim.x;

    int t = blockIdx.x;
    if (t >= total) return;

    // taps that do not depend on the tile: FIR filters, single-phase resize steps
    for (int i = 0; i < ns; ++i) {
        const FastStep& s = p.ax.s[i];
        float* st = stap + p.tap_off[i];
        if (s.kind == AVIRB200_STEP_FIR) {
            for (int q = tid; q < s.ntaps; q += kFastThreads) st[q] = __ldg(s.taps + q);
        } else if (p.uniform_taps[i]) {
            for (int q = tid; q < s.ntaps_pad; q += kFastThreads) st[q] = __ldg(s.taps + q);
        }
    }
    if (raw_src && p.px.gamma_in && p.src_type == AVIRB200_U8)
        for (int q = tid; q < 256; q += kFastThreads) slut[q] = __ldg(p.px.srgb_lut + q);
    // records of the first two tiles
    if (tid < kTileRec) {
        srec[0][tid] = __ldg(p.tile_ranges + (size_t)(t % tiles_x) * kTileRec + tid);
        if (t + G < total) srec[1][tid] = __ldg(p.tile_ranges + (size_t)((t + G) % tiles_x) * kTileRec + tid);
    }
    __syncthreads();
    if (async_src && p.debug != 2) {
        const int lb = t / tiles_x;
        stage_source<IS_V>(p, bufA0, srec[0], lb * kFastLines, imin(kFastLines, p.n_lines - lb * kFastLines), tid);
    }
    if (raw_src) {
        const int lb = t / tiles_x;
        stage_raw(p, raw0, srec[0], lb * kFastLines, imin(kFastLines, p.n_lines - lb * kFastLines), tid);
    }
    const int c0 = (lane & 1) * 2; // first channel of this lane's pair
    const size_t esz = (p.dst_type == AVIRB200_F32 ? 4 : (p.dst_type == AVIRB200_U16 ? 2 : 1));

    for (int it = 0; t < total; t += G, ++it) {
        const int lb = t / tiles_x;
        const int line0 = lb * kFastLines;
        const int nlines = imin(kFastLines, p.n_lines - line0);
        const int* tr = srec[it % 3];
        float2* bufA = (it & 1) ? bufA1 : bufA0;
        auto rng = [&](int i) { return Range{tr[2 * i], tr[2 * i + 1]}; };

        // per-tile tap rows of resize steps with varying phases
        for (int i = 0; i < ns; ++i) {
            const FastStep& s = p.ax.s[i];
            if (s.kind == AVIRB200_STEP_FIR || p.uniform_taps[i]) continue;
            float* st = stap + p.tap_off[i];
            const Range dom = clampr(rng(i + 1), 0, s.out_len);
            const int rows = dom.b - dom.a + 1;
            const int fl4 = s.ntaps_pad >> 2;
            for (int q = tid; q < rows * fl4; q += kFastThreads) {
                const int rr = q / fl4, c4 = q - rr * fl4;
                const int e = __ldg(s.eff + dom.a + rr);
                reinterpret_cast<float4*>(st)[q] =
                    __ldg(reinterpret_cast<const float4*>(s.taps + (size_t)e * s.ntaps_pad) + c4);
            }
        }
        cp_async_wait_all(); // this tile's source and the next tile's record have landed
        __syncthreads();

        // prefetch: record of the tile after next, source of the next tile
        if (t + 2 * G < total && tid < kTileRec / 4)
            cp_async16(&srec[(it + 2) % 3][tid * 4],
                       p.tile_ranges + (size_t)((t + 2 * G) % tiles_x) * kTileRec + tid * 4);
        if (async_src && t + G < total && p.debug != 2) {
            const int lbn = (t + G) / tiles_x;
            stage_source<IS_V>(p, (it & 1) ? bufA0 : bufA1, srec[(it + 1) % 3], lbn * kFastLines,
                               imin(kFastLines, p.n_lines - lbn * kFastLines), tid);
        }

        if (raw_src) {
            if (t + G < total) {
                const int lbn = (t + G) / tiles_x;
                stage_raw(p, (it & 1) ? raw0 : raw1, srec[(it + 1) % 3], lbn * kFastLines,
                          imin(kFastLines, p.n_lines - lbn * kFastLines), tid);
            }
            convert_raw(p, (it & 1) ? raw1 : raw0, bufA, slut, tr[1] - tr[0] + 1, tid);
            __syncthreads();
        }

        // ---- the chain: source(A) -> B -> A -> B ...
        Sink k;
        k.gok = (lane >> 1) < nlines;
        k.grow = (size_t)p.dst_pitch * esz;
        k.grow_base = p.dst_row_base;
        k.gp = static_cast<unsigned char*>(p.dst) + ((size_t)(line0 + (lane >> 1)) * 4 + c0) * esz;
#define AVB_CHAIN_STEP(I, VARI, CTI)                                                                      \
    {                                                                                                  \
        const FastStep& s = p.ax.s[I];                                                                 \
        const float2* xb = (((I) & 1) ? bufB : bufA) + lane;                                           \
        const Range ro = rng((I) + 1);                                                                 \
        k.ob = (((I) & 1) ? bufA : bufB) + lane;                                                       \
        k.oa = ro.a;                                                                                   \
        if (p.debug == 1) {                                                                            \
        } else if (IS_V && (I) == ns - 1)                                                              \
            run_step<SUM, true, VARI, CTI, EPI>(                                                            \
                p, s, xb, tr[2 * (I)], ro, clampr(ro, 0, s.out_len), stap + p.tap_off[I],              \
                p.uniform_taps[I], p.rtaps_step == (I), tr[10 + (I)], tr[14 + (I)], k, warp, c0);      \
        else                                                                                           \
            run_step<SUM, false, VARI, CTI, 0>(                                                           \
                p, s, xb, tr[2 * (I)], ro, clampr(ro, 0, s.out_len), stap + p.tap_off[I],              \
                p.uniform_taps[I], p.rtaps_step == (I), tr[10 + (I)], tr[14 + (I)], k, warp, c0);      \
        __syncthreads();                                                                               \
    }
        if (NS > 0) {
            AVB_CHAIN_STEP(0, V0, (CTS == 0 ? 1 : 0))
            if (NS > 1) AVB_CHAIN_STEP(1, V1, (CTS == 1 ? 1 : 0))
            if (NS > 2) AVB_CHAIN_STEP(2, V2, (CTS == 2 ? 1 : 0))
        } else {
            for (int i = 0; i < ns; ++i) AVB_CHAIN_STEP(i, -1, -1)
        }
#undef AVB_CHAIN_STEP

        if (!IS_V && p.debug != 3) {
            // coalesced store of the row-pass tile: [pos][row] in shared -> rows of float4 pixels
            const float2* ob = (ns & 1) ? bufB : bufA;
            const Range ro = rng(ns);
            const int on = ro.b - ro.a + 1;
            const int px = tid & 31, r0 = tid >> 5;
            for (int r = r0; r < nlines; r += kFastThreads / 32) {
                float4* drow = reinterpret_cast<float4*>(static_cast<float*>(p.dst) +
                                                         (size_t)(line0 + r) * p.dst_pitch) - p.dst_row_base;
                for (int pos = px; pos < on; pos += 32)
                    drow[ro.a + pos] = *reinterpret_cast<const float4*>(ob + pos * kFastPitch + r * 2);
            }
        }
        // (the next iteration's first barrier orders these reads before the buffer's reuse)
    }
}

#endif // __CUDACC__

} // namespace avb
