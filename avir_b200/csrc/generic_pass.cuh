// generic_pass.cuh -- the fully plan-driven pass kernel (sm_90a).
//
// One kernel runs a whole 1-D filtering chain (any mix of FIR / filtered-upsample / resize
// steps, either summation order) for a tile of "lines":
//   row pass    : a line is an image row, lanes = rows-in-block x channels
//   column pass : a line is an image column, lanes = columns-in-block x channels
// A tile of the source lines is staged in shared memory as [position][lane] (so that all
// threads of a warp read consecutive words = no bank conflicts), every intermediate step
// writes its outputs for the tile into the other shared buffer, the last step goes to HBM.
// Each step clamps reads to ITS OWN input line, exactly as upstream replicates edges per
// step (avir.h:3227-3239) -- clamping at the image border only would not be equivalent.
//
// This kernel is the universal path: every chain the planner can emit, 1-4 channels.
// The hot BASELINE chains have specialised kernels (fast_pass.cuh) with identical
// arithmetic; tests compare both against the oracle.
//
// Arithmetic rules (bit-exactness): products and sums are separate IEEE RN operations
// (__fmul_rn/__fadd_rn; the file is also compiled with -fmad=false), in upstream's order.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "device_plan.h"
#include "pixel_ops.cuh"

namespace avb {

struct PassParams {
    DevAxis ax;
    int sum_mode;   // avirb200_sum_mode
    int is_v;       // 0 row pass, 1 column pass
    int channels;
    int n_lines;    // lines in this launch (rows for H, columns for V)
    int lines_per_block;
    int tile_out;   // final outputs per tile
    int out0, out1; // final outputs [out0, out1) to produce (column pass on a shard, either pass of a window)
    int span_a;     // shared rows of buffer 0 (buffer 1 follows it; pass_config.h)
    int pitch;      // shared row pitch in floats (odd)
    // source image / intermediate
    const void* src;
    long long src_pitch;  // elements between consecutive rows
    int src_type;         // avirb200_dtype (column pass: always F32)
    int src_row_base;     // global position of the buffer's position 0 (column pass: row; row pass: column)
    // destination
    void* dst;
    long long dst_pitch;
    int dst_type;
    int dst_row_base;     // global output stored at the destination's position 0 (column pass: row; row pass: column)
    PixelStage px;        // prologue / epilogue
};

__device__ __forceinline__ float epilogue_value(const PassParams& p, float v, int c) {
    if (p.px.gamma_out) {
        if (p.channels == 4 && c == p.px.alpha_index) v = __fmul_rn(v, p.px.out_gamma_mult);
        else v = __fmul_rn(lin2srgb(v), p.px.out_gamma_mult);
    }
    if (p.dst_type != AVIRB200_F32) {
        if (p.px.tr_mul == 1.0f) v = round_out(v, p.px.round_mode);
        else v = __fmul_rn(round_out(__fmul_rn(v, p.px.tr_mul_inv), p.px.round_mode), p.px.tr_mul);
        v = v < 0.0f ? 0.0f : (v > p.px.pk_out ? p.px.pk_out : v);
    }
    return v;
}

__device__ __forceinline__ float load_source(const PassParams& p, long long idx, int c) {
    float raw;
    if (p.src_type == AVIRB200_U8) {
        const unsigned char b = ((const unsigned char*)p.src)[idx];
        if (p.px.gamma_in && !(p.channels == 4 && c == p.px.alpha_index)) return p.px.srgb_lut[b];
        raw = (float)b;
    } else if (p.src_type == AVIRB200_U16) {
        raw = (float)((const unsigned short*)p.src)[idx];
    } else {
        raw = ((const float*)p.src)[idx];
    }
    if (!p.px.gamma_in) return raw;
    if (p.channels == 4 && c == p.px.alpha_index) return __fmul_rn(raw, p.px.in_gamma_mult);
    return srgb2lin(raw, p.px.in_gamma_mult);
}

// ---- one output sample of one step ----------------------------------------------------------

struct TileView {
    const float* buf; // shared, [pos - a][lane]
    int a;            // first position held
    int lo, hi;       // valid index range of the line [lo, hi)
    int pitch;
};

__device__ __forceinline__ float tv(const TileView& t, int n, int lane) {
    n = imin(imax(n, t.lo), t.hi - 1);
    return t.buf[(n - t.a) * t.pitch + lane];
}

__device__ __forceinline__ float hadd8(const float* v) {
    return __fadd_rn(__fadd_rn(__fadd_rn(v[0], v[4]), __fadd_rn(v[1], v[5])),
                     __fadd_rn(__fadd_rn(v[2], v[6]), __fadd_rn(v[3], v[7])));
}

template <int SUM>
__device__ float step_sample(const DevStep& s, const TileView& in, int j, int lane) {
    if (s.kind == AVIRB200_STEP_FIR) {
        if (SUM == AVIRB200_SUM_INL) {
            const int L = s.latency;
            const float* f = s.taps + L;
            const int p = (j - s.edge) * s.resample;
            float sum = __fmul_rn(__ldg(f), tv(in, p, lane));
            for (int i = 1; i <= L; ++i)
                sum = __fadd_rn(sum, __fmul_rn(__ldg(f + i),
                                               __fadd_rn(tv(in, p + i, lane), tv(in, p - i, lane))));
            return sum;
        } else {
            const int p = (j - s.edge) * s.resample - s.latency;
            float ln[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) ln[q] = __fmul_rn(__ldg(s.taps + q), tv(in, p + q, lane));
            for (int i = 8; i < s.ntaps; i += 8) {
#pragma unroll
                for (int q = 0; q < 8; ++q)
                    ln[q] = __fadd_rn(ln[q], __fmul_rn(__ldg(s.taps + i + q),
                                                       tv(in, p + i + q, lane)));
            }
            return hadd8(ln);
        }
    }
    if (s.kind == AVIRB200_STEP_RESIZE) {
        const int FL = s.ntaps;
        const float* c0 = s.taps + (size_t)__ldg(s.phase + j) * FL * (s.order + 1);
        const float* c1 = c0 + FL;
        const float x = __ldg(s.frac + j);
        const int p = __ldg(s.src_pos + j) - (FL / 2 - 1);
        if (SUM == AVIRB200_SUM_INL) {
            float sum = 0.0f;
            bool first = !s.zero_start;
            for (int i = 0; i < FL; ++i) {
                const int n = p + i;
                float xv;
                if (s.upsampled) {
                    if (n & 1) {
                        if (s.skip_odd) continue;
                        xv = 0.0f;
                    } else {
                        xv = tv(in, n >> 1, lane);
                    }
                } else {
                    xv = tv(in, n, lane);
                }
                float t = __ldg(c0 + i);
                if (s.order) t = __fadd_rn(t, __fmul_rn(__ldg(c1 + i), x));
                const float v = __fmul_rn(t, xv);
                if (first) { sum = v; first = false; }
                else sum = __fadd_rn(sum, v);
            }
            return sum;
        } else {
            float ln[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) ln[q] = 0.0f;
            for (int i = 0; i < FL; i += 8) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int n = p + i + q;
                    float xv;
                    if (s.upsampled) xv = (n & 1) ? 0.0f : tv(in, n >> 1, lane);
                    else xv = tv(in, n, lane);
                    float t = __ldg(c0 + i + q);
                    if (s.order) t = __fadd_rn(t, __fmul_rn(__ldg(c1 + i + q), x));
                    const float v = __fmul_rn(t, xv);
                    if (i == 0 && !s.zero_start) ln[q] = v;
                    else ln[q] = __fadd_rn(ln[q], v);
                }
            }
            return hadd8(ln);
        }
    }
    // filtered 2X upsample, gather form of upstream's scatter (avir.h:3404-3733): terms in
    // order of increasing input index, then suffix tail, then prefix tail.
    {
        const int R = s.resample;
        const int first_m = -s.in_prefix;
        const int last_m = s.in_len - 1 + s.in_suffix;
        int m_lo = floordiv(j + s.latency - (s.ntaps - 1) + R - 1, R);
        int m_hi = floordiv(j + s.latency, R);
        m_lo = imax(m_lo, first_m);
        m_hi = imin(m_hi, last_m);
        float sum = 0.0f;
        for (int m = m_lo; m <= m_hi; ++m)
            sum = __fadd_rn(sum, __fmul_rn(__ldg(s.taps + (j - m * R + s.latency)),
                                           tv(in, m, lane)));
        const int sfx = (last_m + 1) * R - s.latency;
        const int pfx = -s.in_prefix * R;
        if (j >= sfx && j < sfx + s.n_suffix_dc)
            sum = __fadd_rn(sum, __fmul_rn(tv(in, s.in_len - 1, lane), __ldg(s.suffix_dc + (j - sfx))));
        if (j >= pfx && j < pfx + s.n_prefix_dc)
            sum = __fadd_rn(sum, __fmul_rn(tv(in, 0, lane), __ldg(s.prefix_dc + (j - pfx))));
        return sum;
    }
}

// ---- the kernel -------------------------------------------------------------------------------

// The tile of final outputs [j0, j1] of the lines [line0, line0 + nlines), every thread of the block.
template <int SUM>
__device__ __forceinline__ void generic_tile(const PassParams& p, float* const bufs[2], int line0, int nlines,
                                             int j0, int j1) {
    const int C = p.channels;
    const int NL = nlines * C;

    // Ranges every step must produce for this tile (uniform; a few integer ops).
    Range rng[AVIRB200_MAX_STEPS + 1];
    const int ns = p.ax.nsteps;
    rng[ns].a = j0;
    rng[ns].b = j1;
    for (int i = ns - 1; i >= 0; --i)
        rng[i] = step_input_range(p.ax.steps[i], rng[i + 1], p.ax.steps[i].src_pos);

    // Stage the source tile: positions rng[0], all lanes.
    {
        const int a = rng[0].a, n = rng[0].b - rng[0].a + 1;
        float* b0 = bufs[0];
        if (p.is_v) {
            // lanes are contiguous floats of an intermediate row
            for (int idx = threadIdx.x; idx < n * NL; idx += blockDim.x) {
                const int pos = idx / NL, lane = idx - pos * NL;
                const long long g = (long long)(a + pos - p.src_row_base) * p.src_pitch +
                                    (long long)line0 * C + lane;
                b0[pos * p.pitch + lane] = ((const float*)p.src)[g];
            }
        } else {
            // consecutive threads walk along x (coalesced); shared pitch is odd
            const int rowlen = n * C;
            for (int idx = threadIdx.x; idx < nlines * rowlen; idx += blockDim.x) {
                const int r = idx / rowlen, e = idx - r * rowlen;
                const int pos = e / C, c = e - pos * C;
                const long long g = (long long)(line0 + r) * p.src_pitch + (long long)(a + pos - p.src_row_base) * C + c;
                b0[pos * p.pitch + r * C + c] = load_source(p, g, c);
            }
        }
    }
    __syncthreads();

    for (int i = 0; i < ns; ++i) {
        const DevStep& s = p.ax.steps[i];
        TileView in;
        in.buf = bufs[i & 1];
        in.a = rng[i].a;
        in.lo = s.in_lo;
        in.hi = s.in_hi;
        in.pitch = p.pitch;
        const int oa = rng[i + 1].a, on = rng[i + 1].b - rng[i + 1].a + 1;
        const bool last = (i == ns - 1);
        float* ob = bufs[(i + 1) & 1];
        for (int idx = threadIdx.x; idx < on * NL; idx += blockDim.x) {
            const int pos = idx / NL, lane = idx - pos * NL;
            float v = step_sample<SUM>(s, in, oa + pos, lane);
            if (last && p.is_v) {
                const int c = lane % C;
                v = epilogue_value(p, v, c);
                const long long g = (long long)(oa + pos - p.dst_row_base) * p.dst_pitch +
                                    (long long)line0 * C + lane;
                if (p.dst_type == AVIRB200_F32) ((float*)p.dst)[g] = v;
                else if (p.dst_type == AVIRB200_U8) ((unsigned char*)p.dst)[g] = (unsigned char)v;
                else ((unsigned short*)p.dst)[g] = (unsigned short)v;
            } else {
                ob[pos * p.pitch + lane] = v;
            }
        }
        __syncthreads();
    }

    if (!p.is_v) {
        // transposed, coalesced store of the row-pass result (fp32 intermediate)
        const float* ob = bufs[ns & 1];
        const int oa = rng[ns].a, on = rng[ns].b - rng[ns].a + 1;
        const int rowlen = on * C;
        for (int idx = threadIdx.x; idx < nlines * rowlen; idx += blockDim.x) {
            const int r = idx / rowlen, e = idx - r * rowlen;
            const int pos = e / C, c = e - pos * C;
            const long long g = (long long)(line0 + r) * p.dst_pitch + (long long)(oa + pos - p.dst_row_base) * C + c;
            ((float*)p.dst)[g] = ob[pos * p.pitch + r * C + c];
        }
    }
}

// blockIdx.x: a tile of outputs.  blockIdx.y: a block of lines, and every gridDim.y-th block after it: a pass
// of more than 65535 line blocks (tall images, one line per block) runs in one launch of at most 65535 rows of
// blocks.  Each output's arithmetic does not depend on which block computes it.
template <int SUM>
__global__ void __launch_bounds__(256)
generic_pass_kernel(const __grid_constant__ PassParams p) {
    extern __shared__ float smem[];
    float* const bufs[2] = {smem, smem + (size_t)p.span_a * p.pitch};
    const int j0 = p.out0 + blockIdx.x * p.tile_out;
    const int j1 = imin(j0 + p.tile_out, p.out1) - 1;
    if (j0 > j1) return;
    for (long long line0 = (long long)blockIdx.y * p.lines_per_block; line0 < p.n_lines;
         line0 += (long long)gridDim.y * p.lines_per_block) {
        generic_tile<SUM>(p, bufs, (int)line0, imin(p.lines_per_block, p.n_lines - (int)line0), j0, j1);
        __syncthreads(); // (the next block of lines stages its source over buffer 0)
    }
}

} // namespace avb
