// lancir.cu -- LANCIR (upstream lancir.h) on sm_90a: column pass, row pass + output.
//
// Arithmetic to mirror (upstream AVX build).  4-channel images (resize4, lancir.h:2466-2515):
// per channel two interleaved partial sums over the taps -- even taps into one, odd taps
// into the other -- added at the end.  1- and 2-channel images (resize1/resize2,
// lancir.h:2101-2320): four chains S0..S3 over taps j mod 4, joined as (S0+S2)+(S1+S3); when
// kl%4 == 2 the last two products join as ((S0+S2)+Pa)+((S1+S3)+Pb).  3-channel images
// (resize3, lancir.h:2322-2440): the same four chains, Pa folded into chain 0, Pb folded
// into chain 1 for channel 0 but added last for channels 1 and 2; tree (S0+S1)+(S2+S3).
// Source reads clamp to the image (upstream pads by
// replication: copyScanlineNv lancir.h:1406-1594, padScanlineNh 1611-1734).  Output
// (lancir.h:1772-2056): optional multiply, clamp, round-to-nearest-even; the last
// `(NewWidth*C) & 3` elements of a row round as (int)(v + 0.5f) instead.
//
// 4-channel images with aligned pixels run one thread per PIXEL with vector loads and stores
// (lancir_col4_kernel / lancir_row4_kernel); other channel counts one thread per output element:
// the column pass with threads along x (coalesced reads of every tap's row), the row pass
// reading its taps' pixels from the fp32 intermediate through the caches.
//
// A destination window (lancirb200_resize_window_*) runs the same four kernels over its region: the
// column pass over the footprint's columns and the window's rows, the row pass over the window's columns
// (LParams x0 / y0 / fx0 / fy0 / mid_w; the whole image is the region at the origin, full size).
//
// Element types (upstream lancir.h:373-381): u8, u16, float, double and uint32_t, read and written by the
// kernels themselves (lload / LPix on input, the row passes' stores on output).  Input is (float) v,
// nearest-even (__double2float_rn / __uint2float_rn; float subnormals are kept, the build does not flush
// them).  double output is (double) of the float result; uint32_t output is u16's output stored 32 bits
// wide, except that a NaN in the half-up tail stores x86's (int)NaN = INT_MIN, as upstream's roundclamp.

#include <cuda_runtime.h>

#include <climits>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "avirb200.h"
#include "host_call.h"
#include "host_util.h"
#include "peer_mailbox.h"

using avb::elem_size;
using avb::fail;

namespace {

struct LAxis {
    int src_len, dst_len, kl, nphases;
    const float* taps;
    const int* src_pos;
    const int* phase;
};

struct LParams {
    LAxis v, h;
    int src_w, src_h, dst_w, dst_h, C;
    int in_type, out_type;
    float out_mul, clamp_max;
    int unity;
    const void* src; long long src_pitch;
    float* mid;          // [win_h][mid_w*C]
    void* dst; long long dst_pitch;
    // The destination region the passes compute (the whole image: 0, 0, dst_w, dst_h; a window: its own)
    // and the source columns / rows the buffers start at: src holds source row fy0 onward, its column 0
    // and the intermediate's are source column fx0, the intermediate is mid_w pixels wide (the whole
    // image: 0, 0, src_w).  Taps clamp to the IMAGE first, then fx0 / fy0 index the buffers.
    int x0, y0, win_w, win_h;
    int fx0, fy0, mid_w;
};

__device__ __forceinline__ float lload(const void* p, int type, long long i) {
    if (type == AVIRB200_U8) return (float)((const unsigned char*)p)[i];
    if (type == AVIRB200_U16) return (float)((const unsigned short*)p)[i];
    if (type == AVIRB200_F64) return __double2float_rn(((const double*)p)[i]);
    if (type == AVIRB200_U32) return __uint2float_rn(((const unsigned int*)p)[i]);
    return ((const float*)p)[i];
}

// One output sample: the tap sum in upstream's order for `C` channels, channel `c`.
template <class G>
__device__ __forceinline__ float ltapsum(const int C, const int c, const int kl,
                                         const float* __restrict__ f, G get) {
    if (C == 4) {
        float ev = __fmul_rn(__ldg(f), get(0)), od = __fmul_rn(__ldg(f + 1), get(1));
        for (int t = 2; t < kl; t += 2) {
            ev = __fadd_rn(ev, __fmul_rn(__ldg(f + t), get(t)));
            od = __fadd_rn(od, __fmul_rn(__ldg(f + t + 1), get(t + 1)));
        }
        return __fadd_rn(ev, od);
    }
    const int n4 = kl & ~3;
    float s0 = __fmul_rn(__ldg(f), get(0)), s1 = __fmul_rn(__ldg(f + 1), get(1));
    float s2 = __fmul_rn(__ldg(f + 2), get(2)), s3 = __fmul_rn(__ldg(f + 3), get(3));
    for (int t = 4; t < n4; t += 4) {
        s0 = __fadd_rn(s0, __fmul_rn(__ldg(f + t), get(t)));
        s1 = __fadd_rn(s1, __fmul_rn(__ldg(f + t + 1), get(t + 1)));
        s2 = __fadd_rn(s2, __fmul_rn(__ldg(f + t + 2), get(t + 2)));
        s3 = __fadd_rn(s3, __fmul_rn(__ldg(f + t + 3), get(t + 3)));
    }
    const bool rem = (kl & 3) == 2;
    float pa = 0.0f, pb = 0.0f;
    if (rem) {
        pa = __fmul_rn(__ldg(f + n4), get(n4));
        pb = __fmul_rn(__ldg(f + n4 + 1), get(n4 + 1));
    }
    if (C == 3) {
        if (rem) s0 = __fadd_rn(s0, pa);
        if (rem && c == 0) s1 = __fadd_rn(s1, pb);
        float r = __fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3));
        if (rem && c != 0) r = __fadd_rn(r, pb);
        return r;
    }
    float a = __fadd_rn(s0, s2), b = __fadd_rn(s1, s3);
    if (rem) { a = __fadd_rn(a, pa); b = __fadd_rn(b, pb); }
    return __fadd_rn(a, b);
}

// Column pass: one thread per (x, c) element of an intermediate row; grid.y = output row (of the region).
__global__ void __launch_bounds__(256) lancir_col_kernel(const __grid_constant__ LParams p) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x; // element within a row
    const int y = blockIdx.y;
    const int row_elems = p.mid_w * p.C;
    if (e >= row_elems) return;
    const int kl = p.v.kl;
    const float* f = p.v.taps + (size_t)__ldg(p.v.phase + p.y0 + y) * kl;
    const int s0 = __ldg(p.v.src_pos + p.y0 + y);
    const void* src = p.src;
    const int in_type = p.in_type, src_h = p.src_h, fy0 = p.fy0;
    const long long pitch = p.src_pitch;
    const float r = ltapsum(p.C, e % p.C, kl, f, [&](int t) {
        int sy = s0 + t;
        sy = sy < 0 ? 0 : (sy >= src_h ? src_h - 1 : sy);
        return lload(src, in_type, (long long)(sy - fy0) * pitch + e);
    });
    p.mid[(size_t)y * row_elems + e] = r;
}

// Row pass + output: one thread per output element of the region; grid.y = row.
__global__ void __launch_bounds__(256) lancir_row_kernel(const __grid_constant__ LParams p) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    const int out_elems = p.win_w * p.C;
    if (e >= out_elems) return;
    const int x = e / p.C, c = e - x * p.C;
    const int kl = p.h.kl;
    const float* f = p.h.taps + (size_t)__ldg(p.h.phase + p.x0 + x) * kl;
    const int s0 = __ldg(p.h.src_pos + p.x0 + x);
    const float* row = p.mid + (size_t)y * p.mid_w * p.C;
    const int C = p.C, src_w = p.src_w, fx0 = p.fx0;
    float v = ltapsum(C, c, kl, f, [&](int t) {
        int sx = s0 + t;
        sx = sx < 0 ? 0 : (sx >= src_w ? src_w - 1 : sx);
        return row[(size_t)(sx - fx0) * C + c];
    });
    if (!p.unity) v = __fmul_rn(v, p.out_mul);
    const long long g = (long long)y * p.dst_pitch + e;
    if (p.out_type == AVIRB200_F32) {
        ((float*)p.dst)[g] = v;
        return;
    }
    if (p.out_type == AVIRB200_F64) {
        ((double*)p.dst)[g] = (double)v;
        return;
    }
    int iv;
    // (the tail is the last (dst_w * C) & 3 elements of a whole destination row, whatever the region)
    const bool tail = p.x0 * C + e >= ((p.dst_w * C) & ~3);
    if (tail) {
        // NaN passes the clamp; x86's (int)NaN is INT_MIN: 0 once truncated to u8 / u16, 2147483648 as u32
        const float cv = v > p.clamp_max ? p.clamp_max : (v < 0.0f ? 0.0f : v);
        iv = cv != cv ? INT_MIN : __float2int_rz(__fadd_rn(cv, 0.5f));
    } else {
        const float cv = fmaxf(fminf(v, p.clamp_max), 0.0f);
        iv = __float2int_rn(cv);
    }
    if (p.out_type == AVIRB200_U8) ((unsigned char*)p.dst)[g] = (unsigned char)iv;
    else if (p.out_type == AVIRB200_U16) ((unsigned short*)p.dst)[g] = (unsigned short)iv;
    else ((unsigned int*)p.dst)[g] = (unsigned int)iv;
}

// ---- 4-channel images: one thread per PIXEL, vector loads and stores ----------------------------
// Same sums as ltapsum's C == 4 branch (resize4: even taps into one chain, odd taps into the
// other, per channel), on float4 values.  The column pass walks a run of output rows per block so
// that the kl source rows an output row reads stay in L1 for the next rows (each source byte
// leaves L2 once per block); the row pass reads its taps' pixels as 16-byte loads.
template <typename T> struct LPix;
template <> struct LPix<unsigned char> {
    static __device__ __forceinline__ float4 load(const void* p, long long i) {
        const uchar4 v = *reinterpret_cast<const uchar4*>(static_cast<const unsigned char*>(p) + i);
        return make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
    }
};
template <> struct LPix<unsigned short> {
    static __device__ __forceinline__ float4 load(const void* p, long long i) {
        const ushort4 v = *reinterpret_cast<const ushort4*>(static_cast<const unsigned short*>(p) + i);
        return make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
    }
};
template <> struct LPix<float> {
    static __device__ __forceinline__ float4 load(const void* p, long long i) {
        return *reinterpret_cast<const float4*>(static_cast<const float*>(p) + i);
    }
};
template <> struct LPix<double> { // a 32-byte pixel: two 16-byte loads
    static __device__ __forceinline__ float4 load(const void* p, long long i) {
        const double2* q = reinterpret_cast<const double2*>(static_cast<const double*>(p) + i);
        const double2 a = q[0], b = q[1];
        return make_float4(__double2float_rn(a.x), __double2float_rn(a.y), __double2float_rn(b.x),
                           __double2float_rn(b.y));
    }
};
template <> struct LPix<unsigned int> {
    static __device__ __forceinline__ float4 load(const void* p, long long i) {
        const uint4 v = *reinterpret_cast<const uint4*>(static_cast<const unsigned int*>(p) + i);
        return make_float4(__uint2float_rn(v.x), __uint2float_rn(v.y), __uint2float_rn(v.z), __uint2float_rn(v.w));
    }
};

__device__ __forceinline__ float4 lmul4(float f, float4 v) {
    return make_float4(__fmul_rn(f, v.x), __fmul_rn(f, v.y), __fmul_rn(f, v.z), __fmul_rn(f, v.w));
}
__device__ __forceinline__ float4 ladd4(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

constexpr int kLColRows = 32; // output rows a block of the column pass walks

// KL: compile-time kernel length (all taps' loads of an output are issued before the first
// product: the loop is unrolled) for the common lengths, 0 = run-time length.
// The column pass of output rows [y0, y1) of the region for pixel px; row(sy, e) loads the 4 elements at e of
// source row sy (clamped to the image).
template <typename TIN, int KL, class Row>
__device__ __forceinline__ void lcol4_rows(const LParams& p, const int px, const int y0, const int y1, Row row) {
    const int kl = KL ? KL : p.v.kl, src_h = p.src_h;
    for (int y = y0; y < y1; ++y) {
        const float* f = p.v.taps + (size_t)__ldg(p.v.phase + p.y0 + y) * kl;
        const int s0 = __ldg(p.v.src_pos + p.y0 + y);
        auto S = [&](int t) {
            int sy = s0 + t;
            sy = sy < 0 ? 0 : (sy >= src_h ? src_h - 1 : sy);
            return row(sy, (long long)px * 4);
        };
        float4 ev, od;
        if (KL) {
            float4 x[KL ? KL : 1];
#pragma unroll
            for (int t = 0; t < KL; ++t) x[t] = S(t);
            ev = lmul4(__ldg(f), x[0]); od = lmul4(__ldg(f + 1), x[1]);
#pragma unroll
            for (int t = 2; t < KL; t += 2) {
                ev = ladd4(ev, lmul4(__ldg(f + t), x[t]));
                od = ladd4(od, lmul4(__ldg(f + t + 1), x[t + 1]));
            }
        } else {
            ev = lmul4(__ldg(f), S(0)); od = lmul4(__ldg(f + 1), S(1));
            for (int t = 2; t < kl; t += 2) {
                ev = ladd4(ev, lmul4(__ldg(f + t), S(t)));
                od = ladd4(od, lmul4(__ldg(f + t + 1), S(t + 1)));
            }
        }
        reinterpret_cast<float4*>(p.mid + (size_t)y * p.mid_w * 4)[px] = ladd4(ev, od);
    }
}

// KL: compile-time kernel length (all taps' loads of an output are issued before the first
// product: the loop is unrolled) for the common lengths, 0 = run-time length.
template <typename TIN, int KL>
__global__ void __launch_bounds__(256) lancir_col4_kernel(const __grid_constant__ LParams p) {
    const int px = blockIdx.x * 256 + threadIdx.x;
    if (px >= p.mid_w) return;
    const int y0 = blockIdx.y * kLColRows;
    const int y1 = (y0 + kLColRows < p.win_h) ? y0 + kLColRows : p.win_h;
    const int fy0 = p.fy0;
    const long long pitch = p.src_pitch;
    lcol4_rows<TIN, KL>(p, px, y0, y1, [&](int sy, long long e) {
        return LPix<TIN>::load(p.src, (long long)(sy - fy0) * pitch + e);
    });
}

// ---- row-sharded calls: the column pass over a source in three segments ---------------------------
// A band's column pass reads source rows [up0, row0) from the segment "from above" (the rank above's last
// rows), its own band [row0, row0 + rows) from the caller's buffer (LParams src / src_pitch, fy0 = row0) and
// the rows after it from the segment "from below".  Taps clamp to the image first, as everywhere.  A segment
// with a flag is a peer mailbox: a block whose rows' taps reach it waits until the flag holds the call's
// sequence number (the rows arrive before the flag, lancirb200_resize_sharded); a segment without one is
// already in place (NCCL, device copies).  Picking a segment per tap costs registers, so the segmented kernels
// run only a band's EDGE rows, [0, top) and [bot0, win_h): the rows whose taps reach beyond the band.  The
// rows between read the band alone and run on the plain kernels (lancir_region).
struct LSeg {
    const void* up; long long up_pitch; // pitches in elements
    const void* dn; long long dn_pitch;
    int up0, row0, rows;
    const volatile unsigned* flag_up;
    const volatile unsigned* flag_dn;
    unsigned seq;
    int top, bot0;
};

__device__ __forceinline__ const void* lseg_row(const LParams& p, const LSeg& s, int sy, long long* off) {
    if (sy < s.row0) {
        *off = (long long)(sy - s.up0) * s.up_pitch;
        return s.up;
    }
    if (sy >= s.row0 + s.rows) {
        *off = (long long)(sy - s.row0 - s.rows) * s.dn_pitch;
        return s.dn;
    }
    *off = (long long)(sy - s.row0) * p.src_pitch;
    return p.src;
}

__device__ __forceinline__ void lseg_spin(const volatile unsigned* flag, unsigned seq) {
    long long spins = 0;
    while ((int)(*flag - seq) < 0) {
        if (++spins > (1ll << 31)) __trap(); // a neighbour never delivered: fail instead of hanging
        __nanosleep(100);
    }
    __threadfence_system();
}

// Every thread of the block calls it: the block's output rows [y0, y1) wait for the mailbox segments
// their taps reach (the span of their clamped taps, as lspan computes it on the host).
__device__ __forceinline__ void lseg_wait(const LParams& p, const LSeg& s, int y0, int y1) {
    if (threadIdx.x == 0 && (s.flag_up || s.flag_dn)) {
        const int kl = p.v.kl, src_h = p.src_h;
        int lo = src_h, hi = -1;
        for (int y = y0; y < y1; ++y) {
            const int s0 = __ldg(p.v.src_pos + p.y0 + y);
            const int a = s0 < 0 ? 0 : (s0 >= src_h ? src_h - 1 : s0);
            const int b = s0 + kl - 1 < 0 ? 0 : (s0 + kl - 1 >= src_h ? src_h - 1 : s0 + kl - 1);
            lo = a < lo ? a : lo;
            hi = b > hi ? b : hi;
        }
        if (s.flag_up && lo < s.row0) lseg_spin(s.flag_up, s.seq);
        if (s.flag_dn && hi >= s.row0 + s.rows) lseg_spin(s.flag_dn, s.seq);
    }
    __syncthreads();
}

// The rows [*y0, *y1) of row group blockIdx.y: groups of G rows over [0, top), then over [bot0, win_h).
template <int G>
__device__ __forceinline__ void lseg_rows(const LParams& p, const LSeg& s, int* y0, int* y1) {
    const int gt = (s.top + G - 1) / G, g = (int)blockIdx.y;
    const int a = g < gt ? g * G : s.bot0 + (g - gt) * G;
    const int e = g < gt ? s.top : p.win_h;
    *y0 = a;
    *y1 = a + G < e ? a + G : e;
}

// lancir_col_kernel over a segmented source
__global__ void __launch_bounds__(256) lancir_col_seg_kernel(const __grid_constant__ LParams p,
                                                             const __grid_constant__ LSeg s) {
    int y, y1;
    lseg_rows<1>(p, s, &y, &y1);
    lseg_wait(p, s, y, y1);
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int row_elems = p.mid_w * p.C;
    if (e >= row_elems) return;
    const int kl = p.v.kl;
    const float* f = p.v.taps + (size_t)__ldg(p.v.phase + p.y0 + y) * kl;
    const int s0 = __ldg(p.v.src_pos + p.y0 + y);
    const int in_type = p.in_type, src_h = p.src_h;
    const float r = ltapsum(p.C, e % p.C, kl, f, [&](int t) {
        int sy = s0 + t;
        sy = sy < 0 ? 0 : (sy >= src_h ? src_h - 1 : sy);
        long long off;
        const void* b = lseg_row(p, s, sy, &off);
        return lload(b, in_type, off + e);
    });
    p.mid[(size_t)y * row_elems + e] = r;
}

// lancir_col4_kernel over a segmented source (every segment's pixels aligned to their size)
template <typename TIN, int KL>
__global__ void __launch_bounds__(256) lancir_col4_seg_kernel(const __grid_constant__ LParams p,
                                                              const __grid_constant__ LSeg s) {
    int y0, y1;
    lseg_rows<kLColRows>(p, s, &y0, &y1);
    lseg_wait(p, s, y0, y1);
    const int px = blockIdx.x * 256 + threadIdx.x;
    if (px >= p.mid_w) return;
    lcol4_rows<TIN, KL>(p, px, y0, y1, [&](int sy, long long e) {
        long long off;
        const void* b = lseg_row(p, s, sy, &off);
        return LPix<TIN>::load(b, off + e);
    });
}

// OUT: 0 float, 1 u8, 2 u16, 3 double, 4 uint32_t
template <int OUT, int KL>
__global__ void __launch_bounds__(256) lancir_row4_kernel(const __grid_constant__ LParams p) {
    const int x = blockIdx.x * 256 + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= p.win_w) return;
    const int kl = KL ? KL : p.h.kl, src_w = p.src_w, fx0 = p.fx0;
    const float* f = p.h.taps + (size_t)__ldg(p.h.phase + p.x0 + x) * kl;
    const int s0 = __ldg(p.h.src_pos + p.x0 + x);
    const float4* row = reinterpret_cast<const float4*>(p.mid + (size_t)y * p.mid_w * 4);
    auto M = [&](int t) {
        int sx = s0 + t;
        sx = sx < 0 ? 0 : (sx >= src_w ? src_w - 1 : sx);
        return row[sx - fx0];
    };
    float4 ev, od;
    if (KL) {
        float4 xw[KL ? KL : 1];
#pragma unroll
        for (int t = 0; t < KL; ++t) xw[t] = M(t);
        ev = lmul4(__ldg(f), xw[0]); od = lmul4(__ldg(f + 1), xw[1]);
#pragma unroll
        for (int t = 2; t < KL; t += 2) {
            ev = ladd4(ev, lmul4(__ldg(f + t), xw[t]));
            od = ladd4(od, lmul4(__ldg(f + t + 1), xw[t + 1]));
        }
    } else {
        ev = lmul4(__ldg(f), M(0)); od = lmul4(__ldg(f + 1), M(1));
        for (int t = 2; t < kl; t += 2) {
            ev = ladd4(ev, lmul4(__ldg(f + t), M(t)));
            od = ladd4(od, lmul4(__ldg(f + t + 1), M(t + 1)));
        }
    }
    float4 v = ladd4(ev, od);
    if (!p.unity) v = lmul4(p.out_mul, v);
    const long long g = (long long)y * p.dst_pitch + (long long)x * 4;
    if (OUT == 0) {
        *reinterpret_cast<float4*>(static_cast<float*>(p.dst) + g) = v;
        return;
    }
    if (OUT == 3) { // two 16-byte stores
        double2* q = reinterpret_cast<double2*>(static_cast<double*>(p.dst) + g);
        q[0] = make_double2((double)v.x, (double)v.y);
        q[1] = make_double2((double)v.z, (double)v.w);
        return;
    }
    // (a row of 4-channel pixels has no (NewWidth*C) & 3 tail: every element rounds nearest-even)
    const float cm = p.clamp_max;
    const int a = __float2int_rn(fmaxf(fminf(v.x, cm), 0.0f)), b = __float2int_rn(fmaxf(fminf(v.y, cm), 0.0f));
    const int c = __float2int_rn(fmaxf(fminf(v.z, cm), 0.0f)), d = __float2int_rn(fmaxf(fminf(v.w, cm), 0.0f));
    if (OUT == 1)
        *reinterpret_cast<uchar4*>(static_cast<unsigned char*>(p.dst) + g) =
            make_uchar4((unsigned char)a, (unsigned char)b, (unsigned char)c, (unsigned char)d);
    else if (OUT == 2)
        *reinterpret_cast<ushort4*>(static_cast<unsigned short*>(p.dst) + g) =
            make_ushort4((unsigned short)a, (unsigned short)b, (unsigned short)c, (unsigned short)d);
    else
        *reinterpret_cast<uint4*>(static_cast<unsigned int*>(p.dst) + g) =
            make_uint4((unsigned int)a, (unsigned int)b, (unsigned int)c, (unsigned int)d);
}

// The source span [lo, lo + n) the outputs [i0, i0 + cnt) of an axis read: every tap position clamped to
// the image, the min / max over the outputs' table entries (the tables need not be monotone).  Zero taps
// count: the kernels multiply every tap, and 0 * NaN is NaN.
void lspan(const int32_t* pos, int kl, int src_len, int i0, int cnt, int32_t* lo, int32_t* n) {
    long long a = src_len, b = -1;
    for (int i = i0; i < i0 + cnt; ++i) {
        long long first = pos[i], last = (long long)pos[i] + kl - 1;
        first = first < 0 ? 0 : (first >= src_len ? src_len - 1 : first);
        last = last < 0 ? 0 : (last >= src_len ? src_len - 1 : last);
        a = first < a ? first : a;
        b = last > b ? last : b;
    }
    *lo = (int32_t)a;
    *n = (int32_t)(b - a + 1);
}

// The footprint of the destination window [x0, x0 + w) x [y0, y0 + h).
int lwindow(const int32_t* hpos, int hkl, const int32_t* vpos, int vkl, int src_w, int src_h, int dst_w, int dst_h,
            int x0, int y0, int w, int h, lancirb200_window_info* info) {
    if (x0 < 0 || y0 < 0 || w < 1 || h < 1 || (long long)x0 + w > dst_w || (long long)y0 + h > dst_h)
        return fail(AVIRB200_ERR_BAD_ARG, "window empty or outside the destination");
    lspan(hpos, hkl, src_w, x0, w, &info->src_x0, &info->src_w);
    lspan(vpos, vkl, src_h, y0, h, &info->src_y0, &info->src_h);
    return 0;
}

// Row-sharded calls: the bands of rank `rank` of `nranks`, by AVIR's partition rule (source rows src_h * r / n,
// destination rows dst_h * r / n).  need_* are SOURCE rows: the band's vertical footprint (lspan) joined with
// its own source band; the halos are the rows of it beyond the band, which the neighbours hold.
int lshard(const int32_t* vpos, int vkl, int src_h, int dst_h, int rank, int nranks, avirb200_shard_info* info) {
    const int r = avb::shard_split(src_h, dst_h, rank, nranks, info);
    if (r != 0) return r;
    if (info->dst_rows > 65535) return fail(AVIRB200_ERR_UNSUPPORTED, "band too tall (more than 65535 destination rows)");
    int32_t lo = 0, n = 0;
    lspan(vpos, vkl, src_h, info->dst_row0, info->dst_rows, &lo, &n);
    return avb::shard_halos(lo, lo + n, src_h, rank, nranks, info);
}

// Bytes of one source row in a halo segment: 16-byte aligned, so that the vector kernel's loads stay aligned.
size_t lhalo_row_bytes(const lancirb200_plan_desc& d) {
    return avb::align_up((size_t)d.src_w * d.channels * elem_size(d.in_type), 16);
}

// A band's workspace: [intermediate: dst_rows x src_w x C floats] [rows from above: halo_up rows]
// [rows from below: halo_down rows] [header: the flags lancirb200_resize_sharded_local raises], each part
// 256-byte aligned.  The halo segments receive the neighbours' rows on the NCCL schedule.
struct LShardWs {
    static constexpr size_t kHeader = 256;
    size_t up = 0, down = 0, header = 0, total = 0;
    LShardWs(const lancirb200_plan_desc& d, const avirb200_shard_info& si) {
        const size_t row = lhalo_row_bytes(d);
        up = avb::align_up((size_t)si.dst_rows * d.src_w * d.channels * sizeof(float), 256);
        down = up + avb::align_up((size_t)si.halo_up * row, 256);
        header = down + avb::align_up((size_t)si.halo_down * row, 256);
        total = header + kHeader;
    }
};

// A rank's mailbox: [256 B header: flag "from above" at +0, flag "from below" at +4]
//   slot 0: [rows from rank-1: halo_up rows] [rows from rank+1: halo_down rows, at +align256(up_bytes)]
//   slot 1: the same
// Rows lhalo_row_bytes apart, in the caller's element type.
struct LBoxLayout {
    static constexpr size_t kHeader = 256;
    size_t up_bytes = 0, down_bytes = 0;
    LBoxLayout() = default;
    LBoxLayout(const lancirb200_plan_desc& d, const avirb200_shard_info& si)
        : up_bytes((size_t)si.halo_up * lhalo_row_bytes(d)), down_bytes((size_t)si.halo_down * lhalo_row_bytes(d)) {}
    size_t slot_bytes() const { return avb::align_up(up_bytes, 256) + avb::align_up(down_bytes, 256); }
    size_t bytes(int slots) const { return kHeader + (size_t)slots * slot_bytes(); }
    char* from_up(char* box, int slot) const { return box + kHeader + (size_t)slot * slot_bytes(); }
    char* from_down(char* box, int slot) const { return from_up(box, slot) + avb::align_up(up_bytes, 256); }
};

} // namespace

struct lancirb200_plan {
    lancirb200_plan_desc desc;
    void* arena = nullptr;
    LAxis dv, dh;
    std::vector<int32_t> pos_v, pos_h; // host copies of the axes' src_pos (window footprints)
    int device = 0;
    std::mutex mx;
    avb::Staging staging;        // host calls: this plan's own staging buffers (host_call.h)
    cudaStream_t stream = nullptr;
    // row-sharded calls
    int opt_overlap = 3;           // AVIRB200_OPT_OVERLAP_HALO: 3 mailboxes, 0 NCCL
    avb::PeerExchange x;           // the halo exchange (opened by the first sharded call of more than one rank)
};

extern "C" {

int lancirb200_plan_create(const lancirb200_plan_desc* d, lancirb200_plan** out) {
    if (d == nullptr || out == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    if (d->channels < 1 || d->channels > 4) return fail(AVIRB200_ERR_BAD_ARG, "channels must be 1..4");
    for (const int t : {d->in_type, d->out_type})
        if (t < AVIRB200_U8 || t > AVIRB200_U32)
            return fail(AVIRB200_ERR_BAD_ARG, "element type must be U8, U16, F32, F64 or U32 (0..4)");
    if (d->v.kernel_len < 4 || d->h.kernel_len < 4 || ((d->v.kernel_len | d->h.kernel_len) & 1))
        return fail(AVIRB200_ERR_BAD_ARG, "kernel length must be even and >= 4");
    if (d->src_w < 1 || d->src_h < 1 || d->dst_w < 1 || d->dst_h < 1)
        return fail(AVIRB200_ERR_BAD_ARG, "bad geometry");
    for (int a = 0; a < 2; ++a) {
        const lancirb200_axis_desc& ax = a ? d->h : d->v;
        if (ax.kernel_len < 2 || ax.nphases < 1 || !ax.taps || !ax.src_pos || !ax.phase)
            return fail(AVIRB200_ERR_BAD_ARG, "bad axis tables");
        for (int i = 0; i < ax.dst_len; ++i)
            if (ax.phase[i] < 0 || ax.phase[i] >= ax.nphases)
                return fail(AVIRB200_ERR_BAD_ARG, "phase index out of range");
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(AVIRB200_ERR_NO_DEVICE, "no CUDA device");
    std::unique_ptr<lancirb200_plan> pl(new (std::nothrow) lancirb200_plan());
    if (!pl) return fail(AVIRB200_ERR_ALLOC, "host allocation failed");
    pl->desc = *d;
    CUDA_TRY(cudaGetDevice(&pl->device));
    size_t bytes = 0;
    for (int a = 0; a < 2; ++a) {
        const lancirb200_axis_desc& ax = a ? d->h : d->v;
        bytes += avb::align_up((size_t)ax.nphases * ax.kernel_len * 4, 256) + 2 * avb::align_up((size_t)ax.dst_len * 4, 256);
    }
    CUDA_TRY(cudaMalloc(&pl->arena, bytes));
    std::vector<char> img(bytes, 0);
    size_t off = 0;
    for (int a = 0; a < 2; ++a) {
        const lancirb200_axis_desc& ax = a ? d->h : d->v;
        LAxis& da = a ? pl->dh : pl->dv;
        da.src_len = ax.src_len; da.dst_len = ax.dst_len; da.kl = ax.kernel_len;
        da.nphases = ax.nphases;
        char* base = static_cast<char*>(pl->arena);
        size_t n = (size_t)ax.nphases * ax.kernel_len * 4;
        std::memcpy(img.data() + off, ax.taps, n);
        da.taps = reinterpret_cast<const float*>(base + off); off += avb::align_up(n, 256);
        n = (size_t)ax.dst_len * 4;
        std::memcpy(img.data() + off, ax.src_pos, n);
        da.src_pos = reinterpret_cast<const int*>(base + off); off += avb::align_up(n, 256);
        std::memcpy(img.data() + off, ax.phase, n);
        da.phase = reinterpret_cast<const int*>(base + off); off += avb::align_up(n, 256);
    }
    CUDA_TRY(cudaMemcpy(pl->arena, img.data(), bytes, cudaMemcpyHostToDevice));
    pl->pos_v.assign(d->v.src_pos, d->v.src_pos + d->v.dst_len);
    pl->pos_h.assign(d->h.src_pos, d->h.src_pos + d->h.dst_len);
    // (the descriptor's tables are the caller's: the plan keeps no pointer to them)
    pl->desc.v.taps = nullptr; pl->desc.h.taps = nullptr;
    pl->desc.v.src_pos = nullptr; pl->desc.h.src_pos = nullptr;
    pl->desc.v.phase = nullptr; pl->desc.h.phase = nullptr;
    *out = pl.release();
    return 0;
}

void lancirb200_plan_destroy(lancirb200_plan* pl) {
    if (!pl) return;
    cudaFree(pl->arena);
    if (pl->stream) cudaStreamDestroy(pl->stream);
    pl->x.close();
    delete pl;
}

int lancirb200_plan_workspace_bytes(const lancirb200_plan* pl, size_t* bytes) {
    if (!pl || !bytes) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    *bytes = (size_t)pl->desc.dst_h * pl->desc.src_w * pl->desc.channels * sizeof(float);
    return 0;
}

} // extern "C"

namespace {

// Both passes over the destination region [x0, x0 + w) x [y0, y0 + h): d_src holds the source from row fy0
// on, its column 0 is source column fx0, and the intermediate in d_ws is h rows of fw pixels.  seg: the
// column pass reads a segmented source (row-sharded calls; fy0 is then the band's first row).
int lancir_region(const lancirb200_plan* pl, int x0, int y0, int w, int h, int fx0, int fw, int fy0,
                  const void* d_src, size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_ws, void* stream,
                  const LSeg* seg = nullptr) {
    const lancirb200_plan_desc& d = pl->desc;
    LParams p;
    p.v = pl->dv; p.h = pl->dh;
    p.src_w = d.src_w; p.src_h = d.src_h; p.dst_w = d.dst_w; p.dst_h = d.dst_h; p.C = d.channels;
    p.in_type = d.in_type; p.out_type = d.out_type;
    p.out_mul = d.out_mul; p.clamp_max = d.clamp_max; p.unity = d.is_unity_mul;
    p.src = d_src; p.src_pitch = (long long)src_pitch;
    p.mid = static_cast<float*>(d_ws);
    p.dst = d_dst; p.dst_pitch = (long long)dst_pitch;
    p.x0 = x0; p.y0 = y0; p.win_w = w; p.win_h = h;
    p.fx0 = fx0; p.fy0 = fy0; p.mid_w = fw;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (h > 65535) return fail(AVIRB200_ERR_UNSUPPORTED, "image too tall");
    (void)cudaGetLastError(); // (a stale non-sticky error of another library is not this launch's)
    // 4-channel images whose pixels are aligned to their own size: the vector kernels (a segmented source's
    // halo segments are aligned by construction)
    const bool vec_in = d.channels == 4 && (src_pitch % 4) == 0 && ((uintptr_t)d_src % (4 * elem_size(d.in_type))) == 0 &&
                        ((uintptr_t)d_ws % 16) == 0;
    const bool vec_out = d.channels == 4 && (dst_pitch % 4) == 0 && ((uintptr_t)d_dst % (4 * elem_size(d.out_type))) == 0 &&
                         ((uintptr_t)d_ws % 16) == 0;
    // a band (seg): the plain kernel over its interior rows [top, bot0), the segmented one over its edge rows
    LParams pi = p;
    LSeg s;
    std::memset(&s, 0, sizeof s);
    int ni = h, ne = 0; // interior rows, edge row groups
    if (seg) {
        s = *seg;
        pi.y0 += s.top;
        pi.win_h = ni = s.bot0 - s.top;
        pi.mid += (size_t)s.top * fw * d.channels;
    }
    if (vec_in) {
        auto groups = [](int rows) { return (rows + kLColRows - 1) / kLColRows; };
        if (seg) ne = groups(s.top) + groups(h - s.bot0);
        const dim3 g1((fw + 255) / 256, groups(ni)), ge((fw + 255) / 256, ne);
#define LCOL1(T, KL)                                                                                    \
    do {                                                                                                \
        if (ni > 0) lancir_col4_kernel<T, KL><<<g1, 256, 0, st>>>(pi);                                  \
        if (ne > 0) lancir_col4_seg_kernel<T, KL><<<ge, 256, 0, st>>>(p, s);                            \
    } while (0)
#define LCOL(KL)                                                                                        \
    do {                                                                                                \
        if (d.in_type == AVIRB200_U8) LCOL1(unsigned char, KL);                                         \
        else if (d.in_type == AVIRB200_U16) LCOL1(unsigned short, KL);                                  \
        else if (d.in_type == AVIRB200_F64) LCOL1(double, KL);                                          \
        else if (d.in_type == AVIRB200_U32) LCOL1(unsigned int, KL);                                    \
        else LCOL1(float, KL);                                                                          \
    } while (0)
        switch (pl->dv.kl) { // la = 3: 6 taps when upsizing, 12 at k = 2, 18 at k = 3, 24 at k = 4
        case 6: LCOL(6); break;
        case 12: LCOL(12); break;
        case 18: LCOL(18); break;
        case 24: LCOL(24); break;
        default: LCOL(0); break;
        }
#undef LCOL
#undef LCOL1
    } else {
        if (seg) ne = s.top + (h - s.bot0);
        const dim3 g1((fw * d.channels + 255) / 256, ni), ge((fw * d.channels + 255) / 256, ne);
        if (ni > 0) lancir_col_kernel<<<g1, 256, 0, st>>>(pi);
        if (ne > 0) lancir_col_seg_kernel<<<ge, 256, 0, st>>>(p, s);
    }
    if (vec_out) {
        dim3 g2((w + 255) / 256, h);
#define LROW(KL)                                                                                        \
    do {                                                                                                \
        if (d.out_type == AVIRB200_U8) lancir_row4_kernel<1, KL><<<g2, 256, 0, st>>>(p);                \
        else if (d.out_type == AVIRB200_U16) lancir_row4_kernel<2, KL><<<g2, 256, 0, st>>>(p);          \
        else if (d.out_type == AVIRB200_F64) lancir_row4_kernel<3, KL><<<g2, 256, 0, st>>>(p);          \
        else if (d.out_type == AVIRB200_U32) lancir_row4_kernel<4, KL><<<g2, 256, 0, st>>>(p);          \
        else lancir_row4_kernel<0, KL><<<g2, 256, 0, st>>>(p);                                          \
    } while (0)
        switch (pl->dh.kl) {
        case 6: LROW(6); break;
        case 12: LROW(12); break;
        case 18: LROW(18); break;
        case 24: LROW(24); break;
        default: LROW(0); break;
        }
#undef LROW
    } else {
        dim3 g2((w * d.channels + 255) / 256, h);
        lancir_row_kernel<<<g2, 256, 0, st>>>(p);
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int lancir_window(const lancirb200_plan* pl, int x0, int y0, int w, int h, lancirb200_window_info* info) {
    const lancirb200_plan_desc& d = pl->desc;
    return lwindow(pl->pos_h.data(), pl->dh.kl, pl->pos_v.data(), pl->dv.kl, d.src_w, d.src_h, d.dst_w, d.dst_h, x0, y0,
                   w, h, info);
}

} // namespace

extern "C" {

int lancirb200_resize_device(const lancirb200_plan* pl, const void* d_src, size_t src_pitch,
                             void* d_dst, size_t dst_pitch, void* d_ws, void* stream) {
    if (!pl || !d_src || !d_dst || !d_ws) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const lancirb200_plan_desc& d = pl->desc;
    return lancir_region(pl, 0, 0, d.dst_w, d.dst_h, 0, d.src_w, 0, d_src, src_pitch, d_dst, dst_pitch, d_ws, stream);
}

int lancirb200_resize_host(lancirb200_plan* pl, const void* h_src, size_t src_pitch, void* h_dst,
                           size_t dst_pitch) {
    if (!pl || !h_src || !h_dst) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const lancirb200_plan_desc& d = pl->desc;
    const size_t sw = (size_t)d.src_w * d.channels, dw = (size_t)d.dst_w * d.channels;
    const avb::HostRect src = avb::host_rect(h_src, src_pitch, sw, elem_size(d.in_type), 0, sw, 0, d.src_h);
    const avb::HostRect dst = avb::host_rect(h_dst, dst_pitch, dw, elem_size(d.out_type), 0, dw, 0, d.dst_h);
    size_t ws = 0;
    lancirb200_plan_workspace_bytes(pl, &ws);
    return avb::staged_call(pl->mx, pl->staging, pl->device, &pl->stream, src, dst, ws,
                            [&](const void* s, void* o, void* w, cudaStream_t st) {
                                return lancirb200_resize_device(pl, s, sw, o, dw, w, st);
                            });
}

int lancirb200_window_query(const lancirb200_plan* pl, int x0, int y0, int w, int h, lancirb200_window_info* info) {
    if (!pl || !info) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    return lancir_window(pl, x0, y0, w, h, info);
}

int lancirb200_window_query_desc(const lancirb200_plan_desc* d, int x0, int y0, int w, int h,
                                 lancirb200_window_info* info) {
    if (!d || !info) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (d->src_w < 1 || d->src_h < 1 || d->dst_w < 1 || d->dst_h < 1 || !d->h.src_pos || !d->v.src_pos ||
        d->h.dst_len < d->dst_w || d->v.dst_len < d->dst_h || d->h.kernel_len < 1 || d->v.kernel_len < 1)
        return fail(AVIRB200_ERR_BAD_ARG, "bad geometry or axis tables");
    return lwindow(d->h.src_pos, d->h.kernel_len, d->v.src_pos, d->v.kernel_len, d->src_w, d->src_h, d->dst_w,
                   d->dst_h, x0, y0, w, h, info);
}

int lancirb200_window_workspace_bytes(const lancirb200_plan* pl, int x0, int y0, int w, int h, size_t* bytes) {
    if (!pl || !bytes) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    lancirb200_window_info wi;
    const int r = lancir_window(pl, x0, y0, w, h, &wi);
    if (r != 0) return r;
    *bytes = (size_t)h * wi.src_w * pl->desc.channels * sizeof(float);
    return 0;
}

int lancirb200_resize_window_device(const lancirb200_plan* pl, int x0, int y0, int w, int h, const void* d_src,
                                    size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_ws, void* stream) {
    if (!pl || !d_src || !d_dst || !d_ws) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    lancirb200_window_info wi;
    const int r = lancir_window(pl, x0, y0, w, h, &wi);
    if (r != 0) return r;
    const int C = pl->desc.channels;
    if (src_pitch < (size_t)wi.src_w * C || dst_pitch < (size_t)w * C)
        return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    return lancir_region(pl, x0, y0, w, h, wi.src_x0, wi.src_w, wi.src_y0, d_src, src_pitch, d_dst, dst_pitch, d_ws,
                         stream);
}

int lancirb200_resize_window_host(lancirb200_plan* pl, int x0, int y0, int w, int h, const void* h_src,
                                  size_t src_pitch, void* h_dst, size_t dst_pitch) {
    if (!pl || !h_src || !h_dst) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const lancirb200_plan_desc& d = pl->desc;
    lancirb200_window_info wi;
    const int r = lancir_window(pl, x0, y0, w, h, &wi);
    if (r != 0) return r;
    // the footprint only
    const size_t C = d.channels;
    const avb::HostRect src = avb::host_rect(h_src, src_pitch, d.src_w * C, elem_size(d.in_type), wi.src_x0 * C,
                                             wi.src_w * C, wi.src_y0, wi.src_h);
    const avb::HostRect dst = avb::host_rect(h_dst, dst_pitch, w * C, elem_size(d.out_type), 0, w * C, 0, h);
    const size_t ws = (size_t)h * wi.src_w * C * sizeof(float);
    return avb::staged_call(pl->mx, pl->staging, pl->device, &pl->stream, src, dst, ws,
                            [&](const void* s, void* o, void* wsp, cudaStream_t st) {
                                return lancir_region(pl, x0, y0, w, h, wi.src_x0, wi.src_w, wi.src_y0, s, wi.src_w * C,
                                                     o, w * C, wsp, st);
                            });
}

} // extern "C"

// ---- row-sharded calls ---------------------------------------------------------------------------

namespace {

int lshard_plan(const lancirb200_plan* pl, int rank, int nranks, avirb200_shard_info* si) {
    const lancirb200_plan_desc& d = pl->desc;
    return lshard(pl->pos_v.data(), pl->dv.kl, d.src_h, d.dst_h, rank, nranks, si);
}

// `n` source rows of a band from its row `r0` into a halo segment (rows lhalo_row_bytes apart) on `st`, then,
// when `flag` is given, the 4-byte `word` into it.
int lpush_rows(const lancirb200_plan* pl, void* seg, const void* band, size_t src_pitch, int r0, int n, void* flag,
               const unsigned* word, cudaStream_t st) {
    const lancirb200_plan_desc& d = pl->desc;
    const size_t el = elem_size(d.in_type);
    return avb::push_rows(seg, lhalo_row_bytes(d), static_cast<const char*>(band) + (size_t)r0 * src_pitch * el,
                          src_pitch * el, (size_t)d.src_w * d.channels * el, n, flag, word, st);
}

// A band's passes: the column pass over its segmented source (s: the segments, flags and sequence number),
// the row pass over its destination rows, full width.
int lband(const lancirb200_plan* pl, const avirb200_shard_info& si, const void* band_src, size_t src_pitch,
          void* band_dst, size_t dst_pitch, void* d_ws, LSeg s, cudaStream_t st) {
    const lancirb200_plan_desc& d = pl->desc;
    s.up0 = si.need_row0; s.row0 = si.src_row0; s.rows = si.src_rows;
    // the edge rows: the leading and trailing destination rows whose clamped taps leave the band; the rows
    // between must all stay inside it, or every row is an edge row (the tables need not be monotone)
    const int kl = pl->dv.kl, n = si.dst_rows, r0 = si.src_row0, r1 = si.src_row0 + si.src_rows;
    auto inside = [&](int y) {
        const long long a = pl->pos_v[si.dst_row0 + y], b = a + kl - 1;
        const long long ca = a < 0 ? 0 : (a >= d.src_h ? d.src_h - 1 : a), cb = b < 0 ? 0 : (b >= d.src_h ? d.src_h - 1 : b);
        return ca >= r0 && cb < r1;
    };
    int top = 0, bot0 = n;
    while (top < n && !inside(top)) ++top;
    while (bot0 > top && !inside(bot0 - 1)) --bot0;
    for (int y = top; y < bot0; ++y)
        if (!inside(y)) {
            top = bot0 = n;
            break;
        }
    if (top >= bot0) top = bot0 = n;
    s.top = top; s.bot0 = bot0;
    return lancir_region(pl, 0, si.dst_row0, d.dst_w, si.dst_rows, 0, d.src_w, si.src_row0, band_src, src_pitch,
                         band_dst, dst_pitch, d_ws, st, &s);
}

int lcheck(const lancirb200_plan* pl, size_t src_pitch, size_t dst_pitch) {
    const lancirb200_plan_desc& d = pl->desc;
    if (src_pitch < (size_t)d.src_w * d.channels || dst_pitch < (size_t)d.dst_w * d.channels)
        return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    return avb::check_device(pl->device);
}

// lancirb200_resize_sharded for nranks > 1; the caller holds pl->mx.
int lsharded(lancirb200_plan* pl, void* comm, int rank, int nranks, const void* d_src, size_t src_pitch, void* d_dst,
             size_t dst_pitch, void* d_ws, cudaStream_t st) {
    const lancirb200_plan_desc& d = pl->desc;
    avirb200_shard_info si, up, dn; // this rank's bands and its neighbours'
    std::memset(&up, 0, sizeof up);
    std::memset(&dn, 0, sizeof dn);
    int r = lshard_plan(pl, rank, nranks, &si);
    if (r == 0 && rank > 0) r = lshard_plan(pl, rank - 1, nranks, &up);
    if (r == 0 && rank + 1 < nranks) r = lshard_plan(pl, rank + 1, nranks, &dn);
    if (r != 0) return r;
    avb::Nccl* nc = nullptr;
    if ((r = avb::comm_nccl(comm, &nc)) != 0) return r;
    avb::PeerExchange& x = pl->x;
    const LBoxLayout mine(d, si), above(d, up), below(d, dn);
    if (pl->opt_overlap && (r = x.open(comm, rank, nranks, mine.bytes(2), LBoxLayout::kHeader, st)) != 0) return r;
    // A pair of neighbours exchanges through the mailboxes when rows travel both ways (DESIGN.md section 7: then
    // neither can run two calls ahead of the other); otherwise, and on the NCCL schedule, through NCCL.
    const bool boxes = pl->opt_overlap && x.usable;
    const bool box_up = boxes && rank > 0 && si.halo_up > 0 && up.halo_down > 0;
    const bool box_dn = boxes && rank + 1 < nranks && si.halo_down > 0 && dn.halo_up > 0;
    const bool nccl_up = !box_up && rank > 0 && (si.halo_up > 0 || up.halo_down > 0);
    const bool nccl_dn = !box_dn && rank + 1 < nranks && (si.halo_down > 0 || dn.halo_up > 0);
    const LShardWs wl(d, si);
    char* wsb = static_cast<char*>(d_ws);
    const size_t el = elem_size(d.in_type), row16 = lhalo_row_bytes(d), rowb = (size_t)d.src_w * d.channels * el;
    const char* srcb = static_cast<const char*>(d_src);
    LSeg s;
    std::memset(&s, 0, sizeof s);
    s.up = wsb + wl.up; s.dn = wsb + wl.down;
    s.up_pitch = s.dn_pitch = (long long)(row16 / el);
    bool pushed = false;
    if (box_up || box_dn) {
        // the rows each neighbour needs go into its mailbox (this call's slot) on the exchange stream, each
        // direction followed by the call's sequence number in the neighbour's flag; no kernel of this call
        // comes before them
        const avb::PeerExchange::Call call = x.next_call();
        s.seq = call.seq;
        if ((r = x.fork(st)) != 0) return r;
        if (box_up) {
            if ((r = lpush_rows(pl, above.from_down(x.box_up, call.slot), d_src, src_pitch, 0, up.halo_down, x.box_up + 4,
                                call.word, x.stream)) != 0)
                return r;
            s.up = mine.from_up(x.box, call.slot);
            s.flag_up = reinterpret_cast<const volatile unsigned*>(x.box);
        }
        if (box_dn) {
            if ((r = lpush_rows(pl, below.from_up(x.box_down, call.slot), d_src, src_pitch, si.src_rows - dn.halo_up,
                                dn.halo_up, x.box_down, call.word, x.stream)) != 0)
                return r;
            s.dn = mine.from_down(x.box, call.slot);
            s.flag_dn = reinterpret_cast<const volatile unsigned*>(x.box + 4);
        }
        pushed = true;
    }
    // the other pairs: one message per row into the workspace's halo segments, grouped before the column pass
    if (nccl_up || nccl_dn) {
        NCCL_TRY(nc->GroupStart());
        if (nccl_up) {
            for (int i = 0; i < up.halo_down; ++i)
                NCCL_TRY(nc->Send(srcb + (size_t)i * src_pitch * el, rowb, 0, rank - 1, comm, st));
            for (int i = 0; i < si.halo_up; ++i) NCCL_TRY(nc->Recv(wsb + wl.up + (size_t)i * row16, rowb, 0, rank - 1, comm, st));
        }
        if (nccl_dn) {
            for (int i = si.src_rows - dn.halo_up; i < si.src_rows; ++i)
                NCCL_TRY(nc->Send(srcb + (size_t)i * src_pitch * el, rowb, 0, rank + 1, comm, st));
            for (int i = 0; i < si.halo_down; ++i)
                NCCL_TRY(nc->Recv(wsb + wl.down + (size_t)i * row16, rowb, 0, rank + 1, comm, st));
        }
        NCCL_TRY(nc->GroupEnd());
    }
    r = lband(pl, si, d_src, src_pitch, d_dst, dst_pitch, d_ws, s, st);
    // the pushes read the caller's source band: the caller's stream does not end before them
    if (const int e = pushed ? x.join(st) : 0) return e;
    return r;
}

} // namespace

extern "C" {

int lancirb200_plan_set_option(lancirb200_plan* pl, int option, int value) {
    if (!pl) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (option != AVIRB200_OPT_OVERLAP_HALO) return fail(AVIRB200_ERR_BAD_ARG, "unknown option (CLancIR plans: AVIRB200_OPT_OVERLAP_HALO)");
    if (value != 0 && value != 3) return fail(AVIRB200_ERR_BAD_ARG, "AVIRB200_OPT_OVERLAP_HALO: 3 (mailboxes) or 0 (NCCL)");
    std::lock_guard<std::mutex> lk(pl->mx);
    pl->opt_overlap = value;
    return 0;
}

int lancirb200_shard_query(const lancirb200_plan* pl, int rank, int nranks, avirb200_shard_info* info) {
    if (!pl || !info) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    return lshard_plan(pl, rank, nranks, info);
}

int lancirb200_shard_query_desc(const lancirb200_plan_desc* d, int rank, int nranks, avirb200_shard_info* info) {
    if (!d || !info) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (d->src_w < 1 || d->src_h < 1 || d->dst_w < 1 || d->dst_h < 1 || !d->v.src_pos || d->v.dst_len < d->dst_h ||
        d->v.kernel_len < 1)
        return fail(AVIRB200_ERR_BAD_ARG, "bad geometry or axis tables");
    return lshard(d->v.src_pos, d->v.kernel_len, d->src_h, d->dst_h, rank, nranks, info);
}

int lancirb200_shard_workspace_bytes(const lancirb200_plan* pl, int rank, int nranks, size_t* bytes) {
    if (!pl || !bytes) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    avirb200_shard_info si;
    const int r = lshard_plan(pl, rank, nranks, &si);
    if (r != 0) return r;
    *bytes = LShardWs(pl->desc, si).total;
    return 0;
}

int lancirb200_resize_sharded(const lancirb200_plan* cpl, void* comm, int rank, int nranks, const void* d_src,
                              size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_ws, void* stream) {
    if (!cpl || !d_src || !d_dst || !d_ws) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    avirb200_shard_info si;
    int r = lshard_plan(cpl, rank, nranks, &si);
    if (r == 0) r = lcheck(cpl, src_pitch, dst_pitch);
    if (r != 0) return r;
    if (nranks == 1) return lancirb200_resize_device(cpl, d_src, src_pitch, d_dst, dst_pitch, d_ws, stream);
    lancirb200_plan* pl = const_cast<lancirb200_plan*>(cpl); // (exchange state is created on first use)
    std::lock_guard<std::mutex> lk(pl->mx);
    return lsharded(pl, comm, rank, nranks, d_src, src_pitch, d_dst, dst_pitch, d_ws, static_cast<cudaStream_t>(stream));
}

int lancirb200_resize_sharded_host(lancirb200_plan* pl, void* comm, int rank, int nranks, const void* h_src,
                                   size_t src_pitch, void* h_dst, size_t dst_pitch) {
    if (!pl || !h_src || !h_dst) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const lancirb200_plan_desc& d = pl->desc;
    avirb200_shard_info si;
    const int r = lshard_plan(pl, rank, nranks, &si);
    if (r != 0) return r;
    const size_t sw = (size_t)d.src_w * d.channels, dw = (size_t)d.dst_w * d.channels;
    const avb::HostRect src = avb::host_rect(h_src, src_pitch, sw, elem_size(d.in_type), 0, sw, 0, si.src_rows);
    const avb::HostRect dst = avb::host_rect(h_dst, dst_pitch, dw, elem_size(d.out_type), 0, dw, 0, si.dst_rows);
    return avb::staged_call(pl->mx, pl->staging, pl->device, &pl->stream, src, dst, LShardWs(d, si).total,
                            [&](const void* s, void* o, void* w, cudaStream_t st) {
                                return nranks == 1 ? lancirb200_resize_device(pl, s, sw, o, dw, w, st)
                                                   : lsharded(pl, comm, rank, nranks, s, sw, o, dw, w, st);
                            });
}

int lancirb200_resize_sharded_local(const lancirb200_plan* cpl, int nranks, const void* d_src, size_t src_pitch,
                                    void* d_dst, size_t dst_pitch, void* d_ws, void* stream) {
    if (!cpl || !d_src || !d_dst || !d_ws) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (nranks < 1) return fail(AVIRB200_ERR_BAD_ARG, "bad rank");
    const lancirb200_plan_desc& d = cpl->desc;
    std::vector<avirb200_shard_info> si(nranks);
    std::vector<char*> ws(nranks);
    std::vector<LShardWs> wl;
    char* base = static_cast<char*>(d_ws);
    for (int r = 0; r < nranks; ++r) { // every band's workspace: as lancirb200_shard_workspace_bytes lays it out
        const int e = lshard_plan(cpl, r, nranks, &si[r]);
        if (e != 0) return e;
        wl.emplace_back(d, si[r]);
        ws[r] = base;
        base += wl[r].total;
    }
    int e = lcheck(cpl, src_pitch, dst_pitch);
    if (e != 0) return e;
    lancirb200_plan* pl = const_cast<lancirb200_plan*>(cpl); // (exchange state is created on first use)
    std::lock_guard<std::mutex> lk(pl->mx);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t in_el = elem_size(d.in_type), out_el = elem_size(d.out_type), el = in_el;
    const char* srcb = static_cast<const char*>(d_src);
    // The exchange of lancirb200_resize_sharded with every band's mailbox in its own workspace (the halo
    // segments and the header's flags, one slot): the same push on the exchange stream and the same segmented
    // column kernel waiting on the flags.  On the NCCL schedule (AVIRB200_OPT_OVERLAP_HALO = 0) the rows are
    // copied into the same segments before the column passes, which then do not wait.
    const bool box = pl->opt_overlap != 0 && nranks > 1;
    avb::PeerExchange& x = pl->x;
    cudaStream_t sx = st;
    if (box) {
        if ((e = x.pin()) != 0) return e;
        for (int r = 0; r < nranks; ++r) CUDA_TRY(cudaMemsetAsync(ws[r] + wl[r].header, 0, 8, st));
        if ((e = x.fork(st)) != 0) return e;
        sx = x.stream;
    }
    const unsigned* one = box ? x.one() : nullptr;
    for (int r = 0; r < nranks; ++r) {
        const avirb200_shard_info& b = si[r];
        char* flags = box ? ws[r] + wl[r].header : nullptr;
        // band r-1's last rows, then band r+1's first rows
        if (b.halo_up > 0 && (e = lpush_rows(pl, ws[r] + wl[r].up, srcb, src_pitch, b.need_row0, b.halo_up, flags, one, sx)) != 0)
            return e;
        if (b.halo_down > 0 && (e = lpush_rows(pl, ws[r] + wl[r].down, srcb, src_pitch, b.src_row0 + b.src_rows, b.halo_down,
                                               flags ? flags + 4 : nullptr, one, sx)) != 0)
            return e;
    }
    int r = 0;
    for (int q = 0; q < nranks && r == 0; ++q) {
        const avirb200_shard_info& b = si[q];
        LSeg s;
        std::memset(&s, 0, sizeof s);
        s.up = ws[q] + wl[q].up; s.dn = ws[q] + wl[q].down;
        s.up_pitch = s.dn_pitch = (long long)(lhalo_row_bytes(d) / el);
        if (box) {
            s.seq = 1;
            if (b.halo_up > 0) s.flag_up = reinterpret_cast<const volatile unsigned*>(ws[q] + wl[q].header);
            if (b.halo_down > 0) s.flag_dn = reinterpret_cast<const volatile unsigned*>(ws[q] + wl[q].header + 4);
        }
        r = lband(pl, b, srcb + (size_t)b.src_row0 * src_pitch * in_el, src_pitch,
                  static_cast<char*>(d_dst) + (size_t)b.dst_row0 * dst_pitch * out_el, dst_pitch, ws[q], s, st);
    }
    if (box && (e = x.join(st)) != 0) return e;
    return r;
}

} // extern "C"
