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

#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "avirb200.h"
#include "host_util.h"

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
    float* mid;          // [dst_h][src_w*C]
    void* dst; long long dst_pitch;
};

__device__ __forceinline__ float lload(const void* p, int type, long long i) {
    if (type == AVIRB200_U8) return (float)((const unsigned char*)p)[i];
    if (type == AVIRB200_U16) return (float)((const unsigned short*)p)[i];
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

// Column pass: one thread per (x, c) element of an output row; grid.y = output row.
__global__ void __launch_bounds__(256) lancir_col_kernel(const __grid_constant__ LParams p) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x; // element within a row
    const int y = blockIdx.y;
    const int row_elems = p.src_w * p.C;
    if (e >= row_elems) return;
    const int kl = p.v.kl;
    const float* f = p.v.taps + (size_t)__ldg(p.v.phase + y) * kl;
    const int s0 = __ldg(p.v.src_pos + y);
    const void* src = p.src;
    const int in_type = p.in_type, src_h = p.src_h;
    const long long pitch = p.src_pitch;
    const float r = ltapsum(p.C, e % p.C, kl, f, [&](int t) {
        int sy = s0 + t;
        sy = sy < 0 ? 0 : (sy >= src_h ? src_h - 1 : sy);
        return lload(src, in_type, (long long)sy * pitch + e);
    });
    p.mid[(size_t)y * row_elems + e] = r;
}

// Row pass + output: one thread per output element; grid.y = row.
__global__ void __launch_bounds__(256) lancir_row_kernel(const __grid_constant__ LParams p) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    const int out_elems = p.dst_w * p.C;
    if (e >= out_elems) return;
    const int x = e / p.C, c = e - x * p.C;
    const int kl = p.h.kl;
    const float* f = p.h.taps + (size_t)__ldg(p.h.phase + x) * kl;
    const int s0 = __ldg(p.h.src_pos + x);
    const float* row = p.mid + (size_t)y * p.src_w * p.C;
    const int C = p.C, src_w = p.src_w;
    float v = ltapsum(C, c, kl, f, [&](int t) {
        int sx = s0 + t;
        sx = sx < 0 ? 0 : (sx >= src_w ? src_w - 1 : sx);
        return row[(size_t)sx * C + c];
    });
    if (!p.unity) v = __fmul_rn(v, p.out_mul);
    const long long g = (long long)y * p.dst_pitch + e;
    if (p.out_type == AVIRB200_F32) {
        ((float*)p.dst)[g] = v;
        return;
    }
    int iv;
    const bool tail = e >= (out_elems & ~3);
    if (tail) {
        const float cv = v > p.clamp_max ? p.clamp_max : (v < 0.0f ? 0.0f : v);
        iv = __float2int_rz(__fadd_rn(cv, 0.5f));
    } else {
        const float cv = fmaxf(fminf(v, p.clamp_max), 0.0f);
        iv = __float2int_rn(cv);
    }
    if (p.out_type == AVIRB200_U8) ((unsigned char*)p.dst)[g] = (unsigned char)iv;
    else ((unsigned short*)p.dst)[g] = (unsigned short)iv;
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

__device__ __forceinline__ float4 lmul4(float f, float4 v) {
    return make_float4(__fmul_rn(f, v.x), __fmul_rn(f, v.y), __fmul_rn(f, v.z), __fmul_rn(f, v.w));
}
__device__ __forceinline__ float4 ladd4(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

constexpr int kLColRows = 32; // output rows a block of the column pass walks

// KL: compile-time kernel length (all taps' loads of an output are issued before the first
// product: the loop is unrolled) for the common lengths, 0 = run-time length.
template <typename TIN, int KL>
__global__ void __launch_bounds__(256) lancir_col4_kernel(const __grid_constant__ LParams p) {
    const int px = blockIdx.x * 256 + threadIdx.x;
    if (px >= p.src_w) return;
    const int y0 = blockIdx.y * kLColRows;
    const int y1 = (y0 + kLColRows < p.dst_h) ? y0 + kLColRows : p.dst_h;
    const int kl = KL ? KL : p.v.kl, src_h = p.src_h;
    const long long pitch = p.src_pitch;
    for (int y = y0; y < y1; ++y) {
        const float* f = p.v.taps + (size_t)__ldg(p.v.phase + y) * kl;
        const int s0 = __ldg(p.v.src_pos + y);
        auto S = [&](int t) {
            int sy = s0 + t;
            sy = sy < 0 ? 0 : (sy >= src_h ? src_h - 1 : sy);
            return LPix<TIN>::load(p.src, (long long)sy * pitch + (long long)px * 4);
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
        reinterpret_cast<float4*>(p.mid + (size_t)y * p.src_w * 4)[px] = ladd4(ev, od);
    }
}

// OUT: 0 float, 1 u8, 2 u16
template <int OUT, int KL>
__global__ void __launch_bounds__(256) lancir_row4_kernel(const __grid_constant__ LParams p) {
    const int x = blockIdx.x * 256 + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= p.dst_w) return;
    const int kl = KL ? KL : p.h.kl, src_w = p.src_w;
    const float* f = p.h.taps + (size_t)__ldg(p.h.phase + x) * kl;
    const int s0 = __ldg(p.h.src_pos + x);
    const float4* row = reinterpret_cast<const float4*>(p.mid + (size_t)y * src_w * 4);
    auto M = [&](int t) {
        int sx = s0 + t;
        sx = sx < 0 ? 0 : (sx >= src_w ? src_w - 1 : sx);
        return row[sx];
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
    // (a row of 4-channel pixels has no (NewWidth*C) & 3 tail: every element rounds nearest-even)
    const float cm = p.clamp_max;
    const int a = __float2int_rn(fmaxf(fminf(v.x, cm), 0.0f)), b = __float2int_rn(fmaxf(fminf(v.y, cm), 0.0f));
    const int c = __float2int_rn(fmaxf(fminf(v.z, cm), 0.0f)), d = __float2int_rn(fmaxf(fminf(v.w, cm), 0.0f));
    if (OUT == 1)
        *reinterpret_cast<uchar4*>(static_cast<unsigned char*>(p.dst) + g) =
            make_uchar4((unsigned char)a, (unsigned char)b, (unsigned char)c, (unsigned char)d);
    else
        *reinterpret_cast<ushort4*>(static_cast<unsigned short*>(p.dst) + g) =
            make_ushort4((unsigned short)a, (unsigned short)b, (unsigned short)c, (unsigned short)d);
}

} // namespace

struct lancirb200_plan {
    lancirb200_plan_desc desc;
    void* arena = nullptr;
    LAxis dv, dh;
    int device = 0;
    std::mutex mx;
    void* d_src = nullptr;
    void* d_dst = nullptr;
    void* d_ws = nullptr;
    size_t src_bytes = 0, dst_bytes = 0, ws_bytes = 0;
    cudaStream_t stream = nullptr;
};

extern "C" {

int lancirb200_plan_create(const lancirb200_plan_desc* d, lancirb200_plan** out) {
    if (d == nullptr || out == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    if (d->channels < 1 || d->channels > 4) return fail(AVIRB200_ERR_BAD_ARG, "channels must be 1..4");
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
    pl->desc.v.taps = nullptr; pl->desc.h.taps = nullptr;
    *out = pl.release();
    return 0;
}

void lancirb200_plan_destroy(lancirb200_plan* pl) {
    if (!pl) return;
    cudaFree(pl->arena); cudaFree(pl->d_src); cudaFree(pl->d_dst); cudaFree(pl->d_ws);
    if (pl->stream) cudaStreamDestroy(pl->stream);
    delete pl;
}

int lancirb200_plan_workspace_bytes(const lancirb200_plan* pl, size_t* bytes) {
    if (!pl || !bytes) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    *bytes = (size_t)pl->desc.dst_h * pl->desc.src_w * pl->desc.channels * sizeof(float);
    return 0;
}

int lancirb200_resize_device(const lancirb200_plan* pl, const void* d_src, size_t src_pitch,
                             void* d_dst, size_t dst_pitch, void* d_ws, void* stream) {
    if (!pl || !d_src || !d_dst || !d_ws) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const lancirb200_plan_desc& d = pl->desc;
    LParams p;
    p.v = pl->dv; p.h = pl->dh;
    p.src_w = d.src_w; p.src_h = d.src_h; p.dst_w = d.dst_w; p.dst_h = d.dst_h; p.C = d.channels;
    p.in_type = d.in_type; p.out_type = d.out_type;
    p.out_mul = d.out_mul; p.clamp_max = d.clamp_max; p.unity = d.is_unity_mul;
    p.src = d_src; p.src_pitch = (long long)src_pitch;
    p.mid = static_cast<float*>(d_ws);
    p.dst = d_dst; p.dst_pitch = (long long)dst_pitch;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (d.dst_h > 65535) return fail(AVIRB200_ERR_UNSUPPORTED, "image too tall");
    (void)cudaGetLastError(); // (a stale non-sticky error of another library is not this launch's)
    // 4-channel images whose pixels are aligned to their own size: the vector kernels
    const bool vec_in = d.channels == 4 && (src_pitch % 4) == 0 && ((uintptr_t)d_src % (4 * elem_size(d.in_type))) == 0 &&
                        ((uintptr_t)d_ws % 16) == 0;
    const bool vec_out = d.channels == 4 && (dst_pitch % 4) == 0 && ((uintptr_t)d_dst % (4 * elem_size(d.out_type))) == 0 &&
                         ((uintptr_t)d_ws % 16) == 0;
    if (vec_in) {
        dim3 g1((d.src_w + 255) / 256, (d.dst_h + kLColRows - 1) / kLColRows);
#define LCOL(KL)                                                                                        \
    do {                                                                                                \
        if (d.in_type == AVIRB200_U8) lancir_col4_kernel<unsigned char, KL><<<g1, 256, 0, st>>>(p);     \
        else if (d.in_type == AVIRB200_U16) lancir_col4_kernel<unsigned short, KL><<<g1, 256, 0, st>>>(p); \
        else lancir_col4_kernel<float, KL><<<g1, 256, 0, st>>>(p);                                      \
    } while (0)
        switch (pl->dv.kl) { // la = 3: 6 taps when upsizing, 12 at k = 2, 18 at k = 3, 24 at k = 4
        case 6: LCOL(6); break;
        case 12: LCOL(12); break;
        case 18: LCOL(18); break;
        case 24: LCOL(24); break;
        default: LCOL(0); break;
        }
#undef LCOL
    } else {
        dim3 g1((d.src_w * d.channels + 255) / 256, d.dst_h);
        lancir_col_kernel<<<g1, 256, 0, st>>>(p);
    }
    if (vec_out) {
        dim3 g2((d.dst_w + 255) / 256, d.dst_h);
#define LROW(KL)                                                                                        \
    do {                                                                                                \
        if (d.out_type == AVIRB200_U8) lancir_row4_kernel<1, KL><<<g2, 256, 0, st>>>(p);                \
        else if (d.out_type == AVIRB200_U16) lancir_row4_kernel<2, KL><<<g2, 256, 0, st>>>(p);          \
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
        dim3 g2((d.dst_w * d.channels + 255) / 256, d.dst_h);
        lancir_row_kernel<<<g2, 256, 0, st>>>(p);
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int lancirb200_resize_host(lancirb200_plan* pl, const void* h_src, size_t src_pitch, void* h_dst,
                           size_t dst_pitch) {
    if (!pl || !h_src || !h_dst) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const lancirb200_plan_desc& d = pl->desc;
    std::lock_guard<std::mutex> lk(pl->mx);
    CUDA_TRY(cudaSetDevice(pl->device));
    const size_t in_row = (size_t)d.src_w * d.channels * elem_size(d.in_type);
    const size_t out_row = (size_t)d.dst_w * d.channels * elem_size(d.out_type);
    size_t ws = 0;
    lancirb200_plan_workspace_bytes(pl, &ws);
    if (!pl->stream) CUDA_TRY(cudaStreamCreateWithFlags(&pl->stream, cudaStreamNonBlocking));
    if (pl->src_bytes < in_row * d.src_h) {
        cudaFree(pl->d_src); pl->d_src = nullptr; pl->src_bytes = 0;
        CUDA_TRY(cudaMalloc(&pl->d_src, in_row * d.src_h)); pl->src_bytes = in_row * d.src_h;
    }
    if (pl->dst_bytes < out_row * d.dst_h) {
        cudaFree(pl->d_dst); pl->d_dst = nullptr; pl->dst_bytes = 0;
        CUDA_TRY(cudaMalloc(&pl->d_dst, out_row * d.dst_h)); pl->dst_bytes = out_row * d.dst_h;
    }
    if (pl->ws_bytes < ws) {
        cudaFree(pl->d_ws); pl->d_ws = nullptr; pl->ws_bytes = 0;
        CUDA_TRY(cudaMalloc(&pl->d_ws, ws)); pl->ws_bytes = ws;
    }
    CUDA_TRY(cudaMemcpy2DAsync(pl->d_src, in_row, h_src, src_pitch * elem_size(d.in_type), in_row,
                                d.src_h, cudaMemcpyHostToDevice, pl->stream));
    int r = lancirb200_resize_device(pl, pl->d_src, (size_t)d.src_w * d.channels, pl->d_dst,
                                     (size_t)d.dst_w * d.channels, pl->d_ws, pl->stream);
    if (r != 0) return r;
    CUDA_TRY(cudaMemcpy2DAsync(h_dst, dst_pitch * elem_size(d.out_type), pl->d_dst, out_row, out_row,
                                d.dst_h, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    return 0;
}

} // extern "C"
