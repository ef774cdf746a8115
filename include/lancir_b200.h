// lancir_b200.h -- header-only drop-in front-end: avir::CLancIR on NVIDIA H100.
//
// Same public API as upstream lancir.h (CLancIRParams, CLancIR::resizeImage incl. the
// legacy overload; lancir.h:260-307, 386-390, 744-755).  The host designs the Lanczos
// fractional-delay filters and positions exactly as upstream does (double precision,
// 1/1000 phase quantisation); the two filtering passes (columns first, then rows) and the
// output conversion run as sm_90a kernels behind the C ABI in avirb200.h.
//
// Element types: uint8_t, uint16_t, float, double and uint32_t, for Tin and Tout alike (lancir.h:373-381).
//
// Bit-exact scope: upstream's AVX build.  Its tap-sum tree differs per channel count
// (resize1..resize4, lancir.h:2101-2515); the kernels mirror each of the four.
// There is no CPU fallback.

#ifndef LANCIR_B200_H
#define LANCIR_B200_H

#include <cmath>
#include <cstdint>
#include <cstring>
#include <type_traits>
#include <vector>

#include "avirb200.h"

#if defined(__clang__)
#pragma clang fp contract(off)
#elif defined(__GNUC__)
#pragma GCC push_options
#pragma GCC optimize("fp-contract=off")
#endif

#ifndef AVIRB200_NAMESPACE
#define AVIRB200_NAMESPACE avir
#endif

namespace AVIRB200_NAMESPACE {

// Upstream lancir.h:260-307.
class CLancIRParams {
public:
    int SrcSSize;
    int NewSSize;
    double kx;
    double ky;
    double ox;
    double oy;
    double la;

    CLancIRParams(const int aSrcSSize = 0, const int aNewSSize = 0, const double akx = 0.0,
                  const double aky = 0.0, const double aox = 0.0, const double aoy = 0.0)
        : SrcSSize(aSrcSSize), NewSSize(aNewSSize), kx(akx), ky(aky), ox(aox), oy(aoy), la(3.0) {}
};

namespace lancir_detail {

// Lanczos fractional-delay filter set for one axis; results must equal
// CLancIR::CResizeFilters (lancir.h:882-1156) before tap replication.
class FilterSet {
public:
    int kernel_len = 0;
    int half = 0; // fl2
    void configure(double la, double k) {
        const double norm = (k <= 1.0 ? 1.0 : 1.0 / k);
        freq_ = 3.1415926535897932 * norm;
        freq_a_ = freq_ / la;
        len2_ = la / norm;
        half = static_cast<int>(std::ceil(len2_));
        kernel_len = half + half;
        slot_.assign(kFrac + 1, -1);
        taps.clear();
        nphases = 0;
    }
    // Phase index for fractional offset x in [0,1): quantised to 1/1000 (lancir.h:940-967).
    int phase(double x) {
        const int fr = static_cast<int>(x * kFrac + 0.5);
        if (slot_[fr] < 0) {
            slot_[fr] = nphases++;
            taps.resize(static_cast<size_t>(nphases) * kernel_len);
            design(&taps[static_cast<size_t>(slot_[fr]) * kernel_len],
                   1.0 - static_cast<double>(fr) / kFrac);
        }
        return slot_[fr];
    }
    std::vector<float> taps;
    int nphases = 0;

private:
    static constexpr int kFrac = 1000;
    double freq_ = 0, freq_a_ = 0, len2_ = 0;
    std::vector<int> slot_;

    struct Osc { // lancir.h:1039-1057
        double cur, prev, coef;
        Osc(double step, double ph)
            : cur(std::sin(ph)), prev(std::sin(ph - step)), coef(2.0 * std::cos(step)) {}
        double next() {
            const double r = cur;
            cur = coef * r - prev;
            prev = r;
            return r;
        }
    };

    // lancir.h:1076-1156: sinc * sinc-window sampled at t + delay, t = -half .. half-1,
    // taps rounded to float before the DC sum, then normalised to unity DC.
    void design(float* op, double delay) const {
        Osc f(freq_, freq_ * (delay - half));
        Osc fw(freq_a_, freq_a_ * (delay - half));
        float* const op0 = op;
        double s = 0.0;
        int t = -half;
        if (t + delay < -len2_) {
            f.next(); fw.next();
            *op++ = 0.0f;
            ++t;
        }
        int zero_x = (std::fabs(delay - 1.0) < 2.3e-13) ? 1 : 0;
        int mt = 0 - zero_x;
        zero_x |= (std::fabs(delay) < 2.3e-13) ? 1 : 0;
        while (t < mt) {
            const double ut = t + delay;
            *op = static_cast<float>(f.next() * fw.next() / (ut * ut));
            s += *op;
            ++op; ++t;
        }
        if (zero_x) {
            *op = static_cast<float>(freq_ * freq_a_);
            s += *op;
            f.next(); fw.next();
        } else {
            const double ut = delay;
            *op = static_cast<float>(f.next() * fw.next() / (ut * ut));
            s += *op;
        }
        mt = half - 2;
        while (t < mt) {
            ++op; ++t;
            const double ut = t + delay;
            *op = static_cast<float>(f.next() * fw.next() / (ut * ut));
            s += *op;
        }
        ++op;
        const double ut = t + 1 + delay;
        if (ut > len2_) {
            *op = 0.0f;
        } else {
            *op = static_cast<float>(f.next() * fw.next() / (ut * ut));
            s += *op;
        }
        s = 1.0 / s;
        for (float* p = op0; p <= op; ++p) *p = static_cast<float>(*p * s);
    }
};

struct AxisTables {
    std::vector<int32_t> src_pos, phase;
};

// Per-output source index of the first tap and phase (lancir.h:1290-1351).
inline void positions(AxisTables& at, FilterSet& fs, int dst_len, double o, double k) {
    at.src_pos.resize(dst_len);
    at.phase.resize(dst_len);
    for (int i = 0; i < dst_len; ++i) {
        const double ox = o + k * i;
        const int ix = static_cast<int>(std::floor(ox));
        at.phase[i] = fs.phase(ox - ix);
        at.src_pos[i] = ix - (fs.half - 1);
    }
}

// Buffer element types (upstream lancir.h:373-381): uint8_t, uint16_t, float, double, and uint32_t, which
// upstream treats as uint16_t.  Upstream leaves signed and larger integer types unsupported (they compile
// there and give garbage); here they do not compile.
template <typename T> struct dtype_of {
    static_assert(sizeof(T) == 0,
                  "CLancIR element types are uint8_t, uint16_t, float, double and uint32_t (lancir.h:373-381)");
    static constexpr int value = -1;
};
template <> struct dtype_of<uint8_t> { static constexpr int value = AVIRB200_U8; };
template <> struct dtype_of<uint16_t> { static constexpr int value = AVIRB200_U16; };
template <> struct dtype_of<float> { static constexpr int value = AVIRB200_F32; };
template <> struct dtype_of<double> { static constexpr int value = AVIRB200_F64; };
template <> struct dtype_of<uint32_t> { static constexpr int value = AVIRB200_U32; };

} // namespace lancir_detail

class CLancIR {
public:
    CLancIR() {}
    ~CLancIR() { if (Plan != nullptr) lancirb200_plan_destroy(Plan); }
    CLancIR(const CLancIR&) = delete;
    CLancIR& operator=(const CLancIR&) = delete;

    // Upstream lancir.h:386-390.  Returns NewHeight, or 0 on a parameter error (upstream's
    // convention) and on configurations the GPU path does not cover (see file header).
    template <typename Tin, typename Tout>
    int resizeImage(const Tin* const SrcBuf, const int SrcWidth, const int SrcHeight,
                    Tout* const NewBuf, const int NewWidth, const int NewHeight, const int ElCount,
                    const CLancIRParams* const aParams = nullptr) {
        if ((SrcWidth < 0) | (SrcHeight < 0) | (NewWidth <= 0) | (NewHeight <= 0) |
            (SrcBuf == nullptr) | (NewBuf == nullptr) | ((const void*)SrcBuf == (const void*)NewBuf))
            return 0; // lancir.h:392-399
        static const CLancIRParams DefParams;
        const CLancIRParams& Params = (aParams != nullptr ? *aParams : DefParams);
        if (Params.la < 2.0) return 0; // lancir.h:405-408
        const int OutSLen = NewWidth * ElCount;
        const size_t NewScanlineSize = (size_t)(Params.NewSSize < 1 ? OutSLen : Params.NewSSize);
        if ((SrcWidth == 0) | (SrcHeight == 0)) { // lancir.h:414-426
            Tout* op = NewBuf;
            for (int i = 0; i < NewHeight; i++) {
                std::memset(op, 0, (size_t)OutSLen * sizeof(Tout));
                op += NewScanlineSize;
            }
            return NewHeight;
        }
        const size_t SrcScanlineSize =
            (size_t)(Params.SrcSSize < 1 ? SrcWidth * ElCount : Params.SrcSSize);
        if (!ensurePlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCount, Params))
            return 0;
        if (lancirb200_resize_host(Plan, SrcBuf, SrcScanlineSize, NewBuf, NewScanlineSize) != 0)
            return 0;
        return NewHeight;
    }

    // Legacy overload, upstream lancir.h:744-755.
    template <typename Tin, typename Tout>
    int resizeImage(const Tin* const SrcBuf, const int SrcWidth, const int SrcHeight,
                    const int SrcSSize, Tout* const NewBuf, const int NewWidth,
                    const int NewHeight, const int NewSSize, const int ElCount,
                    const double kx0 = 0.0, const double ky0 = 0.0, double ox = 0.0,
                    double oy = 0.0) {
        const CLancIRParams Params(SrcSSize, NewSSize, kx0, ky0, ox, oy);
        return resizeImage(SrcBuf, SrcWidth, SrcHeight, NewBuf, NewWidth, NewHeight, ElCount,
                           &Params);
    }

    // GPU extension: the destination window [WinX, WinX + WinWidth) x [WinY, WinY + WinHeight) of
    // resizeImage(SrcBuf, SrcWidth, SrcHeight, NewBuf, NewWidth, NewHeight, ElCount, aParams), bit for
    // bit, reading only the window's source footprint (windowFootprint).  SrcBuf is the WHOLE source
    // (Params.SrcSSize its scanline size), NewBuf receives the window (Params.NewSSize its scanline
    // size, < 1: WinWidth * ElCount).  Returns WinHeight, or 0 as resizeImage does and for a window
    // that is empty or not inside the destination.  Every window of one geometry shares the plan
    // resizeImage caches.
    template <typename Tin, typename Tout>
    int resizeImageWindow(const Tin* const SrcBuf, const int SrcWidth, const int SrcHeight,
                          Tout* const NewBuf, const int NewWidth, const int NewHeight, const int ElCount,
                          const int WinX, const int WinY, const int WinWidth, const int WinHeight,
                          const CLancIRParams* const aParams = nullptr) {
        if ((SrcBuf == nullptr) | ((const void*)SrcBuf == (const void*)NewBuf) ||
            !windowArgs(SrcWidth, SrcHeight, NewBuf, NewWidth, NewHeight, WinX, WinY, WinWidth, WinHeight, aParams))
            return 0;
        const CLancIRParams& Params = params(aParams);
        const size_t NewScanlineSize =
            (size_t)(Params.NewSSize < 1 ? WinWidth * ElCount : Params.NewSSize);
        if ((SrcWidth == 0) | (SrcHeight == 0)) { // lancir.h:414-426, for the window's pixels
            Tout* op = NewBuf;
            for (int i = 0; i < WinHeight; i++) {
                std::memset(op, 0, (size_t)WinWidth * ElCount * sizeof(Tout));
                op += NewScanlineSize;
            }
            return WinHeight;
        }
        const size_t SrcScanlineSize =
            (size_t)(Params.SrcSSize < 1 ? SrcWidth * ElCount : Params.SrcSSize);
        if (!ensurePlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCount, Params))
            return 0;
        if (lancirb200_resize_window_host(Plan, WinX, WinY, WinWidth, WinHeight, SrcBuf, SrcScanlineSize, NewBuf,
                                          NewScanlineSize) != 0)
            return 0;
        return WinHeight;
    }

    // The same with DEVICE pointers, asynchronous on `Stream` (a cudaStream_t): dSrcBuf points at the
    // footprint's first pixel and holds its src_w x src_h pixels (Params.SrcSSize elements apart, < 1:
    // src_w * ElCount), dNewBuf receives the window, `Workspace` holds windowWorkspaceBytes() bytes of
    // device memory.  Returns WinHeight or 0; an empty source has no footprint and returns 0.
    template <typename Tin, typename Tout>
    int resizeImageWindowDevice(const Tin* const dSrcBuf, const int SrcWidth, const int SrcHeight,
                                Tout* const dNewBuf, const int NewWidth, const int NewHeight, const int ElCount,
                                const int WinX, const int WinY, const int WinWidth, const int WinHeight,
                                void* const Workspace, void* const Stream = nullptr,
                                const CLancIRParams* const aParams = nullptr) {
        lancirb200_window_info wi;
        if ((dSrcBuf == nullptr) | ((const void*)dSrcBuf == (const void*)dNewBuf) | (Workspace == nullptr) ||
            windowFootprint<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCount, WinX, WinY, WinWidth,
                                       WinHeight, &wi, aParams) == 0)
            return 0;
        const CLancIRParams& Params = params(aParams);
        const size_t SrcScanlineSize = (size_t)(Params.SrcSSize < 1 ? wi.src_w * ElCount : Params.SrcSSize);
        const size_t NewScanlineSize = (size_t)(Params.NewSSize < 1 ? WinWidth * ElCount : Params.NewSSize);
        if (lancirb200_resize_window_device(Plan, WinX, WinY, WinWidth, WinHeight, dSrcBuf, SrcScanlineSize, dNewBuf,
                                            NewScanlineSize, Workspace, Stream) != 0)
            return 0;
        return WinHeight;
    }

    // The source pixels a window reads (clamped to the image) into *Info.  Returns WinHeight or 0.
    template <typename Tin, typename Tout>
    int windowFootprint(const int SrcWidth, const int SrcHeight, const int NewWidth, const int NewHeight,
                        const int ElCount, const int WinX, const int WinY, const int WinWidth, const int WinHeight,
                        lancirb200_window_info* const Info, const CLancIRParams* const aParams = nullptr) {
        if ((Info == nullptr) | (SrcWidth < 1) | (SrcHeight < 1) ||
            !windowArgs(SrcWidth, SrcHeight, Info, NewWidth, NewHeight, WinX, WinY, WinWidth, WinHeight, aParams) ||
            !ensurePlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCount, params(aParams)) ||
            lancirb200_window_query(Plan, WinX, WinY, WinWidth, WinHeight, Info) != 0)
            return 0;
        return WinHeight;
    }

    // Bytes of device workspace resizeImageWindowDevice needs for the window, or 0 where it would
    // return 0.
    template <typename Tin, typename Tout>
    size_t windowWorkspaceBytes(const int SrcWidth, const int SrcHeight, const int NewWidth, const int NewHeight,
                                const int ElCount, const int WinX, const int WinY, const int WinWidth,
                                const int WinHeight, const CLancIRParams* const aParams = nullptr) {
        lancirb200_window_info wi;
        size_t b = 0;
        if (windowFootprint<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCount, WinX, WinY, WinWidth,
                                       WinHeight, &wi, aParams) == 0 ||
            lancirb200_window_workspace_bytes(Plan, WinX, WinY, WinWidth, WinHeight, &b) != 0)
            return 0;
        return b;
    }

    // Host-only: fills the C descriptor for a call (tables owned by *this).
    template <typename Tin, typename Tout>
    bool buildDescriptor(lancirb200_plan_desc& d, const int SrcWidth, const int SrcHeight,
                         const int NewWidth, const int NewHeight, const int ElCount,
                         const CLancIRParams& Params) {
        double ox = Params.ox, oy = Params.oy, kx, ky; // lancir.h:430-457
        if (Params.kx >= 0.0) {
            kx = (Params.kx == 0.0 ? (double)SrcWidth / NewWidth : Params.kx);
            ox += (kx - 1.0) * 0.5;
        } else {
            kx = -Params.kx;
        }
        if (Params.ky >= 0.0) {
            ky = (Params.ky == 0.0 ? (double)SrcHeight / NewHeight : Params.ky);
            oy += (ky - 1.0) * 0.5;
        } else {
            ky = -Params.ky;
        }
        FltV.configure(Params.la, ky);
        lancir_detail::positions(TabV, FltV, NewHeight, oy, ky);
        FltH.configure(Params.la, kx);
        lancir_detail::positions(TabH, FltH, NewWidth, ox, kx);

        std::memset(&d, 0, sizeof(d));
        d.src_w = SrcWidth; d.src_h = SrcHeight; d.dst_w = NewWidth; d.dst_h = NewHeight;
        d.channels = ElCount;
        d.in_type = lancir_detail::dtype_of<Tin>::value;
        d.out_type = lancir_detail::dtype_of<Tout>::value;
        const bool InF = std::is_floating_point<Tin>::value;
        const bool OutF = std::is_floating_point<Tout>::value;
        // lancir.h:521-533
        d.is_unity_mul = ((InF && OutF) || (InF == OutF && sizeof(Tin) == sizeof(Tout))) ? 1 : 0;
        const float Clamp = (sizeof(Tout) == 1 ? 255.0f : 65535.0f);
        d.clamp_max = Clamp;
        d.out_mul = (OutF ? 1.0f : Clamp) / (InF ? 1.0f : (sizeof(Tin) == 1 ? 255.0f : 65535.0f));
        fill(d.v, FltV, TabV, SrcHeight, NewHeight);
        fill(d.h, FltH, TabH, SrcWidth, NewWidth);
        return true;
    }

private:
    lancirb200_plan* Plan = nullptr;
    lancir_detail::FilterSet FltV, FltH;
    lancir_detail::AxisTables TabV, TabH;
    struct Key {
        int tin, tout, sw, sh, nw, nh, c;
        double kx, ky, ox, oy, la;
        bool operator==(const Key& o) const {
            return tin == o.tin && tout == o.tout && sw == o.sw && sh == o.sh && nw == o.nw &&
                   nh == o.nh && c == o.c && kx == o.kx && ky == o.ky && ox == o.ox && oy == o.oy &&
                   la == o.la;
        }
    } Cur{-1, -1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};

    static const CLancIRParams& params(const CLancIRParams* const aParams) {
        static const CLancIRParams DefParams;
        return aParams != nullptr ? *aParams : DefParams;
    }

    // resizeImage's argument rules (lancir.h:392-408) for the window calls, plus a non-empty window
    // inside the destination.
    static bool windowArgs(const int SrcWidth, const int SrcHeight, const void* const NewBuf, const int NewWidth,
                           const int NewHeight, const int WinX, const int WinY, const int WinWidth,
                           const int WinHeight, const CLancIRParams* const aParams) {
        if ((SrcWidth < 0) | (SrcHeight < 0) | (NewWidth <= 0) | (NewHeight <= 0) | (NewBuf == nullptr))
            return false;
        if ((WinX < 0) | (WinY < 0) | (WinWidth <= 0) | (WinHeight <= 0) | (WinX > NewWidth - WinWidth) |
            (WinY > NewHeight - WinHeight))
            return false;
        return params(aParams).la >= 2.0;
    }

    static void fill(lancirb200_axis_desc& a, const lancir_detail::FilterSet& f,
                     const lancir_detail::AxisTables& t, int src_len, int dst_len) {
        a.src_len = src_len; a.dst_len = dst_len;
        a.kernel_len = f.kernel_len; a.nphases = f.nphases;
        a.taps = f.taps.data(); a.src_pos = t.src_pos.data(); a.phase = t.phase.data();
    }

    // Upstream caches filters and positions between calls with equal geometry
    // (lancir.h:459-483); here the whole device plan is kept.
    template <typename Tin, typename Tout>
    bool ensurePlan(const int SrcWidth, const int SrcHeight, const int NewWidth,
                    const int NewHeight, const int ElCount, const CLancIRParams& Params) {
        const Key k{lancir_detail::dtype_of<Tin>::value, lancir_detail::dtype_of<Tout>::value,
                    SrcWidth, SrcHeight, NewWidth, NewHeight, ElCount,
                    Params.kx, Params.ky, Params.ox, Params.oy, Params.la};
        if (Plan != nullptr && k == Cur) return true;
        if (Plan != nullptr) { lancirb200_plan_destroy(Plan); Plan = nullptr; }
        lancirb200_plan_desc d;
        if (!buildDescriptor<Tin, Tout>(d, SrcWidth, SrcHeight, NewWidth, NewHeight, ElCount, Params))
            return false;
        if (lancirb200_plan_create(&d, &Plan) != 0) { Plan = nullptr; return false; }
        Cur = k;
        return true;
    }
};

} // namespace AVIRB200_NAMESPACE

#if defined(__GNUC__) && !defined(__clang__)
#pragma GCC pop_options
#endif

#endif // LANCIR_B200_H
